"""Scoring, top-N and evaluation kernels (csrc/score.cu, csrc/eval.cu) against fp64 numpy references, at the shapes and
values where such kernels go wrong: cutoffs at and above the row length, 200 K-item rows, heavy ties, rows that are
mostly -inf, non-finite and signed-zero scores, up to 1 536 factors, user blocks that do not fill a CTA, more rows than
the grid, and launches past the 65 535 limit of gridDim.y.  The kernels are called through the C ABI with torch device
tensors; the evaluator runs through EvaluatorHoldout against oracle.evaluator_oracle.evaluate_scores, and the ranking
contract through recommend() -- `-m gpu`.

The ranking contract (BaseRecommender.py:189-207, oracle/evaluator_oracle.py) is np.lexsort((arange, -s)): +inf, finite
scores descending, -inf, NaN, ties by ascending item (-0 and +0 tie); only finite entries of the first `cutoff`
positions are recommendations."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.evaluator_oracle import evaluate_scores
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_evaluation import _stub

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24  # unit roundoff of fp32


def _L():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan_like(shape, dtype=None):
    import torch
    return torch.full(shape, float("nan"), dtype=dtype or torch.float32, device="cuda")


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _sm_count():
    return _L().device_info()[1]


def _order(s):
    return np.lexsort((np.arange(len(s)), -np.asarray(s, np.float64)))


# ------------------------------------------------------------------------------------------------------------ top-N
def _topn(S, cutoff):
    import torch
    L = _L()
    d = _dev(S)
    items = torch.full((S.shape[0], cutoff), -7, dtype=torch.int32, device="cuda")
    vals = _nan_like((S.shape[0], cutoff))
    L.check(L.load().b200_score_topn_device(d.data_ptr(), S.shape[0], S.shape[1], cutoff, items.data_ptr(), vals.data_ptr(),
                                            _stream()))
    return items.cpu().numpy(), vals.cpu().numpy()


def _check_topn(S, orders, cutoff):
    """Item ids exact, scores bitwise; past the end of a row -1 / -inf."""
    items, vals = _topn(S, cutoff)
    bad = []
    for r, o in enumerate(orders):
        o = o[:cutoff]
        want_items = np.full(cutoff, -1, np.int32)
        want_vals = np.full(cutoff, -np.inf, np.float32)
        want_items[:len(o)] = o
        want_vals[:len(o)] = S[r, o]
        if not (np.array_equal(items[r], want_items) and np.array_equal(vals[r].view(np.uint32), want_vals.view(np.uint32))):
            bad.append(r)
    assert not bad, "cutoff %d: rows %s differ from the lexsort ranking" % (cutoff, bad)


def _score_rows(n, rng):
    """One row per score family, float32 [n_rows, n]."""
    rows = [rng.standard_normal(n).astype(np.float32),                              # continuous
            rng.integers(0, 3, n).astype(np.float32),                               # values in {0, 1, 2}: massive ties
            np.full(n, 0.25, np.float32),                                           # all equal
            (-rng.random(n) * 100 - 1e-3).astype(np.float32)]                       # all negative
    base = np.where(rng.random(n) < 0.5, 0x3F800000, 0xBF800000).astype(np.uint32)  # +-1 and neighbours one ulp apart
    rows.append((base + rng.integers(0, 40, n).astype(np.uint32)).view(np.float32))
    for k in (0, 1, 5, 600, 1000):  # all but k items at -inf (k < cutoff for some cutoffs, > for others)
        s = np.full(n, -np.inf, np.float32)
        s[rng.choice(n, min(k, n), replace=False)] = rng.integers(-1, 2, min(k, n))
        rows.append(s)
    s = rng.standard_normal(n).astype(np.float32)  # NaN, +inf and -inf mixed in, NaNs of both signs and with a payload
    u = rng.random(n)
    s[u < 0.1] = np.nan
    s[(u >= 0.1) & (u < 0.2)] = np.inf
    s[(u >= 0.2) & (u < 0.3)] = -np.inf
    bits = s.view(np.uint32)
    bits[(u >= 0.3) & (u < 0.33)] = 0xFFC00000
    bits[(u >= 0.33) & (u < 0.36)] = 0x7FC00001
    rows.append(s)
    rows.append(rng.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), n))  # signed zeros tie
    return np.stack(rows)


@pytest.mark.parametrize("n_items", [1, 2, 1023, 1024, 1025, 50_000, 200_000])
def test_topn_matches_lexsort(n_items):
    rng = np.random.default_rng(n_items)
    S = _score_rows(n_items, rng)
    orders = [_order(s) for s in S]
    for cutoff in (1, 7, 1023, 1024):
        _check_topn(S, orders, cutoff)


def test_topn_more_rows_than_the_grid():
    """sm_count * 8 CTAs walk the rows grid-stride; every row is different, some mostly -inf."""
    rng = np.random.default_rng(5)
    n_rows, n_items = 2 * 8 * _sm_count() + 5, 1500
    S = rng.integers(0, 50, (n_rows, n_items)).astype(np.float32)
    S[::7, 3:] = -np.inf
    orders = [_order(s) for s in S]
    for cutoff in (7, 1024):
        _check_topn(S, orders, cutoff)


def test_topn_rejects_cutoff_out_of_range():
    S = np.zeros((2, 10), np.float32)
    for cutoff in (0, 1025):
        with pytest.raises(ValueError):
            _topn(S, cutoff)


# ------------------------------------------------------------------------------------------- MF scores and transpose
def _transpose(d_in):
    import torch
    L = _L()
    rows, cols = d_in.shape
    out = torch.full((cols, rows), float("nan"), dtype=torch.float32, device="cuda")
    L.check(L.load().b200_transpose_device(d_in.data_ptr(), rows, cols, out.data_ptr(), _stream()))
    return out


def _mf(users, d_U, d_VT, biases=None):
    L = _L()
    f, n_items = d_VT.shape
    d_users = _dev(np.asarray(users, np.int32))
    out = _nan_like((len(users), n_items))
    bu, bi, mu = (None, None, None) if biases is None else biases
    L.check(L.load().b200_score_mf_device(d_users.data_ptr(), len(users), d_U.data_ptr(), d_VT.data_ptr(), f, n_items,
                                          _ptr(bu), _ptr(bi), _ptr(mu), out.data_ptr(), _stream()))
    return out.cpu().numpy()


def _user_block(rng, n_users, size):
    """`size` users in no particular order, one of them twice when size >= 3."""
    u = rng.permutation(n_users)[:size]
    if size >= 3:
        u[2] = u[0]
    return u


def _mf_case(rng, f, n_items, integer):
    n_users = 40
    draw = (lambda *s: rng.integers(-3, 4, s)) if integer else (lambda *s: rng.standard_normal(s))
    U, V = draw(n_users, f).astype(np.float32), draw(n_items, f).astype(np.float32)
    bu, bi, mu = draw(n_users).astype(np.float32), draw(n_items).astype(np.float32), draw(1).astype(np.float32)
    d_U, d_V = _dev(U), _dev(V)
    d_VT = _transpose(d_V)
    assert np.array_equal(d_VT.cpu().numpy(), V.T)
    return U, V, (bu, bi, mu), d_U, d_VT, tuple(_dev(b) for b in (bu, bi, mu))


def _mf_ref(U, V, biases, users, with_bias):
    ref = U[users].astype(np.float64) @ V.T.astype(np.float64)
    if with_bias:
        bu, bi, mu = (b.astype(np.float64) for b in biases)
        ref += mu[0] + bu[users][:, None] + bi[None, :]
    return ref


F_LIST = [1, 7, 8, 33, 256, 1536]  # 1 536: the 48 KB shared-memory limit of 8 user rows
N_ITEMS_LIST = [1, 255, 256, 257]


@pytest.mark.parametrize("n_items", N_ITEMS_LIST)
@pytest.mark.parametrize("f", F_LIST)
def test_mf_scores_exact_on_integer_factors(f, n_items):
    """Factors and biases in [-3, 3]: every fp32 partial sum is an integer below 2^24, so the result is exact and any
    indexing or skipped term shows."""
    rng = np.random.default_rng(f * 1000 + n_items)
    U, V, biases, d_U, d_VT, d_biases = _mf_case(rng, f, n_items, integer=True)
    for size in (1, 7, 8, 9):
        users = _user_block(rng, U.shape[0], size)
        for with_bias in (False, True):
            got = _mf(users, d_U, d_VT, d_biases if with_bias else None)
            want = _mf_ref(U, V, biases, users, with_bias).astype(np.float32)
            assert np.array_equal(got, want), "f=%d n_items=%d block=%d bias=%s" % (f, n_items, size, with_bias)


@pytest.mark.parametrize("n_items", N_ITEMS_LIST)
@pytest.mark.parametrize("f", F_LIST)
def test_mf_scores_within_fp32_dot_bound(f, n_items):
    """Random factors: |s - s64| <= gamma_f * sum_k |u_k v_k| (a length-f fp32 dot product, with or without FMA) plus the
    rounding of the three bias additions."""
    rng = np.random.default_rng(7 + f * 1000 + n_items)
    U, V, biases, d_U, d_VT, d_biases = _mf_case(rng, f, n_items, integer=False)
    gamma = f * U32 / (1 - f * U32)
    for size in (1, 7, 8, 9):
        users = _user_block(rng, U.shape[0], size)
        absdot = np.abs(U[users].astype(np.float64)) @ np.abs(V.T.astype(np.float64))
        for with_bias in (False, True):
            got = _mf(users, d_U, d_VT, d_biases if with_bias else None)
            want = _mf_ref(U, V, biases, users, with_bias)
            tol = gamma * absdot
            if with_bias:
                bu, bi, mu = (np.abs(b.astype(np.float64)) for b in biases)
                tol = tol + 4 * U32 * (absdot + mu[0] + bu[users][:, None] + bi[None, :])
            err = np.abs(got - want)
            assert (err <= tol).all(), "f=%d n_items=%d block=%d bias=%s: err %g > tol %g" % (
                f, n_items, size, with_bias, err.max(), tol[np.unravel_index(np.argmax(err - tol), err.shape)])


def test_mf_scores_600k_users_in_one_call():
    """More than 65 535 * 8 users: one call covers them all (gridDim.y holds 8 users per block)."""
    rng = np.random.default_rng(3)
    n_users, n_items, f = 600_000, 32, 8
    U = rng.integers(-3, 4, (n_users, f)).astype(np.float32)
    V = rng.integers(-3, 4, (n_items, f)).astype(np.float32)
    users = rng.permutation(n_users)
    got = _mf(users, _dev(U), _transpose(_dev(V)))
    assert np.array_equal(got, (U[users].astype(np.float64) @ V.T.astype(np.float64)).astype(np.float32))


def test_transpose_2_2m_rows():
    """More than 65 535 * 32 rows (item factors of a 2.2 M-item catalogue)."""
    rng = np.random.default_rng(4)
    A = rng.standard_normal((2_200_000, 4)).astype(np.float32)
    assert np.array_equal(_transpose(_dev(A)).cpu().numpy(), A.T)


# ---------------------------------------------------------------------------------------------------------------- SpMM
def _spmm(users, A, B, n_out, dense):
    L = _L()
    d_users = _dev(np.asarray(users, np.int32))
    a = [_dev(x) for x in (A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float32))]
    if dense:
        b_ptr = b_idx = None
        b_val = _dev(B.toarray().astype(np.float32))
    else:
        b_ptr, b_idx, b_val = (_dev(x) for x in (B.indptr.astype(np.int32), B.indices.astype(np.int32), B.data.astype(np.float32)))
    out = _nan_like((len(users), n_out))
    L.check(L.load().b200_score_spmm_device(d_users.data_ptr(), len(users), a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(),
                                            _ptr(b_ptr), _ptr(b_idx), b_val.data_ptr(), n_out, out.data_ptr(), _stream()))
    return out.cpu().numpy()


@pytest.mark.parametrize("dense", [False, True], ids=["csr_B", "dense_B"])
@pytest.mark.parametrize("n_out", [1, 37, 1000])
def test_spmm_exact_on_integer_values(n_out, dense):
    """Integer values: every sum is an integer below 2^24, exact whatever order the atomics land in.  User row 0 is
    empty, row 1 has 300 entries (more than the 16 warps of a CTA); B rows hold up to ~n_out / 3 entries (more than a
    warp's 32 lanes for n_out = 1000); the block repeats users and has more rows than the grid (sm_count * 4)."""
    rng = np.random.default_rng(n_out + dense)
    n_users, n_mid = 300, 400
    A = sps.random(n_users, n_mid, density=0.05, format="lil", random_state=n_out, dtype=np.float32)
    A[0, :] = 0
    A[1, rng.choice(n_mid, 300, replace=False)] = 1
    A = sps.csr_matrix(A)
    A.data = rng.integers(1, 4, A.nnz).astype(np.float32)
    A.sort_indices()
    B = sps.random(n_mid, n_out, density=0.3, format="csr", random_state=n_out + 1, dtype=np.float32)
    B.data = rng.choice(np.array([-3, -2, -1, 1, 2, 3], np.float32), B.nnz)
    B.sort_indices()
    n_block = 2 * 4 * _sm_count() + 3
    users = rng.integers(0, n_users, n_block)
    users[:4] = [1, 0, 1, 0]
    got = _spmm(users, A, B, n_out, dense)
    want = (A[users].astype(np.float64) @ B.astype(np.float64)).toarray()
    assert np.abs(want).max() < 2 ** 24
    assert np.array_equal(got, want.astype(np.float32))


# --------------------------------------------------------------------------------------------------------------- masks
def test_masks_seen_items_and_keep():
    rng = np.random.default_rng(8)
    n_users, n_items = 300, 777
    dense = synth_urm(n_users, n_items, 0.05, seed=8).toarray()
    dense[0] = 1  # a user who has seen every item
    dense[1] = 0  # and one who has seen none
    URM = sps.csr_matrix(dense, dtype=np.float32)
    users = rng.integers(0, n_users, 500)
    users[:3] = [0, 1, 0]
    scores = rng.standard_normal((len(users), n_items)).astype(np.float32)
    keep = (rng.random(n_items) < 0.6).astype(np.uint8)
    d_users, d_ptr, d_idx = _dev(users.astype(np.int32)), _dev(URM.indptr.astype(np.int32)), _dev(URM.indices.astype(np.int32))
    d_keep = _dev(keep)
    L = _L()
    for seen, with_keep in ((True, False), (False, True), (True, True)):
        d = _dev(scores)
        L.check(L.load().b200_score_mask_device(_ptr(d_users) if seen else None, len(users), _ptr(d_ptr) if seen else None,
                                                _ptr(d_idx) if seen else None, _ptr(d_keep) if with_keep else None, n_items,
                                                d.data_ptr(), _stream()))
        want = scores.copy()
        if with_keep:
            want[:, keep == 0] = -np.inf
        if seen:
            for b, u in enumerate(users):
                want[b, URM.indices[URM.indptr[u]:URM.indptr[u + 1]]] = -np.inf
        assert np.array_equal(d.cpu().numpy().view(np.uint32), want.view(np.uint32)), (seen, with_keep)


# ----------------------------------------------------------------------------------------------------------- evaluator
def _evaluate(train, test, S, cutoffs, block_size, **kw):
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout
    res, _ = EvaluatorHoldout(test, cutoffs, verbose=False, **kw).evaluateRecommender(_stub(train, S), block_size=block_size)
    return res, evaluate_scores(train, test, S, cutoffs, **kw)


def _assert_metrics(res, ref, rtol, ndcg_rtol=None):
    assert list(res.keys()) == list(ref.keys())
    for c in ref:
        assert set(res[c].keys()) == set(ref[c].keys())
        for k, v in ref[c].items():
            r = ndcg_rtol if (k == "NDCG" and ndcg_rtol) else rtol
            assert np.isclose(res[c][k], v, rtol=r, atol=1e-12), "cutoff %s %s: %r vs %r" % (c, k, res[c][k], v)


def _mixed_scores(rng, n_users, n_items):
    """Half the rows continuous, half integer-valued (ties on the item id)."""
    S = rng.standard_normal((n_users, n_items)).astype(np.float32)
    S[1::2] = rng.integers(0, 6, (n_users // 2, n_items))
    return S


def test_evaluator_twenty_unsorted_cutoffs_and_short_lists():
    """20 cutoffs in no order, 1 024 and 701 above the 700 items; users 0-4 have seen all but 3 items (lists shorter
    than most cutoffs) and hold those 3 in their test rows; block size 37 does not divide the 400 users."""
    rng = np.random.default_rng(21)
    n_users, n_items = 400, 700
    train = synth_urm(n_users, n_items, 0.05, seed=22, values="ratings").toarray()
    test = synth_urm(n_users, n_items, 0.03, seed=23, values="ratings").toarray()
    test[train != 0] = 0
    for u in range(5):
        unseen = rng.choice(n_items, 3, replace=False)
        train[u] = rng.integers(1, 6, n_items)
        train[u, unseen] = 0
        test[u] = 0
        test[u, unseen] = rng.integers(1, 6, 3)
    train, test = sps.csr_matrix(train, dtype=np.float32), sps.csr_matrix(test, dtype=np.float32)
    cutoffs = [10, 1024, 1, 700, 5, 701, 3, 50, 2, 999, 20, 7, 100, 4, 300, 15, 699, 6, 30, 8]
    res, ref = _evaluate(train, test, _mixed_scores(rng, n_users, n_items), cutoffs, block_size=37)
    _assert_metrics(res, ref, 1e-9)


def test_evaluator_test_rows_longer_than_1024_half_star():
    """Ten users with 1 100-1 500 test items (more hits than list positions), half-star ratings: the gain 2^r - 1 is
    exp2f in fp32, so nDCG is compared at 1e-6 and everything else at 1e-9."""
    rng = np.random.default_rng(31)
    n_users, n_items = 150, 3000
    train = synth_urm(n_users, n_items, 0.02, seed=32, values="ratings")
    test = synth_urm(n_users, n_items, 0.01, seed=33, values="ratings").tolil()
    for u in range(10):
        test[u, rng.choice(n_items, int(rng.integers(1100, 1500)), replace=False)] = 1
    test = sps.csr_matrix(test, dtype=np.float32)
    test.data = rng.integers(1, 11, test.nnz).astype(np.float32) / 2
    S = _mixed_scores(rng, n_users, n_items)
    S[:10] += 10 * (test[:10].toarray() != 0)  # the long-test users' hits crowd the top of their lists
    res, ref = _evaluate(train, test, S, [1024, 1, 10, 500], block_size=64)
    assert res[1024]["HIT_RATE"] > 0
    _assert_metrics(res, ref, 1e-9, ndcg_rtol=1e-6)


def _non_finite_case(with_nan):
    rng = np.random.default_rng(41 + with_nan)
    n_users, n_items = 300, 1500
    train = synth_urm(n_users, n_items, 0.02, seed=42, values="ratings")
    test = synth_urm(n_users, n_items, 0.02, seed=43, values="ratings")
    S = _mixed_scores(rng, n_users, n_items)
    u = rng.random(S.shape)
    frac = rng.choice([0.0, 0.05, 0.3, 0.75], n_users)[:, None]  # from none to more +inf entries than list positions
    S[u < frac] = np.inf
    S[(u >= frac) & (u < frac + 0.1)] = -np.inf
    if with_nan:
        S[(u >= frac + 0.1) & (u < frac + 0.2)] = np.nan
        S[5] = np.nan
    return train, test, S


def test_evaluator_skips_infinite_scores():
    """+inf and -inf scores are not recommendations; +inf entries still take their places in the first max_cutoff
    positions of the ranking (the reference filters after cutting), so the rest of the list moves up."""
    train, test, S = _non_finite_case(with_nan=False)
    res, ref = _evaluate(train, test, S, [1024, 5, 20, 100], block_size=100)
    _assert_metrics(res, ref, 1e-9)


def test_evaluator_skips_nan_scores():
    """NaN scores rank after -inf and are not recommendations (one user has only NaN scores)."""
    train, test, S = _non_finite_case(with_nan=True)
    res, ref = _evaluate(train, test, S, [1024, 5, 20, 100], block_size=100)
    _assert_metrics(res, ref, 1e-9)


def test_recommend_ranks_non_finite_scores_like_the_host_path():
    """recommend() on the device (cutoff <= 1024) and on the host (cutoff > 1024) give the oracle's lists on rows with
    NaN, +inf and -inf mixed in, all-NaN and all-+inf rows included."""
    rng = np.random.default_rng(51)
    n_users, n_items = 60, 3000
    train = synth_urm(n_users, n_items, 0.01, seed=52)
    S = _mixed_scores(rng, n_users, n_items)
    u = rng.random(S.shape)
    S[u < 0.1] = np.nan
    S[(u >= 0.1) & (u < 0.15)] = np.inf
    S[(u >= 0.15) & (u < 0.25)] = -np.inf
    S[3], S[4] = np.nan, np.inf
    rec = _stub(train, S)
    users = rng.permutation(n_users)
    for cutoff in (1, 5, 1024, 1025, n_items):
        want = []
        for usr in users:
            s = S[usr].astype(np.float64)
            s[train.indices[train.indptr[usr]:train.indptr[usr + 1]]] = -np.inf
            o = _order(s)[:cutoff]
            want.append(o[np.isfinite(s[o])].tolist())
        assert rec.recommend(users, cutoff=cutoff) == want, cutoff
