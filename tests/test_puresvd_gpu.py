"""PureSVDRecommender (csrc/puresvd.cu) against scikit-learn's randomized_svd (oracle/puresvd_oracle.py).  Host cases: the
sketch (transpose, n_iter, Omega and the generator state) and argument errors.  -m gpu: the CSR transpose, SVQB, the Jacobi
eigensolver and svd_flip through the test hook, whole fits against scikit-learn's float64 run with the same seed, and the
recommender-level calls."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.puresvd_oracle import puresvd_reference
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm

gpu = pytest.mark.gpu


# ---- host ----------------------------------------------------------------------------------------------------------
def _sklearn_sketch(shape, k, random_state):
    """(transpose, n_iter, n_random, Omega) as scikit-learn's _randomized_svd draws them, captured from inside its call."""
    import sklearn.utils.extmath as em
    seen = {}
    original = em._randomized_range_finder

    class Recording(np.random.RandomState):
        def normal(self, *a, **kw):
            out = super().normal(*a, **kw)
            seen["omega"] = out.astype(np.float32)
            return out

    def spy(A, *, size, n_iter, power_iteration_normalizer="auto", random_state=None):
        rec = Recording()
        rec.set_state(random_state.get_state())
        seen.update(transpose=A.shape != shape, n_iter=n_iter, size=size)
        Q = original(A, size=size, n_iter=n_iter, power_iteration_normalizer=power_iteration_normalizer, random_state=rec)
        random_state.set_state(rec.get_state())
        return Q

    X = synth_urm(shape[0], shape[1], 0.05, seed=1)
    em._randomized_range_finder = spy
    try:
        em.randomized_svd(X, n_components=k, random_state=random_state)
    finally:
        em._randomized_range_finder = original
    return seen["transpose"], seen["n_iter"], seen["size"], seen["omega"]


@pytest.mark.parametrize("seed", [0, 7, "RandomState", None])
@pytest.mark.parametrize("shape,k", [((300, 80), 5), ((300, 80), 20), ((60, 500), 100), ((90, 90), 3)])
def test_sketch_is_sklearns(seed, shape, k):
    from recsys2019_deeplearning_evaluation_b200.recommenders import randomized_svd_sketch
    rs = (lambda: np.random.RandomState(11)) if seed == "RandomState" else (lambda: seed)
    np.random.seed(123)
    got = randomized_svd_sketch(shape, k, rs())
    state_after = np.random.get_state()
    np.random.seed(123)
    ref = _sklearn_sketch(shape, k, rs())
    assert got[:3] == ref[:3]
    assert got[3].dtype == np.float32 and got[3].shape == (min(shape), k + 10)
    assert np.array_equal(got[3], ref[3])
    if seed is None:  # the global generator advanced exactly as randomized_svd advances it
        from sklearn.utils.extmath import randomized_svd
        np.random.seed(123)
        randomized_svd(synth_urm(shape[0], shape[1], 0.05, seed=1), n_components=k, random_state=None)
        sk_state = np.random.get_state()
        assert all(np.array_equal(a, b) for a, b in zip(state_after, sk_state))


def test_argument_errors():
    from recsys2019_deeplearning_evaluation_b200.recommenders import PureSVDRecommender
    r = PureSVDRecommender(synth_urm(50, 40, 0.1, seed=2), verbose=False)
    for bad in (0, 503, 1000):
        with pytest.raises(ValueError, match="num_factors must be between 1 and 502"):
            r.fit(num_factors=bad)


def test_oracle_is_randomized_svd():
    from sklearn.utils.extmath import randomized_svd
    X = synth_urm(120, 300, 0.05, seed=3)
    U, V, s = puresvd_reference(X, 8, random_seed=4)
    U0, s0, VT0 = randomized_svd(sps.csr_matrix(X, dtype=np.float32), n_components=8, random_state=4)
    assert np.array_equal(U, U0) and np.array_equal(s, s0) and np.allclose(V, (VT0 * s0[:, None]).T, rtol=0, atol=0)


# ---- device: the building blocks -------------------------------------------------------------------------------------
def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _transpose(X):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    n_rows, n_cols = X.shape
    ptr, idx, val = _dev(X.indptr.astype(np.int32)), _dev(X.indices.astype(np.int32)), _dev(X.data.astype(np.float32))
    optr = torch.empty(n_cols + 1, dtype=torch.int32, device="cuda")
    oidx = torch.empty(X.nnz, dtype=torch.int32, device="cuda")
    oval = torch.empty(X.nnz, dtype=torch.float32, device="cuda")
    _lib.check(_lib.load().b200_csr_transpose_device(n_rows, n_cols, X.nnz, ptr.data_ptr(), idx.data_ptr(), val.data_ptr(),
                                                     optr.data_ptr(), oidx.data_ptr(), oval.data_ptr(), _stream()))
    return optr.cpu().numpy(), oidx.cpu().numpy(), oval.cpu().numpy()


@gpu
@pytest.mark.parametrize("n_rows,n_cols,density", [(300, 120, 0.05), (1, 7, 0.5), (5000, 1, 0.3), (2_200_000, 3000, 2e-4)])
def test_csr_transpose_is_scipys(n_rows, n_cols, density):
    X = synth_urm(n_rows, n_cols, density, seed=4, values="continuous").tolil()
    X[: n_rows // 10, :] = 0  # empty rows
    X[:, : max(n_cols // 10, 0)] = 0  # empty columns
    X = sps.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    T = X.T.tocsr()
    ptr, idx, val = _transpose(X)
    assert np.array_equal(ptr, T.indptr) and np.array_equal(idx, T.indices) and np.array_equal(val, T.data)


@gpu
def test_csr_transpose_of_an_empty_matrix():
    ptr, idx, val = _transpose(sps.csr_matrix((40, 9), dtype=np.float32))
    assert np.array_equal(ptr, np.zeros(10, np.int32)) and idx.size == 0 and val.size == 0


def _orth(Y, passes):
    from recsys2019_deeplearning_evaluation_b200 import _lib
    d = _dev(np.asarray(Y, np.float32))
    _lib.check(_lib.load().b200_svd_debug_device(0, Y.shape[0], Y.shape[1], passes, d.data_ptr(), None, _stream()))
    return d.cpu().numpy().astype(np.float64)


def _check_basis(Y, Q, rank):
    kept = np.abs(Q).max(axis=0) > 0
    assert kept.sum() == rank, (kept.sum(), rank)
    assert np.all(Q[:, ~kept] == 0)
    Qk = Q[:, kept]
    assert np.abs(Qk.T @ Qk - np.eye(rank)).max() <= 1e-6
    Y = Y.astype(np.float64)
    assert np.linalg.norm(Y - Qk @ (Qk.T @ Y)) <= 1e-6 * np.linalg.norm(Y)


@gpu
@pytest.mark.parametrize("m,r", [(5000, 110), (2000, 360), (512, 512), (40, 40), (3000, 1)])
def test_orthonormaliser(m, r):
    rng = np.random.default_rng(m + r)
    Y = rng.standard_normal((m, r)).astype(np.float32)
    _check_basis(Y, _orth(Y, 2), r)
    # column-scaled to condition 1e6
    Ys = (Y * np.logspace(0, 6, r)[None, :]).astype(np.float32)
    _check_basis(Ys, _orth(Ys, 2), r)


@gpu
def test_orthonormaliser_drops_duplicate_and_zero_columns():
    rng = np.random.default_rng(3)
    Y = rng.standard_normal((3000, 40)).astype(np.float32)
    Y[:, 5] = Y[:, 2]
    Y[:, 9] = 0
    Y[:, 30] = Y[:, 31]
    for passes in (1, 2):
        _check_basis(Y, _orth(Y, passes), 37)
    # a tall matrix of rank 3
    Z = (rng.standard_normal((1000, 3)) @ rng.standard_normal((3, 25))).astype(np.float32)
    _check_basis(Z, _orth(Z, 2), 3)
    assert np.all(_orth(np.zeros((100, 12), np.float32), 2) == 0)


def _eigh(A):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    r = A.shape[0]
    out = torch.empty(r + r * r, dtype=torch.float64, device="cuda")
    _lib.check(_lib.load().b200_svd_debug_device(1, r, r, 0, _dev(A.astype(np.float64)).data_ptr(), out.data_ptr(), _stream()))
    o = out.cpu().numpy()
    return o[:r], o[r:].reshape(r, r)


@gpu
@pytest.mark.parametrize("r", [1, 2, 33, 110, 360, 512])
def test_eigensolver_matches_eigh(r):
    rng = np.random.default_rng(r)
    B = rng.standard_normal((r, r))
    cases = [B + B.T]
    # repeated and zero eigenvalues, positive semi-definite
    Qm, _ = np.linalg.qr(rng.standard_normal((r, r)))
    lam = np.concatenate([np.full(r // 3, 2.0), np.zeros(r // 3), rng.random(r - 2 * (r // 3)) * 5])
    cases.append((Qm * lam) @ Qm.T)
    cases[-1] = (cases[-1] + cases[-1].T) / 2
    for A in cases:
        w, V = _eigh(A)
        ref = np.linalg.eigvalsh(A)[::-1]
        lmax = np.abs(ref).max()
        assert np.all(np.diff(w) <= 0)
        assert np.abs(w - ref).max() <= 1e-12 * lmax, np.abs(w - ref).max() / lmax
        assert np.abs(A @ V - V * w).max() <= 1e-12 * lmax * np.sqrt(r)
        assert np.abs(V.T @ V - np.eye(r)).max() <= 1e-12 * r


@gpu
def test_sign_flip():
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    U = np.array([[1, -3, 2, 0, 0.5], [-2, 3, -2, 0, -0.5], [0.5, 1, 1, 0, 0.5]], np.float32)
    O = np.arange(20, dtype=np.float32).reshape(4, 5) - 7
    dU, dO = _dev(U), _dev(O)
    _lib.check(_lib.load().b200_svd_debug_device(2, 3, 5, 4, dU.data_ptr(), dO.data_ptr(), _stream()))
    torch.cuda.synchronize()
    # columns: max |.| at row 1 (negative); tie +-3 -> row 0 (negative); tie +-2 -> row 0 (positive); all zero; tie -> row 0
    sign = np.array([-1, -1, 1, 1, 1], np.float32)
    assert np.array_equal(dU.cpu().numpy(), U * sign) and np.array_equal(dO.cpu().numpy(), O * sign)
    # svd_flip's own decision on the same columns
    from sklearn.utils.extmath import svd_flip
    u, v = svd_flip(U.astype(np.float64).copy(), O.T.astype(np.float64).copy())
    keep = np.abs(U).max(axis=0) > 0
    assert np.array_equal(u[:, keep], (U * sign)[:, keep])


# ---- device: whole fits --------------------------------------------------------------------------------------------
def _device_svd(X, k, seed):
    from recsys2019_deeplearning_evaluation_b200.recommenders import PureSVDRecommender
    r = PureSVDRecommender(X, verbose=False)
    return r._randomized_svd_device(k, seed)


def _compare(X, k, seed, cos_gap=1e-4, check_vectors=True):
    """The device fit against scikit-learn's float64 run with the same seed; the score bar is 4x the distance of scikit-learn's
    own float32 run from it."""
    U, V, s = _device_svd(X, k, seed)
    U64, V64, s64 = puresvd_reference(X, k, random_seed=seed, dtype=np.float64)
    U32, V32, _ = puresvd_reference(X, k, random_seed=seed, dtype=np.float32)
    assert U.shape == U64.shape and V.shape == V64.shape and s.shape == s64.shape
    assert np.all(np.isfinite(U)) and np.all(np.isfinite(V))
    s1 = max(s64[0], 1e-300)
    assert np.abs(s - s64).max() <= 1e-5 * s1, np.abs(s - s64).max() / s1
    S64 = U64 @ V64.T
    smax = np.abs(S64).max()
    dev = np.abs(U.astype(np.float64) @ V.T.astype(np.float64) - S64).max() / smax
    band = np.abs(U32.astype(np.float64) @ V32.T.astype(np.float64) - S64).max() / smax
    assert dev <= 4 * band, (dev, band)
    if not check_vectors:
        return
    kp = len(s64)
    for j in range(kp):
        gap = min([abs(s64[j] - s64[i]) for i in (j - 1, j + 1) if 0 <= i < kp] or [np.inf])
        if gap < cos_gap * s1 or s64[j] <= 1e-3 * s1:
            continue
        for a, b in ((U[:, j], U64[:, j]), (V[:, j], V64[:, j])):
            c = float(a.astype(np.float64) @ b / (np.linalg.norm(a) * np.linalg.norm(b)))
            top = np.sort(np.abs(U64[:, j]))[-2:]
            if top[1] - top[0] > 1e-3 * top[1]:  # svd_flip's decision is well defined: the signs must agree
                assert c > 0, (j, c)
            assert 1 - abs(c) <= 1e-5, (j, 1 - abs(c))


@gpu
@pytest.mark.parametrize("shape,k", [((3000, 800), 10), ((3000, 800), 100), ((800, 3000), 10), ((800, 3000), 100), ((700, 700), 30),
                                     ((3000, 800), 1), ((300, 80), 100), ((80, 300), 75)])
def test_fit_matches_sklearn_fp64(shape, k):
    _compare(synth_urm(shape[0], shape[1], 0.02 if min(shape) > 100 else 0.1, seed=42), k, 7)


@gpu
def test_fit_350_factors_on_ratings():
    _compare(synth_config("C2", values="ratings"), 350, 3)


@gpu
def test_fit_planted_low_rank_and_popularity():
    rng = np.random.default_rng(5)
    L = rng.random((2000, 6)) @ rng.random((6, 700))
    X = sps.csr_matrix(np.where(rng.random((2000, 700)) < 0.05, L, 0), dtype=np.float32)
    _compare(X, 20, 1)
    _compare(synth_urm(3000, 1200, 0.02, seed=8, values="ratings", popularity=0.8), 50, 2)


@gpu
def test_fit_rank_deficient_60_by_500():
    _compare(synth_urm(60, 500, 0.1, seed=6), 100, 0)


@gpu
def test_fit_with_empty_users_and_items():
    X = synth_urm(900, 400, 0.03, seed=9, values="ratings").tolil()
    X[:50, :] = 0
    X[:, 100:140] = 0
    X = sps.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    _compare(X, 40, 4)
    _compare(X.T.tocsr(), 40, 4)


@gpu
def test_fit_all_zero_urm():
    for shape in ((50, 30), (30, 50)):
        U, V, s = _device_svd(sps.csr_matrix(shape, dtype=np.float32), 10, 0)
        assert U.shape == (shape[0], 10) and V.shape == (shape[1], 10)
        assert np.all(np.isfinite(U)) and np.all(np.isfinite(V)) and np.all(s == 0)
        assert np.all(U @ V.T == 0)


@gpu
def test_fit_global_random_state():
    """random_seed=None draws from numpy's global generator: with the same global seed the fit is scikit-learn's."""
    X = synth_urm(1000, 400, 0.03, seed=12)
    np.random.seed(77)
    U, V, s = _device_svd(X, 20, None)
    after = np.random.get_state()[1].copy()
    np.random.seed(77)
    U64, V64, s64 = puresvd_reference(X, 20, random_seed=None, dtype=np.float64)
    assert np.array_equal(after, np.random.get_state()[1])
    assert np.abs(s - s64).max() <= 1e-5 * s64[0]


@gpu
def test_fit_c3_100_factors():
    _compare(synth_config("C3"), 100, 1, check_vectors=True)


# ---- device: recommender level -------------------------------------------------------------------------------------
def _negatives(test, n_users, n_items, seed):
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(n_users):
        cand = np.setdiff1d(rng.choice(n_items, 120, replace=False), test[u].indices)[:100]
        rows += [u] * len(cand)
        cols += list(cand)
    return sps.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_users, n_items))


@gpu
def test_recommender_calls_agree_with_oracle_factors(tmp_path):
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout, EvaluatorNegativeItemSample
    from recsys2019_deeplearning_evaluation_b200.recommenders import PureSVDRecommender
    train = synth_urm(800, 500, 0.04, seed=31, values="ratings")
    test = synth_urm(800, 500, 0.006, seed=32, values="ratings")
    r = PureSVDRecommender(train, verbose=False)
    r.fit(num_factors=16, random_seed=3)
    assert r.USER_factors.shape == (800, 16) and r.ITEM_factors.shape == (500, 16) and not r.use_bias
    W, V, _ = puresvd_reference(train, 16, random_seed=3, dtype=np.float64)
    o = PureSVDRecommender(train, verbose=False)
    o.USER_factors, o.ITEM_factors = W.astype(np.float32), np.asarray(V, np.float32)
    users = np.arange(800)
    a, sa = r.recommend(users, cutoff=10, return_scores=True)
    b, sb = o.recommend(users, cutoff=10, return_scores=True)
    seen = np.isneginf(sb)
    assert np.array_equal(np.isneginf(sa), seen)
    assert np.allclose(sa[~seen], sb[~seen], rtol=1e-4, atol=1e-4 * np.abs(sb[~seen]).max())
    same = np.mean([len(set(x) & set(y)) / max(len(y), 1) for x, y in zip(a, b)])
    assert same > 0.99, same
    for ev in (EvaluatorHoldout(test, cutoff_list=[5, 10], verbose=False),
               EvaluatorNegativeItemSample(test, _negatives(test, 800, 500, 33), cutoff_list=[5, 10], verbose=False)):
        ra, _ = ev.evaluateRecommender(r)
        rb, _ = ev.evaluateRecommender(o)
        for cutoff in (5, 10):
            for metric in ("PRECISION", "RECALL", "MAP", "NDCG"):
                assert abs(ra[cutoff][metric] - rb[cutoff][metric]) <= 2e-3, (cutoff, metric, ra[cutoff][metric], rb[cutoff][metric])
    r.save_model(str(tmp_path) + os.sep, "puresvd")
    r2 = PureSVDRecommender(train, verbose=False)
    r2.load_model(str(tmp_path) + os.sep, "puresvd")
    assert np.array_equal(r2.USER_factors, r.USER_factors) and np.array_equal(r2.ITEM_factors, r.ITEM_factors)
    assert np.array_equal(r2.recommend(users[:50], cutoff=10), r.recommend(users[:50], cutoff=10))
