"""-m gpu: both evaluators on foreign recommenders -- objects that are not this package's mirrors and only offer the
reference's `_compute_item_score` / `get_URM_train` / `set_items_to_ignore` / `reset_items_to_ignore` -- and the fp64 mask
and top-N kernels that rank their float64 score blocks (csrc/score.cu).

The kernels are checked against np.lexsort((arange, -s)) on fp64 rows, the evaluators against the numpy restatements
oracle/evaluator_oracle.py and oracle/diversity_oracle.py fed the same score matrix, and against the mirror path on a
model whose scores are exact."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.diversity_oracle import evaluate_scores_with_diversity, recommendation_lists
from oracle.evaluator_oracle import evaluate_scores
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
ITEM_SENTINEL = 0x5EED
SCORE_SENTINEL = np.uint32(0x7FBADBAD)  # a NaN payload no kernel writes


def _L():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ----------------------------------------------------------------------------------------------------------- kernels
def _image(v):
    """The fp32 image the fp64 top-N table reports: rounded to fp32, finite values saturated to +-FLT_MAX."""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore"):
        f = v.astype(np.float32)
    fin = np.isfinite(v)
    f[fin] = np.clip(f[fin], -FLT_MAX, FLT_MAX)
    return f


def _topn64(S, cutoff):
    """b200_score_topn_f64_device on S; the tables get one guard row past their end, filled with a sentinel."""
    import torch
    L = _L()
    n_rows, n_items = S.shape
    d = _dev(np.asarray(S, np.float64))
    items = torch.full((n_rows + 1, cutoff), ITEM_SENTINEL, dtype=torch.int32, device="cuda")
    vals = _dev(np.full((n_rows + 1, cutoff), SCORE_SENTINEL, np.uint32).view(np.float32))
    L.check(L.load().b200_score_topn_f64_device(d.data_ptr(), n_rows, n_items, cutoff, items.data_ptr(), vals.data_ptr(),
                                                _stream()))
    items, vals = items.cpu().numpy(), vals.cpu().numpy()
    assert np.all(items[n_rows] == ITEM_SENTINEL) and np.all(vals[n_rows].view(np.uint32) == SCORE_SENTINEL), \
        "the guard row past the table was written"
    return items[:n_rows], vals[:n_rows]


def _check_topn64(S, cutoff):
    """Items exact; scores the bitwise fp32 image of the fp64 score (any NaN for NaN); past the row -1 / -inf."""
    items, vals = _topn64(S, cutoff)
    bad = []
    for r, s in enumerate(S):
        o = np.lexsort((np.arange(len(s)), -s))[:cutoff]
        want_items = np.full(cutoff, -1, np.int32)
        want_vals = np.full(cutoff, -np.inf, np.float32)
        want_items[:len(o)] = o
        want_vals[:len(o)] = _image(s[o])
        nan = np.isnan(want_vals)
        if not (np.array_equal(items[r], want_items) and np.array_equal(np.isnan(vals[r]), nan)
                and np.array_equal(vals[r][~nan].view(np.uint32), want_vals[~nan].view(np.uint32))):
            bad.append(r)
    assert not bad, "cutoff %d: rows %s differ from the lexsort ranking" % (cutoff, bad)


def _f64_rows(n, rng):
    """One fp64 row per score family [n_rows, n]."""
    rows = [rng.standard_normal(n),                                                      # continuous
            rng.integers(0, 3, n).astype(np.float64),                                    # massive ties
            np.full(n, 0.25)]                                                            # all equal
    s = rng.standard_normal(n)  # NaN of both signs, +-inf, +-0
    u = rng.random(n)
    s[u < 0.1] = np.nan
    s[(u >= 0.1) & (u < 0.15)] = -np.nan
    s[(u >= 0.15) & (u < 0.25)] = np.inf
    s[(u >= 0.25) & (u < 0.35)] = -np.inf
    s[(u >= 0.35) & (u < 0.45)] = 0.0
    s[(u >= 0.45) & (u < 0.55)] = -0.0
    rows.append(s)
    # magnitudes beyond fp32 (saturated in the table), at its edge, and tiny ones that round to zero or a subnormal
    rows.append(rng.choice(np.array([1e300, -1e300, 3e38, -3e38, 3.5e38, -3.5e38, FLT_MAX, -FLT_MAX, 1e-40, -1e-40,
                                     1e-310, -1e-310, 5e-324, 0.0, 1.0, -1.0]), n))
    # values one fp32 rounding apart at most: they collide in fp32 and not in fp64
    rows.append(1.0 + rng.integers(0, 64, n) * 2.0 ** -40)
    rows.append(-1.0 - rng.integers(0, 64, n) * 2.0 ** -40)
    for k in (0, 1, 5, 600, 1000):  # all but k items at -inf
        s = np.full(n, -np.inf)
        s[rng.choice(n, min(k, n), replace=False)] = rng.integers(-1, 2, min(k, n))
        rows.append(s)
    return np.stack(rows)


@pytest.mark.parametrize("n_items", [1, 2, 1023, 1024, 1025, 50_000, 200_000])
def test_topn_f64_matches_lexsort(n_items):
    rng = np.random.default_rng(n_items)
    S = _f64_rows(n_items, rng)
    for cutoff in (1, 7, 1023, 1024):
        _check_topn64(S, cutoff)


def test_topn_f64_saturates_the_fp32_image():
    """Finite scores outside the fp32 range are reported as +-FLT_MAX (finite), non-finite ones keep their class."""
    S = np.array([[1e300, -1e300, np.inf, -np.inf, np.nan, 3.5e38, -3.5e38, 1e-310, 2.0]])
    items, vals = _topn64(S, 9)
    assert items[0].tolist() == [2, 0, 5, 8, 7, 6, 1, 3, 4]
    assert vals[0][:7].tolist() == [np.inf, FLT_MAX, FLT_MAX, 2.0, 0.0, -FLT_MAX, -FLT_MAX]
    assert vals[0][7] == -np.inf and np.isnan(vals[0][8])
    assert np.array_equal(np.isfinite(vals[0]), np.isfinite(S[0][items[0]]))


def test_topn_f64_rejects_cutoff_out_of_range():
    S = np.zeros((2, 10))
    for cutoff in (0, 1025):
        with pytest.raises(ValueError):
            _topn64(S, cutoff)


def test_evaluators_still_refuse_cutoffs_above_1024():
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout, EvaluatorNegativeItemSample
    test = synth_urm(20, 50, 0.1, seed=1)
    with pytest.raises(ValueError, match="1024"):
        EvaluatorHoldout(test, [10, 1025], verbose=False)
    with pytest.raises(ValueError, match="1024"):
        EvaluatorNegativeItemSample(test, test, [1025], verbose=False)


def test_mask_f64_matches_numpy():
    rng = np.random.default_rng(8)
    n_users, n_items = 300, 777
    dense = synth_urm(n_users, n_items, 0.05, seed=8).toarray()
    dense[0] = 1  # a user who has seen every item
    dense[1] = 0  # and one who has seen none
    URM = sps.csr_matrix(dense, dtype=np.float32)
    users = rng.integers(0, n_users, 500)
    users[:3] = [0, 1, 0]
    scores = rng.standard_normal((len(users), n_items)) * 1e200
    keep = (rng.random(n_items) < 0.6).astype(np.uint8)
    d_users, d_ptr, d_idx = _dev(users.astype(np.int32)), _dev(URM.indptr.astype(np.int32)), _dev(URM.indices.astype(np.int32))
    d_keep = _dev(keep)
    L = _L()
    for seen, with_keep in ((True, False), (False, True), (True, True)):
        d = _dev(scores)
        L.check(L.load().b200_score_mask_f64_device(d_users.data_ptr() if seen else None, len(users),
                                                    d_ptr.data_ptr() if seen else None, d_idx.data_ptr() if seen else None,
                                                    d_keep.data_ptr() if with_keep else None, n_items, d.data_ptr(), _stream()))
        want = scores.copy()
        if with_keep:
            want[:, keep == 0] = -np.inf
        if seen:
            for b, u in enumerate(users):
                want[b, URM.indices[URM.indptr[u]:URM.indptr[u + 1]]] = -np.inf
        assert np.array_equal(d.cpu().numpy().view(np.uint64), want.view(np.uint64)), (seen, with_keep)


# ------------------------------------------------------------------------------------------------- foreign recommenders
class Foreign(object):
    """A reference-style recommender that is not a mirror: a dense score matrix S on the host.  `_compute_item_score`
    behaves like the reference's BaseSimilarityMatrixRecommender: -inf outside `items_to_compute`; `cast` turns the
    returned block into whatever a model might return."""

    def __init__(self, URM_train, S, cast=None):
        self.URM_train = sps.csr_matrix(URM_train)
        self.S = S
        self.cast = cast
        self.items_to_ignore_ID = np.array([], dtype=np.int64)

    def get_URM_train(self):
        return self.URM_train.copy()

    def set_items_to_ignore(self, items_to_ignore):
        self.items_to_ignore_ID = np.array(items_to_ignore, dtype=np.int64)

    def reset_items_to_ignore(self):
        self.items_to_ignore_ID = np.array([], dtype=np.int64)

    def _compute_item_score(self, user_id_array, items_to_compute=None):
        block = self.S[user_id_array]
        if items_to_compute is not None:
            out = np.full(block.shape, -np.inf, dtype=block.dtype)
            out[:, items_to_compute] = block[:, items_to_compute]
            block = out
        return self.cast(block) if self.cast else block


class Wrapped(object):
    """A mirror behind the foreign interface: the evaluators see only the reference's methods."""

    def __init__(self, rec):
        self.rec = rec

    def get_URM_train(self):
        return self.rec.get_URM_train()

    def set_items_to_ignore(self, items_to_ignore):
        self.rec.set_items_to_ignore(items_to_ignore)

    def reset_items_to_ignore(self):
        self.rec.reset_items_to_ignore()

    def _compute_item_score(self, user_id_array, items_to_compute=None):
        return self.rec._compute_item_score(user_id_array, items_to_compute=items_to_compute)


def _case(seed, n_users=150, n_items=600, n_neg=60, dtype=np.float64):
    """train, test, sampled negatives and a score matrix: half the rows continuous, half integer-valued (ties)."""
    rng = np.random.default_rng(seed)
    train = synth_urm(n_users, n_items, 0.03, seed=seed, values="ratings")
    test = synth_urm(n_users, n_items, 0.02, seed=seed + 1, values="ratings")
    rows = np.repeat(np.arange(n_users), n_neg)
    cols = np.concatenate([rng.choice(n_items, n_neg, replace=False) for _ in range(n_users)])
    neg = sps.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_users, n_items))
    S = rng.standard_normal((n_users, n_items))
    S[1::2] = rng.integers(0, 6, (n_users // 2, n_items))
    return train, test, neg, S.astype(dtype)


def _evaluator(kind, test, neg, cutoffs, **kw):
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout, EvaluatorNegativeItemSample
    if kind == "holdout":
        return EvaluatorHoldout(test, cutoffs, verbose=False, **kw)
    return EvaluatorNegativeItemSample(test, neg, cutoffs, verbose=False, **kw)


def _assert_matches(res, ref, rtol=1e-9):
    assert set(res) == set(ref)
    for c in ref:
        assert set(res[c]) == set(ref[c]), c
        for k, v in ref[c].items():
            assert np.isclose(res[c][k], v, rtol=rtol, atol=1e-12, equal_nan=True), \
                "cutoff %s %s: %r vs %r" % (c, k, res[c][k], v)


def _run(kind, train, test, neg, S, block_size, cutoffs, D=None, cast=None, **kw):
    """The evaluator on a Foreign(S) and the oracle on the same S, compared at 1e-9."""
    from recsys2019_deeplearning_evaluation_b200.evaluation import Diversity_similarity
    ev = _evaluator(kind, test, neg, cutoffs, diversity_object=None if D is None else Diversity_similarity(D), **kw)
    res, _ = ev.evaluateRecommender(Foreign(train, S, cast), block_size=block_size)
    okw = dict(kw, URM_test_negative=neg) if kind == "negative" else kw
    S64 = np.asarray(S, np.float64)
    if D is None:
        ref = evaluate_scores(train, test, S64, cutoffs, **okw)
    else:
        ref = evaluate_scores_with_diversity(train, test, S64, cutoffs, D, **okw)
    _assert_matches(res, ref)
    return res


@pytest.mark.parametrize("kind", ["holdout", "negative"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("block_size", [1, 7, 1000])
def test_matches_oracle_block_sizes(kind, dtype, block_size):
    train, test, neg, S = _case(3, dtype=dtype)
    _run(kind, train, test, neg, S, block_size, [1, 5, 10, 1024])


@pytest.mark.parametrize("kind", ["holdout", "negative"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("options", ["keep_seen", "ignore"])
def test_matches_oracle_options(kind, dtype, options):
    train, test, neg, S = _case(5, dtype=dtype)
    if options == "keep_seen":
        kw = dict(exclude_seen=False)
    else:
        kw = dict(ignore_items=np.unique(np.concatenate([test.indices[::5], neg.indices[::9]]))[:80],
                  ignore_users=[0, 3, 17, 40], min_ratings_per_user=2)
    _run(kind, train, test, neg, S, 16, [1, 5, 10, 1024], **kw)


@pytest.mark.parametrize("kind", ["holdout", "negative"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_matches_oracle_with_diversity(kind, dtype):
    train, test, neg, S = _case(7, dtype=dtype)
    D = np.random.default_rng(8).random((S.shape[1], S.shape[1]))
    res = _run(kind, train, test, neg, S, 32, [2, 5, 10, 50], D=D)
    assert all(res[c]["DIVERSITY_SIMILARITY"] > 0 for c in res)


@pytest.mark.parametrize("kind", ["holdout", "negative"])
def test_fp64_scores_that_collide_in_fp32(kind):
    """Scores 1 + k 2^-40 round to 1.0 in fp32: ranked in fp64 the test items lead, rounded to fp32 the lowest item ids
    do.  The evaluator matches the oracle on the fp64 scores, and the oracle's lists on the fp32 rounding differ."""
    train, test, neg, _ = _case(9)
    rng = np.random.default_rng(10)
    S = 1.0 + rng.integers(0, 2 ** 10, test.shape) * 2.0 ** -40 + (test.toarray() != 0) * 2.0 ** -30
    assert np.all(S.astype(np.float32) == 1.0)
    cutoffs = [1, 5, 10]
    res = _run(kind, train, test, neg, S, 64, cutoffs)
    okw = dict(URM_test_negative=neg) if kind == "negative" else {}
    users, lists64 = recommendation_lists(train, test, S, cutoffs, **okw)
    _, lists32 = recommendation_lists(train, test, S.astype(np.float32), cutoffs, **okw)
    assert sum(not np.array_equal(a, b) for a, b in zip(lists64, lists32)) > len(users) // 2
    ref32 = evaluate_scores(train, test, S.astype(np.float32), cutoffs, **okw)
    assert res[10]["PRECISION"] > ref32[10]["PRECISION"]


def _mirror_case():
    """ItemKNNCustomSimilarity with an integer W on integer ratings: every score is an exact small integer in fp32."""
    from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCustomSimilarityRecommender
    train, test, neg, _ = _case(11, n_users=120, n_items=400)
    W = sps.random(400, 400, density=0.05, random_state=12, format="csr", dtype=np.float32)
    W.data = np.round(W.data * 8 - 4).astype(np.float32)
    rec = ItemKNNCustomSimilarityRecommender(train, verbose=False)
    rec.fit(W)
    return rec, test, neg


# block_size=1 in the exact comparisons below: the accumulators add the users of one launch with fp64 atomics in no fixed
# order, so only one user per block makes two runs add the same values in the same order.
@pytest.mark.parametrize("kind", ["holdout", "negative"])
def test_same_as_the_mirror(kind):
    rec, test, neg = _mirror_case()
    kw = dict(ignore_items=np.arange(0, 400, 13), exclude_seen=True)
    ev = _evaluator(kind, test, neg, [1, 5, 10, 50], **kw)
    res_mirror, _ = ev.evaluateRecommender(rec, block_size=1)
    res_foreign, _ = ev.evaluateRecommender(Wrapped(rec), block_size=1)
    assert res_foreign == res_mirror
    assert res_mirror[10]["HIT_RATE"] > 0


@pytest.mark.parametrize("kind", ["holdout", "negative"])
def test_repeated_and_interleaved_with_a_mirror(kind):
    rec, test, neg = _mirror_case()
    foreign = Foreign(rec.get_URM_train(), rec._compute_item_score(np.arange(rec.n_users)).astype(np.float64))
    ev = _evaluator(kind, test, neg, [1, 5, 10])
    first, _ = ev.evaluateRecommender(foreign, block_size=1)
    mirror, _ = ev.evaluateRecommender(rec, block_size=1)
    second, _ = ev.evaluateRecommender(foreign, block_size=1)
    assert first == second == mirror


class Recording(Foreign):
    def __init__(self, *args):
        super(Recording, self).__init__(*args)
        self.calls = []

    def get_URM_train(self):
        self.calls.append(("get_URM_train",))
        return super(Recording, self).get_URM_train()

    def set_items_to_ignore(self, items_to_ignore):
        self.calls.append(("set_items_to_ignore", np.array(items_to_ignore)))
        super(Recording, self).set_items_to_ignore(items_to_ignore)

    def reset_items_to_ignore(self):
        self.calls.append(("reset_items_to_ignore",))
        super(Recording, self).reset_items_to_ignore()

    def _compute_item_score(self, user_id_array, items_to_compute=None):
        self.calls.append(("_compute_item_score", np.array(user_id_array),
                           None if items_to_compute is None else np.array(items_to_compute)))
        return super(Recording, self)._compute_item_score(user_id_array, items_to_compute)


def _same_call(got, want):
    if got[0] != want[0] or len(got) != len(want):
        return False
    for a, b in zip(got[1:], want[1:]):
        if (a is None) != (b is None):
            return False
        if a is not None and not (a.dtype == b.dtype and np.array_equal(a, b)):
            return False
    return True


@pytest.mark.parametrize("kind", ["holdout", "negative"])
def test_call_sequence_is_the_references(kind):
    """Hold-out: one call per block of users (consecutive int64 slices, items_to_compute None).  Negative sample: one
    call per user, np.atleast_1d(u) and the user's sorted candidate row.  set_items_to_ignore first, reset_items_to_ignore last."""
    train, test, neg, S = _case(13, n_users=60)
    ignore = np.array([3, 9, 27], dtype=np.int64)
    ev = _evaluator(kind, test, neg, [5], ignore_items=ignore)
    rec = Recording(train, S)
    ev.evaluateRecommender(rec, block_size=7)
    users = np.asarray(ev.users_to_evaluate, dtype=np.int64)
    want = [("set_items_to_ignore", ignore), ("get_URM_train",)]
    if kind == "holdout":
        want += [("_compute_item_score", users[b0:b0 + 7], None) for b0 in range(0, len(users), 7)]
    else:
        R = ev.URM_items_to_rank
        want += [("_compute_item_score", np.atleast_1d(u), R.indices[R.indptr[u]:R.indptr[u + 1]]) for u in users]
        cand = sps.csr_matrix((test + neg).astype(bool))
        cand.sort_indices()
        assert all(np.array_equal(w[2], cand.indices[cand.indptr[u]:cand.indptr[u + 1]]) for w, u in zip(want[2:], users))
    want.append(("reset_items_to_ignore",))
    assert len(rec.calls) == len(want)
    bad = [i for i, (g, w) in enumerate(zip(rec.calls, want)) if not _same_call(g, w)]
    assert not bad, "calls %s differ: %r vs %r" % (bad[:3], rec.calls[bad[0]], want[bad[0]])


@pytest.mark.parametrize("cast", ["int32", "bool", "float16", "matrix"])
def test_other_dtypes_are_ranked_as_float64(cast):
    """The negative-sample evaluator ranks the model's full row, and an integer block has no -inf for the
    non-candidates, so the integer dtypes are checked on the hold-out evaluator only."""
    train, test, neg, S = _case(15)
    rng = np.random.default_rng(16)
    if cast == "int32":
        S = rng.integers(-2 ** 31, 2 ** 31 - 1, S.shape, dtype=np.int64).astype(np.int32)
    elif cast == "bool":
        S = rng.random(S.shape) < 0.3
    elif cast == "float16":
        S = (S / 7).astype(np.float16)
    else:
        S = np.matrix(S)
    for kind in ("holdout", "negative") if cast in ("float16", "matrix") else ("holdout",):
        _run(kind, train, test, neg, S, 50, [1, 5, 10], cast=np.asmatrix if cast == "matrix" else None)


@pytest.mark.parametrize("kind", ["holdout", "negative"])
def test_wrong_blocks_raise(kind):
    train, test, neg, S = _case(17, n_users=40)
    ev = _evaluator(kind, test, neg, [5])
    for cast, match in ((lambda b: b[:, :-1], "shape"), (lambda b: b[0], "shape"), (lambda b: b[None], "shape"),
                        (lambda b: b.astype(np.complex128), "dtype")):
        with pytest.raises(ValueError, match=match):
            ev.evaluateRecommender(Foreign(train, S, cast))
