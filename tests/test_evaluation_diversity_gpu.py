"""DIVERSITY_SIMILARITY (metrics.py:719-775) in both evaluators: the mirror class, the restatement against the formula and
the evaluators' argument rules (CPU); b200_eval_diversity_device through EvaluatorHoldout / EvaluatorNegativeItemSample
against the restatement fed the same scores (-m gpu)."""
import os
import runpy

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.diversity_oracle import diversity_similarity, evaluate_scores_with_diversity
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

HERE = os.path.dirname(os.path.abspath(__file__))
_cases = runpy.run_path(os.path.join(HERE, "golden", "make_golden.py"), run_name="cases")
eval_case, eval_negative_case = _cases["eval_case"], _cases["eval_negative_case"]
ASSERT_TEXT = "item_diversity_matrix contains value greated than 1.0 or lower than 0.0"


def _random_D(n, seed, dtype=np.float64, cols=None):
    """Asymmetric, with entries in [0, 1]."""
    return np.random.default_rng(seed).random((n, cols or n)).astype(dtype)


def _formula(D, r):
    """sum_{a <= L-2} sum_{b <= L-1, b != a} D[r_a, r_b] / (L (L - 1)), as a plain double loop."""
    L = len(r)
    s = 0.0
    for a in range(L - 1):
        for b in range(L):
            if b != a:
                s += float(D[r[a], r[b]])
    return s / (L * (L - 1))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_mirror_class_asserts_like_the_reference():
    from recsys2019_deeplearning_evaluation_b200.evaluation import Diversity_similarity
    for bad in (-1e-9, 1.0 + 1e-6, np.nan):
        D = np.full((4, 4), 0.5)
        D[2, 1] = bad
        with pytest.raises(AssertionError, match="^" + ASSERT_TEXT + "$"):
            Diversity_similarity(D)
    for dtype in (np.float32, np.float64):
        D = _random_D(5, 1, dtype)
        D[0, 0], D[1, 1] = 0.0, 1.0
        assert Diversity_similarity(D).item_diversity_matrix is D


def test_oracle_against_the_formula():
    """An asymmetric D, so that the skipped last row is visible."""
    rng = np.random.default_rng(3)
    D = _random_D(50, 4)
    for L in (2, 3, 7, 31, 50):
        for _ in range(5):
            r = rng.permutation(50)[:L]
            assert np.isclose(diversity_similarity(D, r), _formula(D, r), rtol=1e-13, atol=0)
    r = np.array([4, 9, 2])
    only_last_row = np.zeros((10, 10))
    only_last_row[2, :] = 1.0
    assert diversity_similarity(only_last_row, r) == 0.0
    only_last_column = np.zeros((10, 10))
    only_last_column[:, 2] = 1.0
    assert diversity_similarity(only_last_column, r) == 2.0 / 6.0
    for r in (np.array([], dtype=np.int64), np.array([3])):
        with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
            diversity_similarity(D, r)


def test_oracle_lists_are_evaluate_scores_lists():
    """diversity_oracle restates evaluate_scores' users and ranking: the list-only metric AVERAGE_POPULARITY recomputed on
    its lists must be evaluate_scores' own, on every golden configuration and the negative-sample case."""
    from oracle.diversity_oracle import recommendation_lists
    from oracle.evaluator_oracle import evaluate_scores
    cases = [eval_case(n) for n in range(3)]
    train, test, neg, S, kw = eval_negative_case()
    cases.append((train, test, S, dict(kw, URM_test_negative=neg)))
    for train, test, S, kw in cases:
        users, lists = recommendation_lists(train, test, S, **kw)
        pop = np.ediff1d(sps.csc_matrix(train).indptr).astype(np.float64)
        pop /= pop.max()
        ref = evaluate_scores(train, test, S, **kw)
        for c in kw["cutoff_list"]:
            mine = sum(pop[r[:c]].sum() / len(r[:c]) for r in lists if len(r[:c])) / len(users)
            assert np.isclose(mine, ref[c]["AVERAGE_POPULARITY"], rtol=1e-13, atol=0)


def test_evaluator_constructor_rules():
    from recsys2019_deeplearning_evaluation_b200.evaluation import (Diversity_similarity, EvaluatorHoldout,
                                                                   EvaluatorNegativeItemSample)
    train, test, neg, S, kw = eval_negative_case()
    n_items = test.shape[1]
    ev = EvaluatorHoldout(test, [5], diversity_object=Diversity_similarity(_random_D(n_items, 1, np.float32)), verbose=False)
    assert ev._div.dtype == np.float32 and ev._div.shape == (n_items, n_items)
    big = _random_D(n_items + 3, 2, cols=n_items + 7)
    ev = EvaluatorNegativeItemSample(test, neg, [5], diversity_object=Diversity_similarity(big), verbose=False)
    assert ev._div.dtype == np.float64 and np.array_equal(ev._div, big[:n_items, :n_items])

    class Holder(object):  # any object with the attribute, as the reference's own class
        item_diversity_matrix = (np.random.default_rng(5).random((n_items, n_items)) < 0.5).astype(np.int8)

    ev = EvaluatorHoldout(test, [5], diversity_object=Holder(), verbose=False)
    assert ev._div.dtype == np.float64 and np.array_equal(ev._div, Holder.item_diversity_matrix)
    for shape in ((n_items - 1, n_items), (n_items, n_items - 1), (n_items,), (2, n_items, n_items)):
        Holder.item_diversity_matrix = np.zeros(shape)
        with pytest.raises(ValueError):
            EvaluatorHoldout(test, [5], diversity_object=Holder(), verbose=False)
        with pytest.raises(ValueError):
            EvaluatorNegativeItemSample(test, neg, [5], diversity_object=Holder(), verbose=False)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _stub(train, S):
    import torch
    from recsys2019_deeplearning_evaluation_b200.recommenders import BaseRecommender

    class Stub(BaseRecommender):
        RECOMMENDER_NAME = "Stub"

        def __init__(self, URM_train, S):
            super(Stub, self).__init__(URM_train, verbose=False)
            self._S = torch.from_numpy(np.ascontiguousarray(S, np.float32)).cuda()

        def _scores_device(self, d_users, items_to_compute=None):
            return self._S[d_users.long()].contiguous()

    return Stub(train, S)


def _evaluate(test, rec, D, block_size=None, neg=None, **kw):
    from recsys2019_deeplearning_evaluation_b200.evaluation import (Diversity_similarity, EvaluatorHoldout,
                                                                   EvaluatorNegativeItemSample)
    div = None if D is None else Diversity_similarity(D)
    if neg is None:
        ev = EvaluatorHoldout(test, diversity_object=div, verbose=False, **kw)
    else:
        ev = EvaluatorNegativeItemSample(test, neg, diversity_object=div, verbose=False, **kw)
    return ev.evaluateRecommender(rec, block_size=block_size)


def _check(res, ref, rtol_div, rtol_other=1e-9):
    assert set(res) == set(ref)
    for c in ref:
        assert set(res[c]) == set(ref[c])
        for k, v in ref[c].items():
            rtol = rtol_div if k == "DIVERSITY_SIMILARITY" else rtol_other
            assert np.isclose(res[c][k], v, rtol=rtol, atol=0 if k == "DIVERSITY_SIMILARITY" else 1e-12), \
                "cutoff %s %s: %r vs %r" % (c, k, res[c][k], v)


def _check_others_unchanged(res, res_plain):
    """Every metric but DIVERSITY_SIMILARITY as without the diversity object (up to the order of the fp64 atomics)."""
    for c in res_plain:
        assert [k for k in res[c] if k != "DIVERSITY_SIMILARITY"] == list(res_plain[c])
        for k, v in res_plain[c].items():
            assert np.isclose(res[c][k], v, rtol=1e-12, atol=0) or (np.isnan(v) and np.isnan(res[c][k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(3))
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("block_size", [1, 7, 1000])
def test_holdout_matches_the_oracle(n, dtype, block_size):
    from recsys2019_deeplearning_evaluation_b200.evaluation import METRIC_NAMES
    train, test, S, kw = eval_case(n)
    D = _random_D(test.shape[1], 10 + n, dtype)
    rec = _stub(train, S)
    if 1 in kw["cutoff_list"]:  # a list of one item: the reference divides 0.0 by 0
        with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
            evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D, **kw)
        with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
            _evaluate(test, rec, D, block_size, **kw)
        kw["cutoff_list"] = [2 if c == 1 else c for c in kw["cutoff_list"]]
    res, text = _evaluate(test, rec, D, block_size, **kw)
    _check(res, evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D, **kw), 1e-10)
    res_plain, _ = _evaluate(test, rec, None, block_size, **kw)
    _check_others_unchanged(res, res_plain)
    i = METRIC_NAMES.index("AVERAGE_POPULARITY") + 1
    for c in kw["cutoff_list"]:
        assert list(res[c]) == METRIC_NAMES[:i] + ["DIVERSITY_SIMILARITY"] + METRIC_NAMES[i:]
        assert "AVERAGE_POPULARITY: {:.7f}, DIVERSITY_SIMILARITY: {:.7f}, DIVERSITY_MEAN_INTER_LIST: ".format(
            res[c]["AVERAGE_POPULARITY"], res[c]["DIVERSITY_SIMILARITY"]) in text
    assert list(res_plain[kw["cutoff_list"][0]]) == METRIC_NAMES


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_exact_sums(dtype):
    """Multiples of 1/256 make every per-user sum exact in fp64, whatever the order."""
    train, test, S, kw = eval_case(0)
    D = (np.random.default_rng(20).integers(0, 257, (test.shape[1], test.shape[1])) / 256.0).astype(dtype)
    res, _ = _evaluate(test, _stub(train, S), D, 64, **kw)
    _check(res, evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D, **kw), 1e-13)


@pytest.mark.gpu
def test_long_lists():
    """Full 1 024-item lists (L_max = 1 024), cutoffs unsorted and repeated, D larger than the catalogue."""
    n_users, n_items = 48, 2100
    rng = np.random.default_rng(30)
    train = synth_urm(n_users, n_items, 0.01, seed=31, values="ratings")
    test = synth_urm(n_users, n_items, 0.01, seed=32, values="ratings")
    S = rng.random((n_users, n_items)).astype(np.float32)
    D = _random_D(n_items + 40, 33, np.float32)
    res, _ = _evaluate(test, _stub(train, S), D, 16, cutoff_list=[1024, 2, 37, 37, 3])
    # the restatement accumulates per distinct cutoff value, so it gets each value once
    ref = evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D[:n_items, :n_items], cutoff_list=[1024, 2, 37, 3])
    _check(res, ref, 1e-10)


@pytest.mark.gpu
def test_non_finite_scores():
    """+inf at the top of some rows, NaN and -inf inside the table: the lists are the finite entries, as the oracle's
    isfinite rule (and metrics_kernel) define them."""
    train, test, S, kw = eval_case(0)
    S = S.copy()
    rng = np.random.default_rng(40)
    n_users, n_items = S.shape
    for u in range(0, n_users, 3):
        S[u, rng.choice(n_items, 3, replace=False)] = np.inf
    for u in range(1, n_users, 4):
        S[u, rng.choice(n_items, 10, replace=False)] = np.nan
    for u in range(2, n_users, 5):
        S[u, rng.choice(n_items, 40, replace=False)] = -np.inf
    D = _random_D(n_items, 41)
    res, _ = _evaluate(test, _stub(train, S), D, 50, **kw)
    _check(res, evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D, **kw), 1e-10)


@pytest.mark.gpu
def test_short_lists_raise():
    train, test, S, kw = eval_case(0)
    D = _random_D(test.shape[1], 50)
    rec = _stub(train, S)
    with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
        _evaluate(test, rec, D, cutoff_list=[5, 1])
    S = S.copy()
    S[np.flatnonzero(np.diff(test.indptr))[-1], :] = -np.inf  # an evaluated user with no recommendation at all
    with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
        evaluate_scores_with_diversity(train, test, S, item_diversity_matrix=D, cutoff_list=[5])
    with pytest.raises(ZeroDivisionError, match="^float division by zero$"):
        _evaluate(test, _stub(train, S), D, cutoff_list=[5])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_negative_item_sample(dtype):
    train, test, neg, S, kw = eval_negative_case()
    D = _random_D(test.shape[1], 60, dtype)
    rec = _stub(train, S)
    with pytest.raises(ZeroDivisionError, match="^float division by zero$"):  # its cutoff 1
        _evaluate(test, rec, D, neg=neg, **kw)
    kw = dict(cutoff_list=[2, 5, 10, 40])
    for block_size in (1, 7, 1000):
        res, _ = _evaluate(test, rec, D, block_size, neg=neg, **kw)
        _check(res, evaluate_scores_with_diversity(train, test, S, URM_test_negative=neg, item_diversity_matrix=D, **kw), 1e-10)
        res_plain, _ = _evaluate(test, rec, None, block_size, neg=neg, **kw)
        _check_others_unchanged(res, res_plain)


@pytest.mark.gpu
def test_itemknn_with_a_content_diversity_matrix():
    """The use the reference's docstring describes: D = 1 - the cosine similarity of the items' features, on a fitted
    ItemKNN, against the restatement fed the model's own scores (tolerance as test_cuda_evaluates_itemknn_like_the_oracle:
    the score block is summed with atomics, so near-equal scores may swap)."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import ItemKNNCFRecommender
    train = synth_urm(3000, 1500, 0.02, seed=61, values="ratings", popularity=0.8)
    test = synth_urm(3000, 1500, 0.004, seed=62, values="ratings")
    ICM = synth_urm(1500, 200, 0.05, seed=63, values="continuous").toarray()
    norm = np.linalg.norm(ICM, axis=1)
    norm[norm == 0] = 1.0
    X = ICM / norm[:, None]
    D = np.clip(1.0 - X @ X.T, 0.0, 1.0)
    rec = ItemKNNCFRecommender(train, verbose=False)
    rec.fit(topK=40, shrink=10)
    kw = dict(cutoff_list=[5, 20, 100], min_ratings_per_user=2)
    res, _ = _evaluate(test, rec, D, **kw)
    ref = evaluate_scores_with_diversity(train, test, rec._compute_item_score(np.arange(3000)), item_diversity_matrix=D, **kw)
    _check(res, ref, 1e-4, 1e-4)


@pytest.mark.gpu
def test_upload_once_and_one_launch_per_block():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.evaluation import Diversity_similarity, EvaluatorHoldout
    train, test, S, kw = eval_case(0)
    rec = _stub(train, S)
    D = _random_D(test.shape[1], 70, np.float32)
    ev = EvaluatorHoldout(test, diversity_object=Diversity_similarity(D), verbose=False, **kw)
    ev_plain = EvaluatorHoldout(test, verbose=False, **kw)
    block_size = 16
    n_blocks = -(-len(ev.users_to_evaluate) // block_size)
    counts = []
    for e in (ev_plain, ev, ev_plain, ev):
        before = _lib.launch_count()
        res = e.evaluateRecommender(rec, block_size=block_size)
        counts.append(_lib.launch_count() - before)
        if e is ev:
            ptr = ev._d_div.data_ptr()
            if len(counts) == 2:
                first, first_ptr = res, ptr
    assert counts[0] == counts[2] and counts[1] == counts[3] == counts[0] + n_blocks
    assert ptr == first_ptr
    _check(res[0], first[0], 1e-13, 1e-13)  # equal up to the order of the fp64 atomics across users
