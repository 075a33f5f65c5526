"""-m gpu: EvaluatorNegativeItemSample on blocks of users -- the candidate scorers (csrc/score.cu cand_* kernels) against
the models' own dense score blocks, and the whole evaluation against the numpy restatement (oracle/evaluator_oracle.py)."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle.evaluator_oracle import evaluate_scores
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu


def _candidates(n_users, n_items, lens, seed):
    """CSR of sorted, distinct candidate items per user (lens[u] of them)."""
    rng = np.random.default_rng(seed)
    rows = [np.sort(rng.choice(n_items, size=int(l), replace=False)) for l in lens]
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    idx = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return sps.csr_matrix((np.ones(len(idx), np.float32), idx, ptr), shape=(n_users, n_items))


def _cand_scores(rec, users, C):
    """rec._candidate_scores_device for the given users (rows of C in that order), as a host array aligned with C[users]."""
    import torch
    sub = C[users]
    d_users = rec._users_tensor(users)
    d_ptr = torch.from_numpy(sub.indptr.astype(np.int32)).cuda()
    d_idx = torch.from_numpy(sub.indices.astype(np.int32)).cuda()
    out = torch.full((max(sub.nnz, 1),), float("nan"), dtype=torch.float32, device="cuda")
    rec._candidate_scores_device(d_users, d_ptr, d_idx, out)
    return sub, out.cpu().numpy()[:sub.nnz]


def _at_candidates(rec, users, sub):
    dense = rec._compute_item_score(users)
    return dense[np.repeat(np.arange(len(users)), np.diff(sub.indptr)), sub.indices]


def _check_scorer(rec, exact=False, bitwise=False, seed=0, C=None):
    n_users, n_items = rec.URM_train.shape
    rng = np.random.default_rng(seed)
    if C is None:
        C = _candidates(n_users, n_items, rng.integers(0, min(n_items, 150), size=n_users), seed)
    users = rng.permutation(n_users)[:min(n_users, 300)]
    sub, got = _cand_scores(rec, users, C)
    want = _at_candidates(rec, users, sub)
    if bitwise:
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    elif exact:
        assert np.array_equal(got, want)
    else:  # the dense block adds with atomics in no fixed order, the candidate kernels in a fixed one
        assert np.allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())


def _int_urm(n_users, n_items, density, seed):
    X = synth_urm(n_users, n_items, density, seed=seed, values="ratings")
    return X


def test_item_similarity_scorer_exact_on_integers():
    """ItemKNNCustomSimilarity with an integer W on integer ratings: every sum is exact in fp32."""
    from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCustomSimilarityRecommender
    X = _int_urm(400, 300, 0.05, 1)
    W = sps.random(300, 300, density=0.05, random_state=2, format="csr", dtype=np.float32)
    W.data = np.round(W.data * 8 - 4).astype(np.float32)
    rec = ItemKNNCustomSimilarityRecommender(X, verbose=False)
    rec.fit(W)
    _check_scorer(rec, exact=True)


def test_user_similarity_scorer_exact_on_integers():
    from recsys2019_deeplearning_evaluation_b200.recommenders import UserKNNCFRecommender
    X = _int_urm(400, 300, 0.05, 3)
    W = sps.random(400, 400, density=0.03, random_state=4, format="csr", dtype=np.float32)
    W.data = np.round(W.data * 8 - 4).astype(np.float32)
    rec = UserKNNCFRecommender(X, verbose=False)
    rec.W_sparse = W
    _check_scorer(rec, exact=True)


def test_long_profiles_and_columns():
    """Profiles longer than the shared-memory stage (2 048) and columns longer than the profile: both walk directions."""
    from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCustomSimilarityRecommender
    X = _int_urm(60, 5000, 0.5, 5)
    W = sps.random(5000, 5000, density=0.02, random_state=6, format="csr", dtype=np.float32)
    W.data = np.round(W.data * 8 - 4).astype(np.float32)
    W = sps.hstack([W[:, :10], sps.csr_matrix(np.full((5000, 1), 2, np.float32)), W[:, 11:]], format="csr")  # a dense column
    rec = ItemKNNCustomSimilarityRecommender(X, verbose=False)
    rec.fit(W)
    keep = (np.arange(5000) % 97 < 3) | (np.arange(5000) == 10)  # item 10 and 155 others for every user
    C = sps.csr_matrix(np.tile(keep, (60, 1)).astype(np.float32))
    _check_scorer(rec, exact=True, seed=7, C=C)


def test_fitted_similarity_models():
    from recsys2019_deeplearning_evaluation_b200.recommenders import (ItemKNNCFRecommender, UserKNNCFRecommender, P3alphaRecommender,
                                                                      SLIM_BPR_Cython, EASE_R_Recommender)
    X = synth_urm(500, 250, 0.05, seed=8, values="continuous")
    for cls, kw in ((ItemKNNCFRecommender, dict(topK=30, shrink=5)), (UserKNNCFRecommender, dict(topK=30, shrink=5)),
                    (P3alphaRecommender, dict(topK=40, alpha=0.8)),
                    (SLIM_BPR_Cython, dict(epochs=3, topK=20, learning_rate=0.05, random_seed=2, sgd_mode="adagrad")),
                    (EASE_R_Recommender, dict(topK=None, l2_norm=50.0)), (EASE_R_Recommender, dict(topK=40, l2_norm=50.0))):
        rec = cls(X, verbose=False)
        rec.fit(**kw)
        _check_scorer(rec, seed=9)


def test_ease_dense_exact_on_integers():
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    import torch
    X = _int_urm(300, 200, 0.06, 10)
    rec = EASE_R_Recommender(X, verbose=False)
    rec.fit(topK=None, l2_norm=50.0)
    B = np.round(np.random.default_rng(11).standard_normal((200, 200)) * 4).astype(np.float32)
    rec._d_B = torch.from_numpy(B).cuda()
    _check_scorer(rec, exact=True)


def test_mf_scorers_bitwise():
    from recsys2019_deeplearning_evaluation_b200.recommenders import (MatrixFactorization_BPR_Cython, MatrixFactorization_FunkSVD_Cython,
                                                                      IALSRecommender)
    X = synth_urm(600, 300, 0.05, seed=12, values="ratings")
    bpr = MatrixFactorization_BPR_Cython(X, verbose=False)
    bpr.fit(epochs=2, batch_size=50, num_factors=24, learning_rate=0.05, sgd_mode="adagrad", random_seed=3)
    fk = MatrixFactorization_FunkSVD_Cython(X, verbose=False)
    fk.fit(epochs=2, batch_size=64, num_factors=13, learning_rate=0.02, sgd_mode="adam", use_bias=True, random_seed=3)
    assert fk.use_bias
    np.random.seed(5)
    ials = IALSRecommender(X, verbose=False)
    ials.fit(epochs=2, num_factors=20)
    for rec in (bpr, fk, ials):
        _check_scorer(rec, bitwise=True, seed=13)


def test_fallback_scores_through_the_block():
    """TopPop and a subclass overriding _scores_device take the block + gather path, never a family kernel."""
    import test_evaluation as TE
    from recsys2019_deeplearning_evaluation_b200.nonpersonalized import TopPop
    from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCustomSimilarityRecommender
    X = _int_urm(300, 200, 0.05, 14)
    tp = TopPop(X, verbose=False)
    tp.fit()
    _check_scorer(tp, exact=True)

    class Negated(ItemKNNCustomSimilarityRecommender):
        def _scores_device(self, d_users, items_to_compute=None):
            return -super(Negated, self)._scores_device(d_users)

    neg = Negated(X, verbose=False)
    neg.fit(sps.random(200, 200, density=0.05, random_state=15, format="csr", dtype=np.float32))
    _check_scorer(neg)
    sub, got = _cand_scores(neg, np.arange(20), _candidates(300, 200, np.full(300, 30), 16))
    plain = ItemKNNCustomSimilarityRecommender(X, verbose=False)
    plain.W_sparse = neg.W_sparse
    _, want = _cand_scores(plain, np.arange(20), _candidates(300, 200, np.full(300, 30), 16))
    assert np.allclose(got, -want, rtol=1e-6, atol=1e-6) and np.abs(want).max() > 0
    stub = TE._stub(X, np.random.default_rng(17).standard_normal((300, 200)).astype(np.float32))
    _check_scorer(stub, exact=True)


# ------------------------------------------------------------------------------------------- evaluator vs restatement
def _negatives(test, lens, n_items, seed):
    """Per user max(lens[u] - n_test, 0) negatives outside her test items."""
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(test.shape[0]):
        t = set(test.indices[test.indptr[u]:test.indptr[u + 1]].tolist())
        k = max(int(lens[u]) - len(t), 0)
        pool = np.setdiff1d(np.arange(n_items), np.fromiter(t, np.int64, len(t)))
        pick = rng.choice(pool, size=min(k, len(pool)), replace=False)
        rows.append(np.full(len(pick), u)); cols.append(pick)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    return sps.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(test.shape[0], n_items))


def _case(n_users, n_items, lens, seed, nonfinite=False, ties=False):
    rng = np.random.default_rng(seed)
    train = synth_urm(n_users, n_items, min(0.3, 60.0 / n_items), seed=seed, values="ratings")
    n_test = np.minimum(rng.integers(1, 4, size=n_users), np.maximum(lens, 1))
    rows = np.repeat(np.arange(n_users), n_test)
    cols = np.concatenate([rng.choice(n_items, size=k, replace=False) for k in n_test])
    test = sps.csr_matrix((rng.integers(1, 6, size=len(rows)).astype(np.float32), (rows, cols)), shape=(n_users, n_items))
    neg = _negatives(test, lens, n_items, seed + 1)
    S = rng.standard_normal((n_users, n_items)).astype(np.float32)
    if ties:
        S = np.round(S * 2).astype(np.float32)
    if nonfinite:
        m = rng.random(S.shape)
        S[m < 0.03] = np.nan
        S[(m >= 0.03) & (m < 0.05)] = np.inf
        S[(m >= 0.05) & (m < 0.07)] = -np.inf
    return train, test, neg, S


def _compare(res, ref, rtol=1e-9):
    import test_evaluation as TE
    TE._assert_close(res, ref, rtol, "negative-sample blocks")


def _run(train, test, neg, S, block_size, **kw):
    import test_evaluation as TE
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorNegativeItemSample
    ev = EvaluatorNegativeItemSample(test, neg, verbose=False, **kw)
    res, _ = ev.evaluateRecommender(TE._stub(train, S), block_size=block_size)
    _compare(res, evaluate_scores(train, test, S, URM_test_negative=neg, **kw))


@pytest.mark.parametrize("length", [1, 101, 1000, 5000])
@pytest.mark.parametrize("block_size", [1, 7, 1000])
def test_evaluator_matches_restatement_list_lengths(length, block_size):
    n_users = 12 if length == 5000 else 30
    n_items = 6000 if length >= 1000 else 400
    train, test, neg, S = _case(n_users, n_items, np.full(n_users, length), seed=length + block_size, ties=True)
    _run(train, test, neg, S, block_size, cutoff_list=[1, 5, 10, 1024])


@pytest.mark.parametrize("exclude_seen", [True, False])
def test_evaluator_seen_candidates_and_nonfinite_scores(exclude_seen):
    """Lists of every length class in one block, candidates that are train items, NaN / +-inf scores."""
    lens = np.array([1, 5, 101, 256, 257, 1000, 2500, 40] * 5)
    train, test, neg, S = _case(len(lens), 3000, lens, seed=21, nonfinite=True)
    cand = (test + neg).tocsr()
    assert cand.multiply(train).nnz > 0  # some candidates are seen items
    _run(train, test, neg, S, 16, cutoff_list=[1, 5, 10, 1024], exclude_seen=exclude_seen)


def test_evaluator_ignore_items_users_min_ratings():
    lens = np.array([101, 300, 1, 50] * 10)
    train, test, neg, S = _case(len(lens), 2000, lens, seed=22, ties=True)
    cand = (test + neg).tocsr()
    ignore_items = np.unique(cand.indices[::7])[:60]
    _run(train, test, neg, S, 7, cutoff_list=[10, 5, 1], ignore_items=ignore_items, ignore_users=[0, 3, 17],
         min_ratings_per_user=2)


def _real_model_case():
    rng = np.random.default_rng(30)
    train = synth_urm(800, 500, 0.04, seed=31, values="ratings", popularity=0.6)
    test = synth_urm(800, 500, 0.006, seed=32, values="ratings")
    neg = _negatives(test, np.full(800, 101), 500, 33)
    return rng, train, test, neg


@pytest.mark.parametrize("model", ["mf_bpr", "ials", "itemknn_int", "itemknn", "ease"])
def test_real_models_match_restatement(model):
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorNegativeItemSample
    from recsys2019_deeplearning_evaluation_b200 import recommenders as R
    from recsys2019_deeplearning_evaluation_b200.knn import ItemKNNCustomSimilarityRecommender
    _, train, test, neg = _real_model_case()
    rtol = 1e-9
    if model == "mf_bpr":
        rec = R.MatrixFactorization_BPR_Cython(train, verbose=False)
        rec.fit(epochs=2, batch_size=50, num_factors=16, learning_rate=0.05, sgd_mode="adagrad", random_seed=3)
    elif model == "ials":
        np.random.seed(7)
        rec = R.IALSRecommender(train, verbose=False)
        rec.fit(epochs=2, num_factors=12)
    elif model == "itemknn_int":
        W = sps.random(500, 500, density=0.04, random_state=34, format="csr", dtype=np.float32)
        W.data = np.round(W.data * 6 - 2).astype(np.float32)
        rec = ItemKNNCustomSimilarityRecommender(train, verbose=False)
        rec.fit(W)
    elif model == "itemknn":
        rec = R.ItemKNNCFRecommender(train, verbose=False)
        rec.fit(topK=40, shrink=10)
        rtol = 1e-4  # candidates tied within the fp32 rounding of their sums may swap (the block adds with atomics)
    else:
        rec = R.EASE_R_Recommender(train, verbose=False)
        rec.fit(topK=None, l2_norm=100.0)
        rtol = 1e-4
    kw = dict(cutoff_list=[1, 5, 10, 50], min_ratings_per_user=1)
    res, _ = EvaluatorNegativeItemSample(test, neg, verbose=False, **kw).evaluateRecommender(rec, block_size=128)
    ref = evaluate_scores(train, test, rec._compute_item_score(np.arange(800)), URM_test_negative=neg, **kw)
    _compare(res, ref, rtol)


def test_launches_scale_with_blocks_not_users():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorNegativeItemSample
    from recsys2019_deeplearning_evaluation_b200.recommenders import MatrixFactorization_BPR_Cython
    _, train, test, neg = _real_model_case()
    rec = MatrixFactorization_BPR_Cython(train, verbose=False)
    rec.fit(epochs=1, batch_size=50, num_factors=8, random_seed=3)
    ev = EvaluatorNegativeItemSample(test, neg, cutoff_list=[10], verbose=False)
    n_users = len(ev.users_to_evaluate)
    assert n_users > 300
    ev.evaluateRecommender(rec, block_size=100)  # device copies and caches made once
    before = _lib.launch_count()
    ev.evaluateRecommender(rec, block_size=100)
    n_blocks = -(-n_users // 100)
    launches = _lib.launch_count() - before
    assert launches <= 4 * n_blocks + 4, (launches, n_blocks)
