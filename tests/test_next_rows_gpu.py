"""-m gpu: the SURVEY.md 8(f).4 trainers through the C ABI against their oracles (pinned to the reference on CPU in
tests/test_oracle_next_rows.py) and against the reference's own golden output:
  * SLIM-BPR with train_with_sparse_weights=True (tree mode semantics: cell-exists map, in-epoch row cuts, get_S cutting in place)
  * AsySVD (sequential kernel on the reference's glibc sample stream)
  * SLIM ElasticNet (Gram-matrix coordinate descent, one CTA per item)."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import elasticnet_oracle
from oracle.sgd_oracle import MFOracle, SLIMOracle
from test_oracle_next_rows import ASY_CASES, ENET_CASES, TREE_CASES, asy_urm, enet_urm, tree_kwargs, tree_urm

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "next_rows_golden.npz")


# ------------------------------------------------------------------ tree-sparse SLIM-BPR
def _slim():
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    return SLIM_BPR_Cython_Epoch


def _assert_same_cut(S, R, topk, atol=2e-6, rtol=1e-4):
    """S (fp32 device state) against R (fp64 oracle): the same cells, the same values -- except that a row cut may fall
    between two cells whose fp64 values differ by less than fp32 resolves; such a row may swap cells of (almost) the cut value."""
    same = (S != 0) == (R != 0)
    if not same.all():
        bad_rows = np.flatnonzero(~same.all(axis=1))
        assert topk, "cells differ without any cut"
        for r in bad_rows:
            a, b = S[r][~same[r]], R[r][~same[r]]
            v = np.concatenate([a[a != 0], b[b != 0]])
            kth = np.sort(R[r][R[r] != 0])[0] if (R[r] != 0).any() else 0.0  # smallest survivor = the cut
            assert np.abs(v - kth).max() <= 1e-5 * max(1.0, abs(kth)) + 1e-6, (r, v, kth)
        assert len(bad_rows) <= max(1, S.shape[0] // 50)
    assert np.allclose(np.where(same, S, 0), np.where(same, R, 0), rtol=rtol, atol=atol), float(np.abs(np.where(same, S - R, 0)).max())


@pytest.mark.parametrize("n", range(len(TREE_CASES)))
def test_tree_mode_matches_the_oracle_epoch_by_epoch(n):
    case = TREE_CASES[n]
    g, o = _slim()(tree_urm(case), **tree_kwargs(case)), SLIMOracle(tree_urm(case), **tree_kwargs(case))
    for e in range(3):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
        S = g.get_S()                      # cuts the device state in place, like the reference's get_S
        R = o.get_S_tree()
        assert sps.issparse(S) and S.shape == (case[1], case[1])
        _assert_same_cut(S.toarray(), R.toarray(), case[3])
    g._dealloc()


def test_tree_mode_matches_the_reference_golden():
    z = np.load(GOLD)
    for n in (1, 2):
        case = TREE_CASES[n]
        g = _slim()(tree_urm(case), **tree_kwargs(case))
        for e in range(3):
            g.epochIteration_Cython()
            _assert_same_cut(g.get_S().toarray(), z["tree%d_S%d" % (n, e)], case[3])


def test_tree_mode_cuts_inside_the_epoch():
    """1000 users: rebalance_tree runs after samples 200, 400, 600, 800 (pyx:318-319); with 943 users it never does."""
    X = tree_urm(TREE_CASES[2])
    kw = dict(tree_kwargs(TREE_CASES[2]), sgd_mode="adagrad", topK=5)
    g = _slim()(X, **kw)
    g.epochIteration_Cython()
    D = g.get_S_dense()                    # the raw state: no diagonal cells, no get_S cut
    o = SLIMOracle(X, **kw)
    o.epochIteration_Cython()
    R = o.S_full()
    per_row = (D != 0).sum(axis=1)
    assert per_row.max() > 5               # rows grow again after the last cut at sample 800 ...
    assert np.array_equal(D != 0, R != 0)  # ... exactly like the oracle's
    assert np.allclose(D, R, rtol=1e-4, atol=2e-6)


def test_tree_mode_argument_rules():
    X = tree_urm(TREE_CASES[0])
    g = _slim()(X, train_with_sparse_weights=True, symmetric=True, topK=10, random_seed=1)
    assert g.symmetric is False            # pyx:111-112
    with pytest.raises(ValueError):
        _slim()(X, train_with_sparse_weights=True, hogwild=True, sampler="philox", random_seed=1)


def test_slim_recommender_tree_mode_keeps_the_row_topk():
    from recsys2019_deeplearning_evaluation_b200.recommenders import SLIM_BPR_Cython
    X = tree_urm(TREE_CASES[1])
    r = SLIM_BPR_Cython(X, verbose=False)
    r.fit(epochs=2, train_with_sparse_weights=True, topK=10, random_seed=3, learning_rate=0.05, sgd_mode="adagrad")
    W = r.W_sparse
    assert sps.issparse(W) and (np.diff(W.tocsr().indptr) <= 10).all() and W.nnz > 0   # SLIM_BPR_Cython.py:178-179
    assert r._compute_item_score(np.arange(5)).shape == (5, X.shape[1])


# ------------------------------------------------------------------ AsySVD
def _mf():
    from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch
    return MatrixFactorization_Cython_Epoch


# fp32 parameters and optimiser state against the fp64 reference over 2 x 2 881 strictly dependent samples: a float32
# re-run of the oracle's recursion sits at 4e-7 (sgd, adagrad) ... 1.8e-5 (adam, rmsprop) from it; the bar leaves 5x.
ASY_RTOL, ASY_ATOL = 1e-3, 1e-4


@pytest.mark.parametrize("n", range(len(ASY_CASES)))
def test_asysvd_matches_the_oracle_on_the_glibc_stream(n):
    kw = ASY_CASES[n]
    common = dict(n_factors=8, algorithm_name="ASY_SVD", batch_size=1, learning_rate=0.01, random_seed=42)
    X = asy_urm()
    g = _mf()(X, **common, **kw)
    o = MFOracle(X, record=2 * (X.nnz + 1), **common, **kw)
    dense = sps.csr_matrix(X, dtype=np.float32).toarray()
    for e in range(2):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
        u, i, r = g.get_samples()
        ou, oi, _ = o.recorded()
        assert len(u) == X.nnz + 1                                     # pyx:402
        assert np.array_equal(u, ou[e * len(u):(e + 1) * len(u)]) and np.array_equal(i, oi[e * len(u):(e + 1) * len(u)])
        assert np.array_equal(r, dense[u, i])  # the oracle records u and i: r is the rating of a positive, 0 for a negative
    assert g.get_USER_factors().shape == (X.shape[1], 8)               # Y: one row per ITEM (pyx:163-166)
    names = ("get_USER_factors", "get_ITEM_factors") + (("get_USER_bias", "get_ITEM_bias", "get_GLOBAL_bias") if kw["use_bias"] else ())
    for name in names:
        a, b = np.asarray(getattr(g, name)(), np.float64), np.asarray(getattr(o, name)(), np.float64)
        assert np.allclose(a, b, rtol=ASY_RTOL, atol=ASY_ATOL), "%s: max abs diff %.3e" % (name, float(np.abs(a - b).max()))
    g._dealloc()


def test_asysvd_matches_the_reference_golden():
    z = np.load(GOLD)
    g = _mf()(asy_urm(), n_factors=8, algorithm_name="ASY_SVD", batch_size=1, learning_rate=0.01, random_seed=42, **ASY_CASES[1])
    for _ in range(2):
        g.epochIteration_Cython()
    got = [g.get_USER_factors(), g.get_ITEM_factors(), g.get_USER_bias(), g.get_ITEM_bias(), np.array([float(g.get_GLOBAL_bias())])]
    for k, a in enumerate(got):
        assert np.allclose(a, z["asy1_%d" % k], rtol=ASY_RTOL, atol=ASY_ATOL), k


def test_asysvd_wide_factors_and_argument_rules():
    X = asy_urm()
    common = dict(algorithm_name="ASY_SVD", learning_rate=0.005, random_seed=5, sgd_mode="adagrad", use_bias=True,
                  negative_interactions_quota=0.2, user_reg=1e-3, item_reg=1e-3)
    g, o = _mf()(X, n_factors=160, batch_size=1, **common), MFOracle(X, n_factors=160, batch_size=1, **common)   # f > 128: lanes loop
    g.epochIteration_Cython()
    o.epochIteration_Cython()
    for name in ("get_USER_factors", "get_ITEM_factors", "get_ITEM_bias"):
        a, b = getattr(g, name)(), getattr(o, name)()
        assert np.allclose(a, b, rtol=ASY_RTOL, atol=ASY_ATOL), name
    with pytest.raises(AssertionError):
        _mf()(X, n_factors=4, batch_size=2, **common)                  # pyx:399
    with pytest.raises(ValueError):
        _mf()(X, n_factors=4, batch_size=1, sampler="philox", **common)


@pytest.mark.parametrize("f,mode", [(10, "adagrad"), (50, "adam"), (3, "sgd"), (17, "rmsprop")])
def test_asysvd_factor_counts_that_are_not_multiples_of_four(f, mode):
    """The device rows are padded to float4s (the padding stays 0 under every optimiser); the reference's usual factor counts
    (10, 50, ...) take this path."""
    kw = dict(n_factors=f, algorithm_name="ASY_SVD", batch_size=1, learning_rate=0.01, random_seed=42, sgd_mode=mode, use_bias=True,
              negative_interactions_quota=0.3, user_reg=1e-3, item_reg=2e-3, bias_reg=1e-3)
    X = asy_urm()
    g, o = _mf()(X, **kw), MFOracle(X, **kw)
    g.epochIteration_Cython()
    o.epochIteration_Cython()
    assert g.get_USER_factors().shape == (X.shape[1], f) and g.get_ITEM_factors().shape == (X.shape[1], f)
    for name in ("get_USER_factors", "get_ITEM_factors", "get_USER_bias", "get_ITEM_bias"):
        a, b = getattr(g, name)(), getattr(o, name)()
        assert np.allclose(a, b, rtol=ASY_RTOL, atol=ASY_ATOL), "%s: max abs diff %.3e" % (name, float(np.abs(a - b).max()))


def test_asysvd_recommender_estimates_user_factors_from_profiles():
    from recsys2019_deeplearning_evaluation_b200.recommenders import MatrixFactorization_AsySVD_Cython
    X = asy_urm()
    r = MatrixFactorization_AsySVD_Cython(X, verbose=False)
    r.fit(epochs=1, num_factors=8, learning_rate=0.01, random_seed=42, sgd_mode="adagrad", use_bias=True, batch_size=64)
    Y = r.ITEM_factors_Y
    assert Y.shape == (X.shape[1], 8) and r.USER_factors.shape == (X.shape[0], 8)
    ref = X.dot(Y) / np.sqrt(np.maximum(np.ediff1d(X.indptr), 1))[:, None]   # MatrixFactorization_Cython.py:256-277
    assert np.allclose(r.USER_factors, ref, rtol=1e-6, atol=1e-9)
    assert r._compute_item_score(np.arange(4)).shape == (4, X.shape[1])


# ------------------------------------------------------------------ SLIM ElasticNet
def _enet_fit(X, l1_ratio, alpha, positive, topK):
    from recsys2019_deeplearning_evaluation_b200.recommenders import SLIMElasticNetRecommender
    r = SLIMElasticNetRecommender(X, verbose=False)
    r.fit(l1_ratio=l1_ratio, alpha=alpha, positive_only=positive, topK=topK)
    return r


@pytest.mark.parametrize("n", range(len(ENET_CASES)))
def test_elasticnet_matches_the_oracle_and_the_reference_golden(n):
    values, l1_ratio, alpha, positive, topK = ENET_CASES[n]
    X = enet_urm(values)
    r = _enet_fit(X, l1_ratio, alpha, positive, topK)
    W = r.W_sparse.toarray()
    assert sps.issparse(r.W_sparse) and r.W_sparse.dtype == np.float32 and (np.diag(W) == 0).all()
    # same algorithm, same coordinate order, fp32 against fp64: tight
    O = elasticnet_oracle.slim_elasticnet_fit(X, l1_ratio, alpha, positive, topK).toarray()
    diff = (W != 0) != (O != 0)
    assert diff.sum() <= 0.002 * (O != 0).sum(), int(diff.sum())
    assert np.abs(np.where(diff, 0, W - O)).max() < 2e-5, float(np.abs(np.where(diff, 0, W - O)).max())
    # the reference's own output (random coordinate order, unseeded): inside its run-to-run band (test_oracle_next_rows.py)
    G = np.load(GOLD)["enet%d_W" % n]
    assert np.abs(W - G).max() < 3e-4
    assert ((W != 0) != (G != 0)).sum() <= 0.002 * (G != 0).sum()
    it = r._n_iter.cpu().numpy()
    assert it.min() >= 1 and it.max() <= 100


def test_elasticnet_large_catalogue_uses_the_global_workspace_and_cold_items_stay_empty():
    """3 * n * 4 bytes > 200 KB (n > 17 066): w / H / q move to the L2-resident workspace; items nobody rated get no model and
    are nobody's neighbour."""
    from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
    n_items = 17500
    X = sps.lil_matrix(synth_urm(600, n_items, 0.004, seed=9, values="binary"))
    X[:, 100] = 0
    X = sps.csr_matrix(X)
    r = _enet_fit(X, 0.1, 1e-3, True, 10)
    W = r.W_sparse.tocsc()
    assert W[:, 100].nnz == 0 and W.tocsr()[100].nnz == 0
    cols = [5, 17499]
    Xd = X.toarray().astype(np.float64)
    G = Xd.T @ Xd
    for j in cols:
        Q = G.copy(); Q[j, :] = 0; Q[:, j] = 0
        q = G[:, j].copy(); q[j] = 0
        w, _, _ = elasticnet_oracle.enet_cd_gram(Q, q, G[j, j], 1e-3 * 0.1 * 600, 1e-3 * 0.9 * 600, True)
        rows, vals = elasticnet_oracle.select_topk(w, 10)
        ref = np.zeros(n_items); ref[rows] = vals
        got = np.asarray(W[:, j].todense()).ravel()
        assert np.abs(got - ref).max() < 2e-5, (j, float(np.abs(got - ref).max()))


def test_dense_topk_drop_last_mode():
    """mode 2 of the dense top-K kernel: min(nnz - 1, K) largest non-zero values per line (SLIMElasticNetRecommender.py:103)."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import dense_topk_to_sparse
    rng = np.random.default_rng(0)
    n, K = 300, 12
    D = rng.standard_normal((n, n)).astype(np.float32)
    D[rng.random((n, n)) < 0.93] = 0
    D[3] = 0; D[4] = 0; D[4, 7] = 0.5; D[5] = 0; D[5, :3] = [-1.0, 2.0, 0.25]
    T = dense_topk_to_sparse(torch.from_numpy(D).cuda(), n, K, along_columns=False, mode=2).toarray()
    for r in range(n):
        rows, vals = elasticnet_oracle.select_topk(D[r].astype(np.float64), K)
        ref = np.zeros(n); ref[rows] = vals
        assert np.array_equal(T[r], ref.astype(np.float32)), r
