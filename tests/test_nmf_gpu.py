"""NMFRecommender (csrc/nmf.cu) against scikit-learn (oracle/nmf_oracle.py).  Host cases: the random init, argument errors and
the oracle itself.  -m gpu: the SpMM and Gram building blocks against fp64 numpy, solves of k iterations from the same init
against sklearn's float64 solvers, full fits with their iteration counts, and the recommender-level calls."""
import ctypes
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.nmf_oracle import nmf_reference, solve_from
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm

gpu = pytest.mark.gpu
SOLVER_LOSS = [("multiplicative_update", "frobenius"), ("multiplicative_update", "kullback-leibler"),
               ("coordinate_descent", "frobenius")]


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


def _small_urm():
    """Ratings with empty user rows (0..4) and empty item columns (0..2)."""
    X = synth_urm(300, 120, 0.05, seed=5, values="ratings").tolil()
    X[:5, :] = 0
    X[:, :3] = 0
    X = sps.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    return X


# ---- host ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 7, None])
def test_random_init_is_sklearns(seed):
    from sklearn.decomposition._nmf import _initialize_nmf
    from recsys2019_deeplearning_evaluation_b200.recommenders import nmf_random_init
    X = synth_urm(200, 90, 0.05, seed=1, values="ratings")
    for f in (1, 13):
        np.random.seed(123)
        W, H = nmf_random_init(X, f, seed)
        np.random.seed(123)
        W0, H0 = _initialize_nmf(X, f, "random", random_state=seed)
        assert W.dtype == W0.dtype == np.float32 and H.dtype == H0.dtype == np.float32
        assert np.array_equal(W, W0) and np.array_equal(H, H0)


def test_argument_errors_match_the_reference():
    from recsys2019_deeplearning_evaluation_b200.recommenders import NMFRecommender
    r = NMFRecommender(synth_urm(50, 40, 0.1, seed=2), verbose=False)
    with pytest.raises(AssertionError, match="NMFRecommender: l1_ratio must be between 0 and 1, provided value was 1.5"):
        r.fit(l1_ratio=1.5)
    with pytest.raises(ValueError) as e:
        r.fit(solver="als")
    assert str(e.value) == ("Value for 'solver' not recognized. Acceptable values are dict_keys(['multiplicative_update', "
                            "'coordinate_descent']), provided was 'als'")
    with pytest.raises(ValueError) as e:
        r.fit(init_type="nndsvd")
    assert str(e.value) == "Value for 'init_type' not recognized. Acceptable values are ['random', 'nndsvda'], provided was 'nndsvd'"
    with pytest.raises(ValueError) as e:
        r.fit(beta_loss="itakura-saito")
    assert str(e.value) == ("Value for 'beta_loss' not recognized. Acceptable values are ['frobenius', 'kullback-leibler'], "
                            "provided was 'itakura-saito'")
    with pytest.raises(ValueError) as e:
        r.fit(solver="coordinate_descent", beta_loss="kullback-leibler")
    assert str(e.value) == "Invalid beta_loss parameter: solver 'cd' does not handle beta_loss = 'kullback-leibler'"
    # the same text as scikit-learn's own check
    from sklearn.decomposition import NMF
    with pytest.raises(ValueError) as e2:
        NMF(n_components=2, init="random", solver="cd", beta_loss="kullback-leibler").fit(r.URM_train)
    assert str(e2.value) == str(e.value)


def test_nndsvda_is_refused():
    from recsys2019_deeplearning_evaluation_b200.recommenders import NMFRecommender
    r = NMFRecommender(synth_urm(50, 40, 0.1, seed=2), verbose=False)
    with pytest.raises(NotImplementedError, match=r"init_type='nndsvda' is not on the CUDA path \(it needs a truncated SVD"):
        r.fit(init_type="nndsvda")


@pytest.mark.parametrize("solver,beta_loss", SOLVER_LOSS)
def test_oracle_is_fit_then_transform(solver, beta_loss):
    from sklearn.decomposition import NMF
    from sklearn.exceptions import ConvergenceWarning
    X = synth_urm(120, 60, 0.08, seed=3)
    W, V, n_fit, n_tr = nmf_reference(X, 6, solver=solver, beta_loss=beta_loss, random_seed=4)
    m = NMF(n_components=6, init="random", solver={"multiplicative_update": "mu", "coordinate_descent": "cd"}[solver],
            beta_loss=beta_loss, random_state=4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        m.fit(X)
        W1 = m.transform(X)
    assert np.array_equal(W, W1) and np.array_equal(V, m.components_.T) and n_fit == m.n_iter_
    assert 1 <= n_tr <= 200


# ---- device: the building blocks -------------------------------------------------------------------------------------
def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@gpu
@pytest.mark.parametrize("f", [1, 7, 33, 100, 350])
def test_spmm_and_gram_match_fp64(f):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    lib = _lib.load()
    X = _small_urm()
    M = np.random.default_rng(f).random((X.shape[1], f)).astype(np.float32)
    ptr, idx, val = _dev(X.indptr.astype(np.int32)), _dev(X.indices.astype(np.int32)), _dev(X.data.astype(np.float32))
    out = torch.empty((X.shape[0], f), dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_nmf_debug_device(0, X.shape[0], f, ptr.data_ptr(), idx.data_ptr(), val.data_ptr(), _dev(M).data_ptr(),
                                         out.data_ptr(), _stream()))
    ref = X.astype(np.float64) @ M.astype(np.float64)
    got = out.cpu().numpy()
    assert np.all(got[:5] == 0)  # empty rows
    assert np.allclose(got, ref, rtol=2e-7, atol=0)
    # Gram of a tall matrix (more rows than one split) with zero rows
    T = np.random.default_rng(f + 1).random((5000, f)).astype(np.float32)
    T[100:300] = 0
    G = torch.empty((f, f), dtype=torch.float64, device="cuda")
    _lib.check(lib.b200_nmf_debug_device(1, T.shape[0], f, None, None, None, _dev(T).data_ptr(), G.data_ptr(), _stream()))
    Gref = T.astype(np.float64).T @ T.astype(np.float64)
    assert np.allclose(G.cpu().numpy(), Gref, rtol=1e-12, atol=0)


def _solve(X, W, Ht, solver, beta_loss, update_h, max_iter, tol):
    """b200_nmf_solve_device on float32 copies; returns (W, Ht, n_iter)."""
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    X = sps.csr_matrix(X, dtype=np.float32)
    Xt = sps.csr_matrix(X.T, dtype=np.float32)
    Xt.sort_indices()
    d = [_dev(a) for a in (X.indptr.astype(np.int32), X.indices.astype(np.int32), X.data, Xt.indptr.astype(np.int32),
                           Xt.indices.astype(np.int32), Xt.data)]
    dW, dHt = _dev(np.asarray(W, np.float32)), _dev(np.asarray(Ht, np.float32))
    n_iter, last = ctypes.c_int32(), ctypes.c_double()
    _lib.check(_lib.load().b200_nmf_solve_device(
        {"mu": 0, "cd": 1}[solver], {"frobenius": 0, "kullback-leibler": 1}[beta_loss], int(update_h), X.shape[0], X.shape[1],
        dW.shape[1], *[t.data_ptr() for t in d], dW.data_ptr(), dHt.data_ptr(), max_iter, float(tol), ctypes.byref(n_iter),
        ctypes.byref(last), _stream()))
    torch.cuda.synchronize()
    return dW.cpu().numpy(), dHt.cpu().numpy(), n_iter.value


@gpu
@pytest.mark.parametrize("solver,beta_loss", [("mu", "frobenius"), ("mu", "kullback-leibler"), ("cd", "frobenius")])
@pytest.mark.parametrize("k", [1, 10, 37])
def test_k_iterations_match_sklearn_fp64(solver, beta_loss, k):
    from recsys2019_deeplearning_evaluation_b200.recommenders import nmf_random_init
    X = _small_urm()
    f = 16
    W0, H0 = nmf_random_init(X, f, 3)
    # fit: W and H alternate
    W, Ht, n = _solve(X, W0, H0.T, solver, beta_loss, True, k, 0.0)
    Wr, Hr, nr = solve_from(X, W0, H0, solver, beta_loss, k, 0.0, True)
    assert n == nr == k
    assert _rel(W, Wr) <= 1e-5 and _rel(Ht, Hr.T) <= 1e-5, (_rel(W, Wr), _rel(Ht, Hr.T))
    assert np.all(W[:5] == 0) and np.all(Ht[:3] == 0)  # empty users / items end at zero
    # transform: H fixed, W from full(avg) (mu) or zeros (cd)
    Wt0 = np.full_like(W0, np.sqrt(X.mean() / f)) if solver == "mu" else np.zeros_like(W0)
    W, Ht2, n = _solve(X, Wt0, Hr.T, solver, beta_loss, False, k, 0.0)
    Wr, _, nr = solve_from(X, Wt0, Hr.astype(np.float32), solver, beta_loss, k, 0.0, False)
    assert n == nr == k
    assert np.array_equal(Ht2, Hr.T.astype(np.float32))
    assert _rel(W, Wr) <= 1e-5, _rel(W, Wr)


@gpu
@pytest.mark.parametrize("solver,beta_loss", [("mu", "frobenius"), ("mu", "kullback-leibler"), ("cd", "frobenius")])
@pytest.mark.parametrize("n_users,n_items,f,density", [(2000, 1050, 100, 0.02), (20000, 16890, 32, 0.002),
                                                       (100000, 16880, 1, 0.0005)])
def test_shapes_where_the_item_side_takes_more_splits(solver, beta_loss, n_users, n_items, f, density):
    """The fp64 split reductions (Grams, column sums) pick their split count per row count, and the smaller side can take
    more splits than the larger one (rows per split go up in steps of 32); both factors' reductions run here."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import nmf_random_init
    X = synth_urm(n_users, n_items, density, seed=9, values="ratings")
    W0, H0 = nmf_random_init(X, f, 2)
    W, Ht, n = _solve(X, W0, H0.T, solver, beta_loss, True, 2, 0.0)
    Wr, Hr, nr = solve_from(X, W0, H0, solver, beta_loss, 2, 0.0, True)
    assert n == nr == 2
    assert _rel(W, Wr) <= 1e-5 and _rel(Ht, Hr.T) <= 1e-5, (_rel(W, Wr), _rel(Ht, Hr.T))


@gpu
def test_cd_sweep_with_a_zero_component():
    """HHt[t, t] == 0 (component t of H all zero) leaves W[:, t] as it was in the W step; empty users stay at 0."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import nmf_random_init
    X = _small_urm()
    W0, H0 = nmf_random_init(X, 9, 11)
    H0[4] = 0
    W0[:5] = 0
    W, Ht, _ = _solve(X, W0, H0.T, "cd", "frobenius", True, 1, 0.0)
    Wr, Hr, _ = solve_from(X, W0, H0, "cd", "frobenius", 1, 0.0, True)
    assert np.array_equal(W[:, 4], W0[:, 4])
    assert np.all(W[:5] == 0)
    assert _rel(W, Wr) <= 1e-5 and _rel(Ht, Hr.T) <= 1e-5


# ---- device: whole fits --------------------------------------------------------------------------------------------
def _fit(X, f, solver, beta_loss, seed):
    from recsys2019_deeplearning_evaluation_b200.recommenders import NMFRecommender
    r = NMFRecommender(X, verbose=False)
    r.fit(num_factors=f, solver=solver, beta_loss=beta_loss, random_seed=seed)
    return r


# sklearn's own float32 run differs from its float64 run on this case by at most 5.0e-6 (mu, Frobenius), 5.1e-6 (cd) and
# 1.4e-3 (mu, KL: the KL iteration amplifies rounding); the bars are 1e-4, and 5e-3 for KL.
BARS = {"frobenius": 1e-4, "kullback-leibler": 5e-3}


@gpu
@pytest.mark.parametrize("solver,beta_loss", SOLVER_LOSS)
def test_full_fit_matches_sklearn(solver, beta_loss):
    X = synth_urm(3000, 800, 0.02, seed=42)
    r = _fit(X, 32, solver, beta_loss, 7)
    W, V, n_fit, n_tr = nmf_reference(X, 32, solver=solver, beta_loss=beta_loss, random_seed=7, dtype=np.float64)
    assert r.USER_factors.dtype == np.float32 and r.ITEM_factors.dtype == np.float32
    assert (r.n_iter_, r.n_iter_transform_) == (n_fit, n_tr)
    bar = BARS[beta_loss]
    S, Sr = r.USER_factors.astype(np.float64) @ r.ITEM_factors.T, W @ V.T
    assert _rel(r.ITEM_factors, V) <= bar and _rel(r.USER_factors, W) <= bar and _rel(S, Sr) <= bar, (
        _rel(r.ITEM_factors, V), _rel(r.USER_factors, W), _rel(S, Sr))
    # top-10 lists, tie-aware: every recommended item scores (in the float64 run) within the bar of the 10th best unseen item
    users = np.arange(0, 3000, 7)
    rec = r.recommend(users, cutoff=10)
    tol = bar * np.abs(Sr).max()
    for u, items in zip(users, rec):
        s = Sr[u].copy()
        s[X[u].indices] = -np.inf
        assert s[items].min() >= np.sort(s)[-10] - tol


@gpu
def test_full_fit_iteration_counts_on_ratings():
    X = synth_urm(700, 300, 0.05, seed=8, values="ratings")
    for solver, beta_loss in SOLVER_LOSS:
        r = _fit(X, 12, solver, beta_loss, 5)
        _, _, n_fit, n_tr = nmf_reference(X, 12, solver=solver, beta_loss=beta_loss, random_seed=5, dtype=np.float64)
        assert (r.n_iter_, r.n_iter_transform_) == (n_fit, n_tr), (solver, beta_loss)


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
    from recsys2019_deeplearning_evaluation_b200.recommenders import NMFRecommender
    train = synth_urm(800, 500, 0.04, seed=31, values="ratings")
    test = synth_urm(800, 500, 0.006, seed=32, values="ratings")
    r = _fit(train, 16, "multiplicative_update", "frobenius", 3)
    W, V, _, _ = nmf_reference(train, 16, random_seed=3, dtype=np.float64)
    o = NMFRecommender(train, verbose=False)
    o.USER_factors, o.ITEM_factors = W.astype(np.float32), V.astype(np.float32)
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
    # save / load round trip
    r.save_model(str(tmp_path) + os.sep, "nmf")
    r2 = NMFRecommender(train, verbose=False)
    r2.load_model(str(tmp_path) + os.sep, "nmf")
    assert np.array_equal(r2.USER_factors, r.USER_factors) and np.array_equal(r2.ITEM_factors, r.ITEM_factors)
    assert np.array_equal(r2.recommend(users[:50], cutoff=10), r.recommend(users[:50], cutoff=10))


@gpu
def test_c3_shape_fit_is_finite():
    X = synth_config("C3")
    r = _fit(X, 100, "multiplicative_update", "frobenius", 1)
    assert r.USER_factors.shape == (X.shape[0], 100) and r.ITEM_factors.shape == (X.shape[1], 100)
    assert np.all(np.isfinite(r.USER_factors)) and np.all(np.isfinite(r.ITEM_factors))
    assert np.all(r.USER_factors >= 0) and 1 <= r.n_iter_ <= 200
