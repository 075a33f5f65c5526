"""SLIM ElasticNet against a sparse Gram matrix (b200_slim_enet_sparse_device): the routing rule and its footprint on the
CPU; on the GPU the Gram CSR against scipy and the dense-mode Gram matrix, and the recommender forced onto the sparse path
against the dense path on the same URM."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import elasticnet_oracle
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_oracle_next_rows import ENET_CASES, enet_urm

H100_SMS = 132


def _workspace(n, n_sms):
    from recsys2019_deeplearning_evaluation_b200 import _lib
    ws = ctypes.c_int64()
    _lib.check(_lib.load().b200_slim_enet_workspace_bytes(n, n_sms, ctypes.byref(ws)))
    return int(ws.value)


# ---------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("n,n_sms,expect", [(100, 132, 0), (17066, 132, 0), (17067, 132, 132 * 3 * 17067 * 4),
                                            (100000, 132, 132 * 3 * 100000 * 4), (20000, 16, 16 * 3 * 20000 * 4)])
def test_workspace_is_the_vectors_beyond_200_kb(n, n_sms, expect):
    assert _workspace(n, n_sms) == expect


@pytest.mark.parametrize("n,topK", [(120, 20), (120, 500), (17500, 100), (100000, 100)])
def test_dense_footprint_is_the_buffer_sizes(n, topK):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_URM_COPIES, ease_urm_bytes, slim_enet_dense_bytes
    X = synth_urm(300, 120, 0.05, seed=2)
    urm = ease_urm_bytes(X)
    k = min(topK, n)
    G = coefT = 4 * n * n
    table = n * k * 4 + n * k * 4 + n * 4  # idx, val, cnt
    want = G + coefT + _workspace(n, H100_SMS) + table + EASE_URM_COPIES * urm
    assert slim_enet_dense_bytes(n, topK, H100_SMS, urm) == want


@pytest.mark.parametrize("n", [120, 17700, 100000, 150000])
def test_rule_takes_the_sparse_path_only_when_the_dense_one_does_not_fit(n):
    from recsys2019_deeplearning_evaluation_b200.recommenders import slim_enet_dense_bytes, slim_enet_sparse_for_device
    dense = slim_enet_dense_bytes(n, 100, H100_SMS, 10 ** 6)
    rule = lambda free, pos=True, nonneg=True: slim_enet_sparse_for_device(n, free, pos, nonneg, 100, H100_SMS, 10 ** 6)
    assert not rule(dense) and not rule(10 ** 13)          # fits: the dense path
    assert rule(dense - 1) and rule(0)
    for free in (0, dense - 1, dense, 10 ** 13):           # positive_only=False or a negative rating: always the dense path
        assert not rule(free, pos=False)
        assert not rule(free, nonneg=False)
        assert not rule(free, pos=False, nonneg=False)


def test_rule_figure_for_an_h100():
    """8 n^2 bytes: an 80 GB H100 (84.5 GB free) keeps the dense path to about 100 K items."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import slim_enet_sparse_for_device
    free = int(84.5e9)
    assert not slim_enet_sparse_for_device(100000, free, True, True, 100, H100_SMS)
    assert slim_enet_sparse_for_device(104000, free, True, True, 100, H100_SMS)


# ---------------------------------------------------------------------------------------------------------------- GPU


def _fit(X, sparse, monkeypatch=None, **kw):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import recommenders
    r = recommenders.SLIMElasticNetRecommender(X, verbose=False)
    if not sparse:
        r.fit(**kw)
        return r
    n = X.shape[1]
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    dense = recommenders.slim_enet_dense_bytes(n, kw.get("topK", 100), sms, recommenders.ease_urm_bytes(X))
    free, total = torch.cuda.mem_get_info()
    assert free > dense
    fit_sparse = recommenders.SLIMElasticNetRecommender._fit_sparse
    called = []

    def spy(self, *args):
        called.append(1)
        return fit_sparse(self, *args)

    with monkeypatch.context() as m:
        m.setattr(torch.cuda, "mem_get_info", lambda *a: (dense - 1, total))
        m.setattr(recommenders.SLIMElasticNetRecommender, "_fit_sparse", spy)
        r.fit(**kw)
    assert called, "the sparse path was not taken"
    return r


def _compare(a, b, label):
    """Dense path a against sparse path b: the same W_sparse pattern, the same passes per item, values within 1e-6
    relative.  Returns how many columns (items) are bit-identical."""
    A, B = a.W_sparse.tocsc(), b.W_sparse.tocsc()
    A.sort_indices(); B.sort_indices()
    assert B.dtype == np.float32 and B.shape == A.shape
    assert np.array_equal(A.indptr, B.indptr) and np.array_equal(A.indices, B.indices), label
    assert np.array_equal(a._n_iter.cpu().numpy(), b._n_iter.cpu().numpy()), label
    err = np.abs(A.data.astype(np.float64) - B.data) / np.maximum(np.abs(A.data.astype(np.float64)), 1e-30)
    assert err.size == 0 or err.max() <= 1e-6, (label, float(err.max()))
    same = sum(np.array_equal(A.data[A.indptr[c]:A.indptr[c + 1]].view(np.int32), B.data[B.indptr[c]:B.indptr[c + 1]].view(np.int32))
               for c in range(A.shape[1]))
    print("%s: %d of %d items bit-identical, max rel diff %.3g" % (label, same, A.shape[1], float(err.max()) if err.size else 0.0))
    return same


def _dense_gram(X):
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    n = X.shape[1]
    sim = Compute_Similarity_Cython(X, shrink=0, topK=n if n > 2048 else 0, normalize=False, similarity="cosine")
    G = sim.compute_dense_device(0, n).cpu().numpy()
    sim._dealloc()
    return G


@pytest.mark.gpu
@pytest.mark.parametrize("values", ["binary", "ratings"])
def test_gram_csr_matches_scipy_and_the_dense_gram(values):
    """3 000 items: three slabs.  Binary counts are exact in fp32, so the CSR equals scipy's X^T X off the diagonal; the
    values are the dense-mode Gram matrix's bits in both cases."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import gram_csr_device
    X = synth_urm(2000, 3000, 0.003, seed=11, values=values, popularity=0.8)
    n = X.shape[1]
    ptr, col, val = gram_csr_device(X)
    ptr, col, val = ptr.cpu().numpy(), col.cpu().numpy(), val.cpu().numpy()
    nnz = int(ptr[-1])
    C = sps.csr_matrix((val[:nnz], col[:nnz], ptr), shape=(n, n))
    for r in range(0, n, 97):
        assert np.all(np.diff(col[ptr[r]:ptr[r + 1]]) > 0), r  # ascending, no duplicates
    assert (C.diagonal() == 0).all() and (val[:nnz] != 0).all()
    D = _dense_gram(X)
    np.fill_diagonal(D, 0)
    Dc = sps.csr_matrix(D)
    assert np.array_equal(Dc.indptr, C.indptr) and np.array_equal(Dc.indices, C.indices)
    assert np.array_equal(Dc.data.view(np.int32), C.data.view(np.int32))
    S = (X.T @ X).astype(np.float64).tolil()
    S.setdiag(0)
    S = sps.csr_matrix(S)
    S.eliminate_zeros()
    assert np.array_equal(S.indptr, C.indptr) and np.array_equal(S.indices, C.indices)
    if values == "binary":
        assert np.array_equal(S.data, C.data.astype(np.float64))
    else:
        assert np.allclose(S.data, C.data, rtol=1e-6, atol=0)


POSITIVE_CASES = [c for c in ENET_CASES if c[3]]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(POSITIVE_CASES)))
@pytest.mark.parametrize("top", ["case", "all"])
def test_sparse_path_matches_the_dense_path_on_the_enet_cases(monkeypatch, case, top):
    """The ENET_CASES shapes with positive_only; topK from the case (below nnz) and topK = n_items (at / above nnz, where
    mode 2 drops each item's smallest weight)."""
    values, l1_ratio, alpha, positive, topK = POSITIVE_CASES[case]
    X = enet_urm(values)
    if top == "all":
        topK = X.shape[1]
    kw = dict(l1_ratio=l1_ratio, alpha=alpha, positive_only=True, topK=topK)
    a, b = _fit(X, False, **kw), _fit(X, True, monkeypatch, **kw)
    _compare(a, b, "enet case %d topK=%d" % (case, topK))


@pytest.mark.gpu
@pytest.mark.parametrize("l1_ratio", [1e-5, 0.1, 1.0])
def test_sparse_path_on_a_long_tailed_catalogue_with_cold_items_and_users(monkeypatch, l1_ratio):
    """A sparse Gram matrix (Zipf popularity), items nobody rated and users with no interaction."""
    X = sps.lil_matrix(synth_urm(3000, 2500, 0.004, seed=5, values="ratings", popularity=0.9))
    X[:, [7, 1200, 2499]] = 0
    X[[0, 10, 2999], :] = 0
    X = sps.csr_matrix(X)
    X.eliminate_zeros()
    kw = dict(l1_ratio=l1_ratio, alpha=1e-3, positive_only=True, topK=50)
    a, b = _fit(X, False, **kw), _fit(X, True, monkeypatch, **kw)
    _compare(a, b, "long tail l1_ratio=%g" % l1_ratio)
    W = b.W_sparse.tocsc()
    for c in (7, 1200, 2499):
        assert W[:, c].nnz == 0 and W.tocsr()[c].nnz == 0
    assert (b._n_iter.cpu().numpy()[[7, 1200, 2499]] == 0).all()


@pytest.mark.gpu
def test_sparse_path_max_iter_reached(monkeypatch):
    X = synth_urm(1500, 800, 0.01, seed=8, values="ratings", popularity=0.7)
    kw = dict(l1_ratio=0.05, alpha=1e-4, positive_only=True, topK=30, max_iter=3, tol=1e-9)
    a, b = _fit(X, False, **kw), _fit(X, True, monkeypatch, **kw)
    _compare(a, b, "max_iter=3")
    it = b._n_iter.cpu().numpy()
    assert (it == 3).sum() > 0.5 * (it > 0).sum()


@pytest.mark.gpu
def test_sparse_path_large_catalogue_uses_the_global_workspace(monkeypatch):
    """3 * n * 4 bytes > 200 KB (n > 17 066): the vectors live in the workspace; a few columns against the fp64 oracle."""
    n_items = 17500
    X = sps.lil_matrix(synth_urm(600, n_items, 0.004, seed=9, values="binary"))
    X[:, 100] = 0
    X = sps.csr_matrix(X)
    X.eliminate_zeros()
    kw = dict(l1_ratio=0.1, alpha=1e-3, positive_only=True, topK=10)
    a, b = _fit(X, False, **kw), _fit(X, True, monkeypatch, **kw)
    _compare(a, b, "17 500 items")
    W = b.W_sparse.tocsc()
    assert W[:, 100].nnz == 0 and W.tocsr()[100].nnz == 0
    Xd = X.toarray().astype(np.float64)
    for j in (5, 17499):
        G = Xd.T @ Xd[:, j:j + 1]
        support = np.flatnonzero(G[:, 0])
        support = support[support != j]
        Gs = Xd[:, support].T @ Xd[:, support]  # the oracle on the support: the other coordinates never act
        q = G[support, 0]
        w, _, _ = elasticnet_oracle.enet_cd_gram(Gs, q, Xd[:, j] @ Xd[:, j], 1e-3 * 0.1 * 600, 1e-3 * 0.9 * 600, True)
        full = np.zeros(n_items); full[support] = w
        rows, vals = elasticnet_oracle.select_topk(full, 10)
        ref = np.zeros(n_items); ref[rows] = vals
        got = np.asarray(W[:, j].todense()).ravel()
        assert np.abs(got - ref).max() < 2e-5, (j, float(np.abs(got - ref).max()))


@pytest.mark.gpu
def test_l1_ratio_zero(monkeypatch):
    """l1 = 0 is where the two paths differ.  On the dense path a coordinate outside the support of its item's row of X^T X
    acts as soon as its H_k, a sum of rounded terms whose exact value is 0, rounds below zero (q_k - H_k > 0 = l1); the
    sparse path never visits it.  Such a weight is a few ulps of H over d + l2, and it moves the item's other weights and
    can change its pass count.  So: every sparse-path weight lies on the support, the dense path's weights off it stay
    below 1e-6 of the item's largest, the two agree on the support to 1e-4 of the item's largest, and a few columns of
    the sparse path match the fp64 oracle (whose coordinates off the support cannot act) to 2e-5."""
    X = synth_urm(1500, 800, 0.01, seed=8, values="ratings", popularity=0.7)
    kw = dict(l1_ratio=0.0, alpha=1e-3, positive_only=True, topK=800)
    a, b = _fit(X, False, **kw), _fit(X, True, monkeypatch, **kw)
    Xd = X.toarray().astype(np.float64)
    G = Xd.T @ Xd
    np.fill_diagonal(G, 0)
    A, B = a.W_sparse.toarray().astype(np.float64), b.W_sparse.toarray().astype(np.float64)
    assert (B[G == 0] == 0).all()
    scale = np.maximum(np.abs(A).max(axis=0, keepdims=True), 1e-30)
    off = np.abs(np.where(G == 0, A, 0)) / scale
    assert off.max() <= 1e-6, float(off.max())
    on = (G != 0) & (A != 0) & (B != 0)
    rel = np.where(on, np.abs(A - B) / scale, 0)
    assert rel.max() <= 1e-4, float(rel.max())
    print("l1_ratio=0: %d dense-path weights off the support (largest %.3g of its item's largest), on the support max "
          "|dW| %.3g of the item's largest, equal passes on %d of %d items" % (
              int(((G == 0) & (A != 0)).sum()), float(off.max()), float(rel.max()),
              int((a._n_iter.cpu().numpy() == b._n_iter.cpu().numpy()).sum()), X.shape[1]))
    for j in (0, 3, 400):
        support = np.flatnonzero(G[:, j])
        Gs = Xd[:, support].T @ Xd[:, support]
        w, _, _ = elasticnet_oracle.enet_cd_gram(Gs, G[support, j], Xd[:, j] @ Xd[:, j], 0.0, 1e-3 * 1500, True)
        full = np.zeros(800); full[support] = w
        rows, vals = elasticnet_oracle.select_topk(full, 800)
        ref = np.zeros(800); ref[rows] = vals
        assert np.abs(B[:, j] - ref).max() < 2e-5, (j, float(np.abs(B[:, j] - ref).max()))


@pytest.mark.gpu
def test_sparse_gram_that_does_not_fit_raises_memory_error(monkeypatch):
    """Free memory below both paths' needs: the rule routes to the sparse path, whose CSR does not fit either."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.recommenders import SLIMElasticNetRecommender
    X = synth_urm(1500, 800, 0.01, seed=8, values="ratings", popularity=0.7)
    total = torch.cuda.mem_get_info()[1]
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1000, total))
    with pytest.raises(MemoryError, match="CSR and the solve's workspace need [0-9]+ bytes of device memory and 1000 are free"):
        SLIMElasticNetRecommender(X, verbose=False).fit(l1_ratio=0.1, alpha=1e-3, positive_only=True, topK=10)
