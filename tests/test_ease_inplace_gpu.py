"""The in-place EASE_R fit (b200_ease_inplace_device): the routing rule on the CPU; on the GPU its stages through the test
hook against fp64 numpy, the whole entry against b200_ease_from_gram_device and the fp64 restatement, and the
recommender forced onto the in-place path against the default path."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

NB = 128
GUARD = 4096  # floats past the matrix that no call may touch


def _workspace(n):
    from recsys2019_deeplearning_evaluation_b200 import _lib
    ws = ctypes.c_int64()
    _lib.check(_lib.load().b200_ease_inplace_workspace_bytes(n, ctypes.byref(ws)))
    return int(ws.value)


def _bounds(n):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_GRAM_SLAB_ROWS
    n_pad = -(-n // NB) * NB
    default = 4 * (2 * n * n + 5 * n_pad * n_pad)
    inplace = 4 * n_pad * n_pad + _workspace(n) + 4 * min(n, EASE_GRAM_SLAB_ROWS) * n
    return default, inplace


# ---------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("n,n_pad", [(127, 128), (128, 128), (129, 256)])
def test_routing_pads_to_128(n, n_pad):
    from recsys2019_deeplearning_evaluation_b200.recommenders import ease_inplace_for_device
    default, inplace = _bounds(n)
    assert default == 4 * (2 * n * n + 5 * n_pad * n_pad)
    # the workspaces are O(n_pad * NB): at this size they outweigh the n_pad^2 the default path spends beyond the buffer
    assert inplace > default
    for free in (0, inplace - 1, default - 1, default, inplace, 10 ** 12):
        assert not ease_inplace_for_device(n, free)


@pytest.mark.parametrize("n", [3000, 17700, 63000, 100000])
def test_routing_thresholds(n):
    from recsys2019_deeplearning_evaluation_b200.recommenders import ease_inplace_for_device
    default, inplace = _bounds(n)
    assert inplace < default
    assert not ease_inplace_for_device(n, default)          # fits today: the default path
    assert not ease_inplace_for_device(n, 10 ** 13)
    assert ease_inplace_for_device(n, default - 1)          # fits only in place
    assert ease_inplace_for_device(n, inplace)
    assert not ease_inplace_for_device(n, inplace - 1)      # fits neither: the default path and its out-of-memory error
    assert not ease_inplace_for_device(n, 0)


def test_routing_counts_the_urm():
    """The in-place need includes EASE_URM_COPIES CSR copies of the URM: free memory that holds the matrix, workspace and
    slab but not the URM copies keeps the default path."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_URM_COPIES, ease_inplace_for_device, ease_urm_bytes
    X = synth_urm(500, 300, 0.05, seed=2)
    assert ease_urm_bytes(X) == 4 * 501 + 8 * X.nnz
    n = 100000
    default, inplace = _bounds(n)
    urm = 10 ** 9
    need = inplace + EASE_URM_COPIES * urm
    assert need < default
    assert not ease_inplace_for_device(n, need - 1, urm)
    assert ease_inplace_for_device(n, need, urm)


@pytest.mark.parametrize("n", [1, 127, 129, 300, 511, 513, 3000, 100000, 140000])
def test_workspace_is_o_n_pad_nb(n):
    n_pad = -(-n // NB) * NB
    ws = _workspace(n)
    assert 0 < ws <= 4 * n_pad * NB * 24
    # the packed operands: K ranges of at most min(512, n_pad), so small catalogues get a tight figure
    assert ws == 4 * (2 * n_pad * NB + 4 * n_pad * min(512, n_pad) + 2 * n + NB * n) + 4


# ---------------------------------------------------------------------------------------------------------------- GPU


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))  # one item: B = [[0]] on both sides


def _spd(n, n_pad, seed):
    """A Gram-like SPD matrix of order n (cond ~ 1e2) padded with an identity block to n_pad."""
    rng = np.random.default_rng(seed)
    Y = rng.standard_normal((n, 2 * n + 8))
    A = np.eye(n_pad)
    A[:n, :n] = Y @ Y.T / Y.shape[1] + 0.05 * np.eye(n)
    return A


def _hook(op, A64, n_pad):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    buf = torch.full((n_pad * n_pad + GUARD,), 7.25, dtype=torch.float32, device="cuda")
    buf[:n_pad * n_pad] = torch.from_numpy(A64.astype(np.float32).ravel()).cuda()
    _lib.check(_lib.load().b200_ease_inplace_debug_device(op, buf.data_ptr(), n_pad, _stream()))
    out = buf.cpu().numpy()
    assert (out[n_pad * n_pad:] == 7.25).all(), "the call wrote past the matrix"
    return out[:n_pad * n_pad].reshape(n_pad, n_pad).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("n_pad", [128, 256, 384, 1024, 2048])
def test_stages_against_fp64(n_pad):
    n = n_pad - 37
    A = _spd(n, n_pad, seed=n_pad)
    L = np.linalg.cholesky(A)
    Linv = np.linalg.inv(L)
    P = np.linalg.inv(A)
    got_L = np.tril(_hook(0, A, n_pad))
    assert _rel(got_L, L) < 1e-4
    got_X = _hook(1, A, n_pad)
    assert (np.triu(got_X, 1) == 0).all()
    assert _rel(got_X, Linv) < 1e-4
    got_P = np.tril(_hook(2, A, n_pad))
    assert _rel(got_P, np.tril(P)) < 1e-4
    # the identity padding block stays identity, and nothing leaks between it and the matrix
    assert np.allclose(got_P[n:, n:], np.eye(n_pad - n), atol=1e-6, rtol=0)
    assert np.abs(got_P[n:, :n]).max() < 1e-6


@pytest.mark.gpu
def test_hook_rejects_indefinite():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    A = _spd(300, 384, seed=3)
    A[200, 200] = -1.0
    with pytest.raises(_lib.NotPositiveDefiniteError, match="not positive definite"):
        _hook(2, A, 384)


def _gram(X):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    r = EASE_R_Recommender(X, verbose=False)
    return r, r._gram_device()


def _inplace(r, G, l2):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    n = G.shape[0]
    n_pad = -(-n // NB) * NB
    buf = torch.full((n_pad * n_pad + GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    buf[:n_pad * n_pad].view(n_pad, n_pad)[:n, :n] = G  # the rest of the matrix stays NaN: the call must overwrite it
    buf[n_pad * n_pad:] = 7.25
    _, d_idx, _ = r._urm_device()
    _lib.check(_lib.load().b200_ease_inplace_device(buf.data_ptr(), n, d_idx.data_ptr(), r.URM_train.nnz, float(l2), _stream()))
    out = buf.cpu().numpy()
    assert (out[n_pad * n_pad:] == 7.25).all(), "the call wrote past the matrix"
    return out[:n * n].reshape(n, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, 2048, 3000])
@pytest.mark.parametrize("l2", [5.0, 200.0])
def test_entry_against_default_path_and_fp64(n, l2):
    import torch
    from oracle.ease_oracle import ease_B
    from recsys2019_deeplearning_evaluation_b200 import _lib
    X = synth_urm(max(400, 2 * n), n, 0.02 if n > 1 else 0.3, seed=n + int(l2), values="binary")
    r, G = _gram(X)
    _, d_idx, _ = r._urm_device()
    B_default = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(_lib.load().b200_ease_from_gram_device(G.data_ptr(), n, d_idx.data_ptr(), X.nnz, float(l2), None,
                                                      B_default.data_ptr(), _stream()))
    B = _inplace(r, G, l2)
    assert np.isfinite(B).all()  # no NaN of the uninitialised padding reached the compacted array
    assert (np.diag(B) == 0).all()
    ref = ease_B(X, l2)
    assert _rel(B, ref) < 1e-4
    assert _rel(B, B_default.cpu().numpy()) < 1e-4


@pytest.mark.gpu
def test_entry_indefinite_ratings_returns_not_spd():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    X = synth_urm(600, 200, 0.05, seed=23, values="ratings")
    G64 = np.asarray((X.T @ X).todense(), dtype=np.float64)
    G64[np.diag_indices_from(G64)] = np.diff(X.tocsc().indptr) + 50.0
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(G64)
    r, G = _gram(X)
    with pytest.raises(_lib.NotPositiveDefiniteError, match="not positive definite"):
        _inplace(r, G, 50.0)
    import torch
    torch.cuda.synchronize()  # the device is still usable
    assert float(torch.ones(4, device="cuda").sum()) == 4.0


# ------------------------------------------------------------------------------------------------ recommender level

N_REC = 3000


def _force_inplace(monkeypatch, n):
    import torch
    default, inplace = _bounds(n)
    free, total = torch.cuda.mem_get_info()
    assert free > default
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (default - 1, total))


def _fit_both(monkeypatch, X, **kw):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    a = EASE_R_Recommender(X, verbose=False)
    a.fit(verbose=False, **kw)
    with monkeypatch.context() as m:
        _force_inplace(m, X.shape[1])
        b = EASE_R_Recommender(X, verbose=False)
        b.fit(verbose=False, **kw)
    return a, b


@pytest.fixture(scope="module")
def rec_data():
    X = synth_urm(6000, N_REC, 0.01, seed=41, values="binary")
    T = synth_urm(6000, N_REC, 0.003, seed=42, values="binary")
    T = sps.csr_matrix(T - T.multiply(X))
    T.eliminate_zeros()
    return X, T


@pytest.mark.gpu
def test_recommender_inplace_dense(monkeypatch, rec_data):
    from recsys2019_deeplearning_evaluation_b200.evaluation import EvaluatorHoldout
    X, T = rec_data
    a, b = _fit_both(monkeypatch, X, topK=None, l2_norm=100.0)
    Wa, Wb = np.asarray(a.W_sparse), np.asarray(b.W_sparse)
    assert Wb.shape == (N_REC, N_REC) and (np.diag(Wb) == 0).all()
    assert _rel(Wb, Wa) < 1e-4
    assert b._d_B.shape == (N_REC, N_REC) and b._d_B.is_contiguous()
    users = np.arange(0, 6000, 97)
    sa, sb = a._compute_item_score(users), b._compute_item_score(users)
    assert _rel(sb, sa) < 1e-4
    # recommend: the in-place lists carry the default path's top scores (ties may reorder near-equal items)
    ra = a.recommend(users, cutoff=10, remove_seen_flag=True)
    rb = b.recommend(users, cutoff=10, remove_seen_flag=True)
    scale = np.abs(sa).max()
    for k, u in enumerate(users):
        assert len(ra[k]) == len(rb[k]) == 10
        assert np.abs(sa[k, rb[k]] - sa[k, ra[k]]).max() <= 1e-4 * scale
    # EvaluatorHoldout: a user whose top-10 list is the same on both paths contributes the same to every metric, so the
    # per-user means (each term in [0, 1], ARHR in [0, H_10]) may differ by at most the share of users whose list changed
    # times that range; with no changed list every metric agrees to rounding
    ev_users = np.flatnonzero(np.diff(T.indptr) > 0)
    la = a.recommend(ev_users, cutoff=10, remove_seen_flag=True)
    lb = b.recommend(ev_users, cutoff=10, remove_seen_flag=True)
    share = sum(list(x) != list(y) for x, y in zip(la, lb)) / len(ev_users)
    assert share <= 0.01, share
    ev = EvaluatorHoldout(T, [10], verbose=False)
    res_a, _ = ev.evaluateRecommender(a)
    res_b, _ = ev.evaluateRecommender(b)
    per_user = {"PRECISION": 1.0, "PRECISION_RECALL_MIN_DEN": 1.0, "RECALL": 1.0, "MAP": 1.0, "MAP_MIN_DEN": 1.0,
                "MRR": 1.0, "NDCG": 1.0, "HIT_RATE": 1.0, "ARHR_ALL_HITS": sum(1.0 / r for r in range(1, 11))}
    for metric, va in res_a[10].items():
        vb = res_b[10][metric]
        if share == 0:
            assert abs(vb - va) <= 1e-9 * max(1.0, abs(va)), metric
        elif metric in per_user:
            assert abs(vb - va) <= share * per_user[metric] + 1e-12, metric


@pytest.mark.gpu
def test_recommender_inplace_topk_and_save_load(monkeypatch, rec_data, tmp_path):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X, _ = rec_data
    a, b = _fit_both(monkeypatch, X, topK=100, l2_norm=100.0)
    assert sps.issparse(b.W_sparse) and (np.diff(b.W_sparse.tocsc().indptr) == 100).all()
    # near-equal coefficients at rank 100 may swap between two fp32 factorisations: compare tie-aware against the
    # default path's dense B -- the kept values within 1e-4 of max|B|, and every column keeps its 100 largest up to that
    dense = EASE_R_Recommender(X, verbose=False)
    dense.fit(topK=None, l2_norm=100.0, verbose=False)
    Bd = np.asarray(dense.W_sparse)
    tol = 1e-4 * np.abs(Bd).max()
    for W in (a.W_sparse.toarray(), b.W_sparse.toarray()):
        nz = W != 0
        assert np.abs(W[nz] - Bd[nz]).max() <= tol
        kth = -np.sort(-Bd, axis=0)[99]
        kept_min = np.where(nz, Bd, np.inf).min(axis=0)
        assert (kept_min >= kth - tol).all()
    users = np.arange(0, 6000, 131)
    folder = str(tmp_path) + "/"
    b.save_model(folder)
    c = EASE_R_Recommender(X, verbose=False)
    c.load_model(folder)
    assert np.allclose(c._compute_item_score(users), b._compute_item_score(users), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_recommender_inplace_indefinite_raises_memory_error(monkeypatch):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(6000, N_REC, 0.01, seed=43, values="ratings")
    l2 = 1.0
    G64 = np.asarray((X.T @ X).todense(), dtype=np.float64)
    G64[np.diag_indices_from(G64)] = np.diff(X.tocsc().indptr) + l2
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(G64)
    _force_inplace(monkeypatch, N_REC)
    r = EASE_R_Recommender(X, verbose=False)
    with pytest.raises(MemoryError, match=r"not positive definite for 3000 items.*fp64 LU inverse needs \d+ bytes.*\d+ are free"):
        r.fit(topK=None, l2_norm=l2, verbose=False)


@pytest.mark.gpu
def test_sharded_ease_keeps_the_default_path(monkeypatch, rec_data):
    """dist.make_sharded_ease: its Gram is an all-reduce every rank joins, so low free memory on a rank must not send that
    rank to the in-place path (which builds its own Gram and would skip the collective).  One rank, the collective faked."""
    import torch
    import torch.distributed as dist
    from recsys2019_deeplearning_evaluation_b200.dist import make_sharded_ease
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X, _ = rec_data
    calls = []
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    monkeypatch.setattr(dist, "all_reduce", lambda t, op=None, group=None: calls.append(t.shape))
    ref = EASE_R_Recommender(X, verbose=False)
    ref.fit(topK=None, l2_norm=100.0, verbose=False)
    _force_inplace(monkeypatch, N_REC)
    r = make_sharded_ease()(X, verbose=False)
    r.fit(topK=None, l2_norm=100.0, verbose=False)
    assert calls == [torch.Size([N_REC, N_REC])]
    assert np.array_equal(np.asarray(r.W_sparse), np.asarray(ref.W_sparse))  # the default path, bit for bit
