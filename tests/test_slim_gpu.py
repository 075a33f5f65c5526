"""-m gpu: SLIM-BPR epochs and the dense top-K kernels against the C oracle / numpy restatements."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle.sgd_oracle import SLIMOracle
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 2e-6


def _cls():
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    return SLIM_BPR_Cython_Epoch


def _oracle_S(o):
    S = o.S_full()
    np.fill_diagonal(S, 0)
    return S


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("mode", ["sgd", "adagrad", "adam", "rmsprop"])
def test_sequential_parity_on_the_glibc_stream(symmetric, mode):
    X = synth_urm(300, 120, 0.08, seed=3)
    kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=2e-3, topK=120, symmetric=symmetric, random_seed=7, sgd_mode=mode)
    g, o = _cls()(X, **kw), SLIMOracle(X, **kw)
    for _ in range(3):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
    S = g.get_S_dense().astype(np.float64)
    R = _oracle_S(o)
    assert np.allclose(S, R, rtol=RTOL, atol=ATOL), float(np.abs(S - R).max())
    assert (np.diag(S) == 0).all()
    if symmetric:
        assert np.array_equal(S, S.T)


def test_get_S_topk_semantics():
    """Row top-K: symmetric = K largest over all cells with zeros dropped (pyx:1335-1415); dense = K largest non-zero
    (similarityMatrixTopK(S.T).T, pyx:371,386).  1 200 items: more rows than the selection kernel's grid of 8 CTAs per SM."""
    for X in (synth_urm(400, 150, 0.06, seed=5), synth_urm(2500, 1200, 0.02, seed=5)):
        n = X.shape[1]
        for symmetric in (True, False):
            kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=1e-3, topK=10, symmetric=symmetric, random_seed=1, sgd_mode="adagrad")
            g = _cls()(X, **kw)
            for _ in range(4):
                g.epochIteration_Cython()
            D = g.get_S_dense().astype(np.float64)
            W = g.get_S()
            assert sps.issparse(W) and W.shape == (n, n)
            W = W.toarray()
            for r in range(n):
                row = D[r]
                if symmetric:
                    order = np.lexsort((np.arange(n), -row))[:10]
                    keep = order[row[order] != 0]
                else:
                    nz = np.flatnonzero(row)
                    keep = nz[np.lexsort((nz, -row[nz]))][:10]
                ref = np.zeros(n)
                ref[keep] = row[keep]
                assert np.allclose(W[r], ref, rtol=1e-6, atol=0), (n, r)


def test_similarityMatrixTopK_gpu_matches_recipe():
    """Base/Recommender_utils_Test.py:18-50: nnz per column and dense == sparse; plus the negatives-survive rule.
    1 200 columns: more lines than the selection kernel's grid of 8 CTAs per SM."""
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import similarityMatrixTopK
    rng = np.random.default_rng(0)
    for n in (200, 1200):
        k = 20
        D = rng.standard_normal((n, n)).astype(np.float32)
        D[rng.random((n, n)) < 0.7] = 0
        D[:, 3] = 0
        D[:5, 7] = [-1, -2, -3, 0.5, 0]; D[5:, 7] = 0   # 1 positive, 3 negatives: all four survive for k >= 4
        W = similarityMatrixTopK(D, k=k)
        assert sps.isspmatrix_csc(W) and W.dtype == np.float32
        Wd = W.toarray()
        for c in range(n):
            col = D[:, c]
            nz = np.flatnonzero(col)
            keep = nz[np.lexsort((nz, -col[nz]))][:k]
            ref = np.zeros(n, np.float32)
            ref[keep] = col[keep]
            assert np.array_equal(Wd[:, c], ref), (n, c)
        assert (np.diff(W.indptr) <= k).all() and W[:, 3].nnz == 0 and W[:, 7].nnz == 4


def test_philox_stream_and_hogwild():
    """Philox samples are valid BPR triples; replaying them through the oracle reproduces the sequential kernel;
    hogwild moves S the same way."""
    X = synth_urm(1500, 300, 0.05, seed=9, popularity=0.7)
    kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=1e-3, topK=300, symmetric=False, random_seed=4, sgd_mode="sgd")
    s = _cls()(X, sampler="philox", **kw)
    hw = _cls()(X, sampler="philox", hogwild=True, **kw)
    streams = []
    for _ in range(2):
        s.epochIteration_Cython()
        hw.epochIteration_Cython()
        streams.append(s.get_samples())
        assert np.array_equal(streams[-1][0], hw.get_samples()[0])
    su, si, sj = (np.concatenate([t[k] for t in streams]) for k in range(3))
    dense = X.toarray()
    assert (dense[su, si] != 0).all() and (dense[su, sj] == 0).all()
    o = SLIMOracle(X, samples=(su, si, sj), **kw)
    for _ in range(2):
        o.epochIteration_Cython()
    S, R = s.get_S_dense().astype(np.float64), _oracle_S(o)
    assert np.allclose(S, R, rtol=RTOL, atol=ATOL)
    H = hw.get_S_dense().astype(np.float64)
    cos = float((H.ravel() @ R.ravel()) / (np.linalg.norm(H) * np.linalg.norm(R)))
    assert cos > 0.98 and abs(np.linalg.norm(H) / np.linalg.norm(R) - 1) < 0.1, cos


def test_sparse_tree_mode_forces_the_full_matrix():
    """train_with_sparse_weights=True (tests/test_next_rows_gpu.py has its parity tests): symmetric is switched off like
    pyx:111-112 does, and the throughput mode is refused."""
    X = synth_urm(50, 20, 0.2)
    g = _cls()(X, train_with_sparse_weights=True, symmetric=True, random_seed=1)
    assert g.symmetric is False and g.train_with_sparse_weights is True
    with pytest.raises(ValueError):
        _cls()(X, train_with_sparse_weights=True, hogwild=True, sampler="philox", random_seed=1)


# ---------------------------------------------------------------------------------------------------------------------
# column-sharded S (dist.ShardedSLIM_BPR, SURVEY.md 8(e) K3).  Several shards live on one GPU here and the test adds their
# partial sums itself (what the all-reduce does between ranks); tools/mgpu_slim_check.py is the NCCL run.

def _sharded(X, ranges, batch_size, **kw):
    from recsys2019_deeplearning_evaluation_b200.dist import ShardedSLIM_BPR
    return [ShardedSLIM_BPR(X, batch_size=batch_size, col_range=r, world_rank=(1, 0), **kw) for r in ranges]


def _sharded_epoch(shards, batch_size):
    n = shards[0].n_users
    for first in range(0, n, batch_size):
        m = min(batch_size, n - first)
        x = None
        for s in shards:
            part = s.partial(first, m)
            x = part.clone() if x is None else x + part
        for s in shards:
            s.apply(first, m, x)


@pytest.mark.parametrize("mode", ["sgd", "adagrad", "adam", "rmsprop"])
def test_column_sharded_batch_1_is_the_reference_recursion(mode):
    """batch_size = 1: partial sums over two column shards + their sum + per-shard updates = the sequential recursion of
    SLIM_BPR_Cython_Epoch.pyx:231-312 on the same (Philox) stream, replayed through the C oracle."""
    import torch
    X = synth_urm(300, 120, 0.08, seed=3)
    kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=2e-3, topK=120, random_seed=7, sgd_mode=mode)
    shards = _sharded(X, [(0, 50), (50, 120)], 1, **kw)
    streams = []
    for _ in range(2):
        _sharded_epoch(shards, 1)
        u = np.empty(300, np.int32); i = np.empty(300, np.int32); j = np.empty(300, np.int32)
        from recsys2019_deeplearning_evaluation_b200 import _lib
        _lib.check(_lib.load().b200_slim_get_samples(shards[0]._h, _lib.ptr(u), _lib.ptr(i), _lib.ptr(j)))
        u2 = np.empty(300, np.int32); i2 = np.empty(300, np.int32); j2 = np.empty(300, np.int32)
        _lib.check(_lib.load().b200_slim_get_samples(shards[1]._h, _lib.ptr(u2), _lib.ptr(i2), _lib.ptr(j2)))
        assert np.array_equal(u, u2) and np.array_equal(i, i2) and np.array_equal(j, j2)  # every shard draws the same stream
        streams.append((u, i, j))
    su, si, sj = (np.concatenate([t[k] for t in streams]) for k in range(3))
    o = SLIMOracle(X, samples=(su, si, sj), symmetric=False, **kw)
    for _ in range(2):
        o.epochIteration_Cython()
    S = torch.cat([s.slab() for s in shards], dim=1).cpu().numpy().astype(np.float64)
    R = _oracle_S(o)
    assert np.abs(R).max() > 0
    assert np.allclose(S, R, rtol=RTOL, atol=ATOL), float(np.abs(S - R).max())


def test_column_sharded_batches_and_row_topk():
    """Batches of 64: three shards against one shard holding every column (same batches, same stream), and the merged
    per-row top-K of the shards against numpy on the assembled matrix."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.dist import ShardedSLIM_BPR
    X = synth_urm(900, 260, 0.05, seed=9, popularity=0.7)
    kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=1e-3, topK=12, random_seed=4, sgd_mode="adagrad")
    three = _sharded(X, [(0, 100), (100, 101), (101, 260)], 64, **kw)
    one = _sharded(X, [(0, 260)], 64, **kw)
    for _ in range(3):
        _sharded_epoch(three, 64)
        _sharded_epoch(one, 64)
    S3 = torch.cat([s.slab() for s in three], dim=1).cpu().numpy()
    S1 = one[0].slab().cpu().numpy()
    assert np.abs(S1).max() > 0 and (np.diag(S1) == 0).all()
    assert np.allclose(S3, S1, rtol=1e-4, atol=2e-5), float(np.abs(S3 - S1).max())  # fp32 atomics: the order of a batch's updates
    W = ShardedSLIM_BPR.merge_row_topk([s.local_row_topk() for s in three], 260, 12)
    assert sps.issparse(W) and W.shape == (260, 260)
    W = W.toarray()
    for r in range(260):
        row = S3[r]
        nz = np.flatnonzero(row)
        keep = nz[np.lexsort((nz, -row[nz]))][:12]
        ref = np.zeros(260, np.float32)
        ref[keep] = row[keep]
        assert np.array_equal(W[r], ref), r
    with pytest.raises(NotImplementedError):
        ShardedSLIM_BPR(X, symmetric=True, random_seed=1, world_rank=(1, 0))
    with pytest.raises(ValueError):
        ShardedSLIM_BPR(X, random_seed=None, world_rank=(1, 0))
