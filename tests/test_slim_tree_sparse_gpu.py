"""-m gpu: the row-sparse tree mode of SLIM-BPR (train_with_sparse_weights=True) at sizes where the cuts fall inside the
epoch and the structure builds span many blocks, bit for bit against the dense trainer when nothing is cut, and on a
catalogue whose dense S does not fit one GPU."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle.sgd_oracle import SLIMOracle
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_next_rows_gpu import _assert_same_cut

pytestmark = pytest.mark.gpu


def _slim():
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    return SLIM_BPR_Cython_Epoch


@pytest.mark.parametrize("mode", ["adagrad", "adam"])
def test_mid_size_tree_mode_matches_the_oracle(mode):
    """40 000 users x 8 000 items, K = 50: about 320 touches per row and epoch, so every in-epoch cut trims rows."""
    X = synth_urm(40_000, 8_000, 0.004, seed=11, values="ratings")
    kw = dict(train_with_sparse_weights=True, learning_rate=0.05, li_reg=1e-3, lj_reg=2e-3, topK=50, random_seed=5, sgd_mode=mode)
    g, o = _slim()(X, **kw), SLIMOracle(X, **kw)
    for _ in range(2):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
        S = g.get_S()
        assert sps.isspmatrix_csr(S) and S.shape == (8_000, 8_000) and S.has_sorted_indices
        assert np.diff(S.indptr).max() <= 50
        _assert_same_cut(S.toarray(), o.get_S_tree().toarray(), 50)
    g._dealloc()


def test_uncut_tree_mode_is_bit_identical_to_the_dense_trainer():
    """topK=False never cuts, so the row-sparse cells carry exactly the dense non-symmetric recursion (Adam powers included,
    across the segment launches)."""
    import torch
    X = synth_urm(60_000, 30_000, 0.0015, seed=4, values="ratings")
    kw = dict(learning_rate=0.01, topK=False, symmetric=False, random_seed=9, sgd_mode="adam", li_reg=1e-3, lj_reg=1e-3)
    tree, dense = _slim()(X, train_with_sparse_weights=True, **kw), _slim()(X, train_with_sparse_weights=False, **kw)
    n = X.shape[1]
    for _ in range(2):
        tree.epochIteration_Cython()
        dense.epochIteration_Cython()
    a = torch.empty((n, n), dtype=torch.float32, device="cuda")
    b = torch.empty((n, n), dtype=torch.float32, device="cuda")
    from recsys2019_deeplearning_evaluation_b200 import _lib
    _lib.check(tree._lib.b200_slim_get_S_dense(tree._h, None, a.data_ptr()))
    _lib.check(dense._lib.b200_slim_get_S_dense(dense._h, None, b.data_ptr()))
    assert int((a != 0).sum()) > 1_000_000
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    tree._dealloc()
    dense._dealloc()


def _touched_keys(X, u, i, j):
    """row * n + col of every cell an epoch's samples touched: row i gains profile(u) minus i, row j gains profile(u)."""
    n = X.shape[1]
    lens = np.diff(X.indptr)[u]
    starts = X.indptr[u]
    pos = np.repeat(starts - np.cumsum(lens) + lens, lens) + np.arange(lens.sum())
    cols = X.indices[pos].astype(np.int64)
    ri = np.repeat(i.astype(np.int64), lens)
    rj = np.repeat(j.astype(np.int64), lens)
    keys = np.concatenate([(ri * n + cols)[cols != ri], rj * n + cols])
    return np.unique(keys)


def test_catalogue_the_dense_layout_cannot_hold():
    """200 000 x 200 000 items: the dense S alone would be 160 GB."""
    n, K = 200_000, 200
    X = synth_urm(200_000, n, 0.0005, seed=2, values="ratings")
    g = _slim()(X, train_with_sparse_weights=True, learning_rate=1e-3, topK=K, random_seed=3, sgd_mode="adagrad")
    g.epochIteration_Cython()
    S = g.get_S()
    assert sps.isspmatrix_csr(S) and S.shape == (n, n) and S.has_sorted_indices and S.nnz > 0
    per_row = np.diff(S.indptr)
    assert per_row.max() <= K
    assert np.isfinite(S.data).all()
    rows = np.repeat(np.arange(n, dtype=np.int64), per_row)
    assert not (rows == S.indices).any()
    stored = rows * n + S.indices.astype(np.int64)
    touched = _touched_keys(X, *g.get_samples())
    assert np.isin(stored, touched).all()
    t_rows = touched // n
    t_per_row = np.bincount(t_rows, minlength=n)
    short = t_per_row < K  # never cut: exactly the touched cells, all non-zero
    assert short.sum() > n // 2
    assert np.array_equal(per_row[short], t_per_row[short])
    assert np.array_equal(stored[short[rows]], touched[short[t_rows]])
    assert (S.data != 0).all()
    g._dealloc()

    from recsys2019_deeplearning_evaluation_b200.recommenders import SLIM_BPR_Cython
    r = SLIM_BPR_Cython(X, verbose=False)
    r.fit(epochs=1, topK=K, train_with_sparse_weights=None, random_seed=3, learning_rate=1e-3)
    assert r.train_with_sparse_weights is True
    W = r.W_sparse
    assert W.shape == (n, n) and W.nnz > 0 and np.diff(W.tocsr().indptr).max() <= K
    recs = r.recommend(np.arange(4), cutoff=10)
    assert len(recs) == 4 and all(len(x) == 10 for x in recs)
    for u, x in enumerate(recs):
        assert not np.isin(x, X.indices[X.indptr[u]:X.indptr[u + 1]]).any()
