"""Host-side mirror of SLIM_BPR/Cython/SLIM_BPR_Cython_Epoch.pyx:60-480 backed by libb200rec.so, plus the GPU
equivalent of Base/Recommender_utils.py:55-122 `similarityMatrixTopK` for dense device matrices.

Same constructor signature as pyx:88-94, `epochIteration_Cython()`, `get_S()`, `_dealloc()`.  Extra keywords:
sampler="glibc"|"philox", hogwild=False (see mf_epoch.py).  S is dense fp32 in HBM, optionally symmetric (lower-triangular
addressing).  `train_with_sparse_weights=True` (Sparse_Matrix_Tree_CSR, pyx:579-1031) is the tree mode with its semantics --
which cells exist, the periodic rebalance_tree(TopK) during the epoch (pyx:318-319), the in-place top-K of get_S
(pyx:762-763) -- and its memory footprint: S is row-sparse on the device, its size follows the cells the rows hold, so a
catalogue whose dense S does not fit trains on one GPU."""
import ctypes

import numpy as np
import scipy.sparse as sps

from . import _lib

_MODE = {"sgd": 0, "adagrad": 1, "rmsprop": 2, "adam": 3}
_SAMPLER = {"glibc": 0, "philox": 1}


def dense_topk_to_sparse(d_matrix, n, k, along_columns, mode):
    """Top-k along rows/columns of a dense [n, n] fp32 CUDA tensor -> scipy CSR float32 with the same orientation
    as the input (entry (r, c) keeps its place)."""
    import torch
    from .similarity import topk_table_to_csr
    lib = _lib.load()
    k = int(min(k, n))
    dev = d_matrix.device
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    val = torch.empty((n, k), dtype=torch.float32, device=dev)
    cnt = torch.empty((n,), dtype=torch.int32, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200_dense_topk_device(d_matrix.data_ptr(), n, k, int(along_columns), int(mode), idx.data_ptr(),
                                          val.data_ptr(), cnt.data_ptr(), st))
    T = topk_table_to_csr(n, k, idx, val, cnt)  # T[idx, line] = val
    if along_columns:
        return T  # line = column, idx = row: already in place
    # line = row, idx = column: T is the transpose; its CSR arrays read as CSC are the matrix itself
    return sps.csc_matrix((T.data, T.indices, T.indptr), shape=(n, n)).tocsr()


def similarityMatrixTopK(item_weights, k=100, verbose=False):
    """GPU version of Base/Recommender_utils.py:55-122 for a dense ndarray / CUDA tensor: per column keep the k largest
    non-zero values; returns CSC float32 like the reference (ties resolve to the ascending row index)."""
    import torch
    if sps.issparse(item_weights):
        item_weights = item_weights.toarray()
    t = item_weights if isinstance(item_weights, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(item_weights, np.float32))
    assert t.shape[0] == t.shape[1], "selectTopK: ItemWeights is not a square matrix"
    t = t.to(device="cuda", dtype=torch.float32).contiguous()
    return dense_topk_to_sparse(t, t.shape[0], k, along_columns=True, mode=0).tocsc()


def sparse_weights_for_device(train_with_sparse_weights, n_items, free_bytes, symmetric=True):
    """The `train_with_sparse_weights` an epoch object gets.  True / False are kept; None (SLIM_BPR_Cython.py:85-103, where
    the reference picks the tree mode when the dense S would not fit in RAM) is the device counterpart of that rule, with a
    different threshold: the dense mode needs S (n_items^2 fp32, allocated in full even when symmetric) plus get_S's
    n_items^2 fp32 buffer, so the tree mode is picked when 8 * n_items^2 bytes exceed the free device memory."""
    if train_with_sparse_weights is not None:
        return bool(train_with_sparse_weights)
    return 8 * int(n_items) * int(n_items) > int(free_bytes)


class SLIM_BPR_Cython_Epoch:
    def __init__(self, URM_mask, train_with_sparse_weights=False, final_model_sparse_weights=True, learning_rate=0.01,
                 li_reg=0.0, lj_reg=0.0, topK=150, symmetric=True, verbose=False, random_seed=None, sgd_mode="adam",
                 gamma=0.995, beta_1=0.9, beta_2=0.999, sampler="glibc", hogwild=False):
        self._h = ctypes.c_void_p()
        self._lib = _lib.load()
        if sgd_mode not in _MODE:
            raise ValueError("SLIM_BPR_Cython_Epoch: sgd_mode '{}' not recognized".format(sgd_mode))
        X = sps.csr_matrix(URM_mask, dtype=np.float32)
        if not X.has_sorted_indices:
            X = X.sorted_indices()
        self.n_users, self.n_items = X.shape
        self.topK = min(topK, self.n_items) if topK is not False else False  # pyx:105
        self.train_with_sparse_weights = bool(train_with_sparse_weights)
        if self.train_with_sparse_weights:
            symmetric = False  # pyx:111-112
            if hogwild:
                raise ValueError("SLIM_BPR_Cython_Epoch: train_with_sparse_weights is a sequential mode (hogwild=False)")
        self.symmetric = bool(symmetric)
        self.final_model_sparse_weights = final_model_sparse_weights
        indptr = np.ascontiguousarray(X.indptr, np.int32)
        indices = np.ascontiguousarray(X.indices, np.int32)
        _lib.check(self._lib.b200_slim_create(
            ctypes.byref(self._h), self.n_users, self.n_items, X.nnz, _lib.ptr(indptr), _lib.ptr(indices), float(learning_rate),
            float(li_reg), float(lj_reg), int(self.symmetric), _MODE[sgd_mode], float(gamma), float(beta_1), float(beta_2),
            int(random_seed is not None), int(random_seed) & 0xFFFFFFFF if random_seed is not None else 0,
            _SAMPLER[sampler], int(bool(hogwild))))
        if self.train_with_sparse_weights:
            _lib.check(self._lib.b200_slim_enable_tree(self._h, int(self.topK) if self.topK else 0))

    def epochIteration_Cython(self):
        import torch
        _lib.check(self._lib.b200_slim_epoch(self._h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def last_epoch_ms(self):
        ms = ctypes.c_float()
        _lib.check(self._lib.b200_slim_last_epoch_ms(self._h, ctypes.byref(ms)))
        return float(ms.value)

    def get_samples(self):
        u = np.empty(self.n_users, np.int32); i = np.empty(self.n_users, np.int32); j = np.empty(self.n_users, np.int32)
        _lib.check(self._lib.b200_slim_get_samples(self._h, _lib.ptr(u), _lib.ptr(i), _lib.ptr(j)))
        return u, i, j

    def get_S_dense(self):
        """Full [n_items, n_items] float32 ndarray (diagonal zeroed, symmetric mode mirrored)."""
        out = np.empty((self.n_items, self.n_items), np.float32)
        _lib.check(self._lib.b200_slim_get_S_dense(self._h, _lib.ptr(out), None))
        return out

    def tree_cells(self):
        """Tree mode: the cells the row-sparse structure holds now (12 bytes of device memory each)."""
        c = ctypes.c_int64()
        _lib.check(self._lib.b200_slim_tree_cells(self._h, ctypes.byref(c)))
        return int(c.value)

    def get_S(self):
        """pyx:340-388: diagonal zeroed, then per ROW top-K -- symmetric: K largest over all cells, zeros dropped
        (Triangular_Matrix.get_scipy_csr, pyx:1335-1415); dense: similarityMatrixTopK(S.T).T (pyx:371,386)."""
        import torch
        n = self.n_items
        if self.train_with_sparse_weights:
            # pyx:349-350 touches the diagonal cells, get_scipy_csr(TopK) (pyx:737-778) cuts every row that holds more than
            # TopK cells IN PLACE and emits the non-zero cells that are left; topK=False emits them all.  No n x n buffer.
            _lib.check(self._lib.b200_slim_tree_prune(self._h, 1, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
            nnz = ctypes.c_int64()
            _lib.check(self._lib.b200_slim_tree_csr_nnz(self._h, ctypes.byref(nnz)))
            indptr = np.empty(n + 1, np.int64)
            indices = np.empty(max(nnz.value, 1), np.int32)
            data = np.empty(max(nnz.value, 1), np.float32)
            _lib.check(self._lib.b200_slim_tree_csr(self._h, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data)))
            nz = nnz.value
            return sps.csr_matrix((data[:nz].astype(np.float64), indices[:nz], indptr), shape=(n, n))
        d = torch.empty((n, n), dtype=torch.float32, device="cuda")
        _lib.check(self._lib.b200_slim_get_S_dense(self._h, None, d.data_ptr()))
        if self.topK is False:
            if self.symmetric or self.final_model_sparse_weights:
                return sps.csr_matrix(d.cpu().numpy())
            return d.cpu().numpy().astype(np.float64)
        if not self.symmetric and not self.final_model_sparse_weights:
            return d.cpu().numpy().astype(np.float64)
        return dense_topk_to_sparse(d, n, self.topK, along_columns=False, mode=1 if self.symmetric else 0)

    def _dealloc(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.b200_slim_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self._dealloc()
        except Exception:
            pass
