"""Host-side mirror of the reference's similarity boundary, backed by libb200rec.so (sm_90a).

`Compute_Similarity_Cython` keeps the constructor / `compute_similarity(start_col, end_col)` signature, argument
meaning and error behaviour of Base/Similarity/Cython/Compute_Similarity_Cython.pyx:52-611 (reference paths are
relative to the reference checkout); `Compute_Similarity` mirrors the dispatcher
Base/Similarity/Compute_Similarity.py:30-126 -- except that nothing here ever falls back to a CPU
implementation (Compute_Similarity.py:108-110 does, silently; SURVEY.md Appendix A quirk 5).

Declared semantic choices (DESIGN.md "K1 semantics"):
  * top-K ties resolve to the ascending neighbour index (the reference's order is numpy-introselect over an
    insertion-ordered scratch array, pyx:536-548, which no parallel implementation can reproduce);
  * signed similarities follow Compute_Similarity_Python.py:335-345 (zeros outrank negatives, zeros dropped)
    instead of the stale-slot behaviour of pyx:531-557;
  * accumulation is fp32 on the device (fp64 in pyx:57); values agree within 1e-4 relative.
"""
import ctypes

import numpy as np
import scipy.sparse as sps

from . import _lib

_KIND = {"cosine": 0, "adjusted": 1, "asymmetric": 2, "pearson": 3, "jaccard": 4, "tanimoto": 4, "dice": 5,
         "tversky": 6}


def _as_csr_f32(dataMatrix):
    """What check_matrix(..., 'csr') + .copy() give the reference (pyx:154,200), plus sorted indices (the
    windowed accumulator needs sorted rows; BaseRecommender-built URMs already are)."""
    if (sps.isspmatrix_csr(dataMatrix) and dataMatrix.dtype == np.float32 and dataMatrix.indices.dtype == np.int32
            and dataMatrix.indptr.dtype == np.int32 and dataMatrix.has_sorted_indices):
        # already in the layout the C ABI takes: hand the caller's arrays over as they are (they are only read -- the
        # reference's defensive .copy(), pyx:154, protects its in-place transforms, which run on the device here).
        # scipy caches has_sorted_indices on the object, so repeated fits on one URM pay the O(nnz) check once.
        return dataMatrix
    if isinstance(dataMatrix, np.ndarray):
        X = sps.csr_matrix(dataMatrix, dtype=np.float32)
        X.eliminate_zeros()
    else:
        X = sps.csr_matrix(dataMatrix, dtype=np.float32)
    if not X.has_sorted_indices:
        X = X.sorted_indices()
    if X.indices.dtype != np.int32 or X.indptr.dtype != np.int32:
        if X.nnz >= 2 ** 31 - 1:
            raise ValueError("Compute_Similarity_Cython: more than 2^31 stored values are not supported")
        X = sps.csr_matrix((X.data, X.indices.astype(np.int32), X.indptr.astype(np.int32)), shape=X.shape)
    return X


class TopKTable:
    """Device-resident result of a column range: idx/val [n, K], cnt [n] as torch CUDA tensors."""

    def __init__(self, idx, val, cnt, start_col, end_col, K):
        self.idx, self.val, self.cnt = idx, val, cnt
        self.start_col, self.end_col, self.K = start_col, end_col, K


class Compute_Similarity_Cython:
    """Drop-in for the Cython class of the same name (pyx:52).  Holds a device handle; `compute_similarity`
    returns the scipy CSR float32 matrix pyx:603-611 returns."""

    def __init__(self, dataMatrix, topK=100, shrink=0, normalize=True, asymmetric_alpha=0.5, tversky_alpha=1.0,
                 tversky_beta=1.0, similarity="cosine", row_weights=None):
        self._h = ctypes.c_void_p()
        self._lib = _lib.load()
        self.n_rows, self.n_columns = dataMatrix.shape
        if similarity not in _KIND:
            # same text as pyx:141-144
            raise ValueError("Cosine_Similarity: value for parameter 'mode' not recognized."
                             " Allowed values are: 'cosine', 'pearson', 'adjusted', 'asymmetric', 'jaccard', 'tanimoto',"
                             "dice, tversky."
                             " Passed value was '{}'".format(similarity))
        if row_weights is not None and dataMatrix.shape[0] != len(row_weights):
            # pyx:188-190
            raise ValueError("Cosine_Similarity: provided row_weights and dataMatrix have different number of rows."
                             "Row_weights has {} rows, dataMatrix has {}.".format(len(row_weights), dataMatrix.shape[0]))
        self.similarity = similarity
        self.TopK = min(topK, self.n_columns)  # pyx:147
        self.shrink = int(shrink)  # `cdef int shrink`, pyx:65: a float shrink is truncated
        self.normalize = bool(normalize)
        # TopK == 0 (dense ndarray out, pyx:510-513) and TopK beyond the selection kernel's buffer go through the dense
        # mode of the kernel; the handle is then created with a token topK
        self._dense_mode = self.TopK == 0 or self.TopK > 2048
        X = _as_csr_f32(dataMatrix)
        rw = None if row_weights is None else np.ascontiguousarray(row_weights, dtype=np.float32)
        self._keep = (X, rw)  # host arrays stay alive for the duration of the (synchronous) create call
        _lib.check(self._lib.b200_sim_create(
            ctypes.byref(self._h), X.shape[0], X.shape[1], X.nnz, _lib.ptr(X.indptr), _lib.ptr(X.indices),
            _lib.ptr(X.data), _KIND[similarity], 1 if self._dense_mode else int(self.TopK), float(self.shrink), int(self.normalize),
            float(asymmetric_alpha), float(tversky_alpha), float(tversky_beta), _lib.ptr(rw), None))
        self._keep = None
        k = ctypes.c_int32(); nw = ctypes.c_int32(); wc = ctypes.c_int32(); bp = ctypes.c_int32(); sd = ctypes.c_int32()
        _lib.check(self._lib.b200_sim_info(self._h, ctypes.byref(k), ctypes.byref(nw), ctypes.byref(wc),
                                           ctypes.byref(bp), ctypes.byref(sd)))
        self.K, self.n_windows, self.window_cells = int(k.value), int(nw.value), int(wc.value)
        self.binary_path, self.signed_data = bool(bp.value), bool(sd.value)

    # ------------------------------------------------------------------ reference API
    def _col_range(self, start_col, end_col):
        lo, hi = 0, self.n_columns  # pyx:444-454 (end_col == n_columns is ignored there; same result here)
        if start_col is not None and 0 < start_col < self.n_columns:
            lo = start_col
        if end_col is not None and lo < end_col < self.n_columns:
            hi = end_col
        return lo, hi

    def compute_similarity(self, start_col=None, end_col=None):
        """pyx:413-611: W_sparse (n_columns x n_columns) CSR float32 holding columns [start_col, end_col)."""
        lo, hi = self._col_range(start_col, end_col)
        if self._dense_mode:
            return self._compute_dense(lo, hi)
        tab = self.compute_topk_device(lo, hi)
        return self.table_to_csr(tab)

    def compute_dense_device(self, lo, hi):
        """[hi - lo, n_columns] float32 CUDA tensor: out[target - lo, neighbour] = W[neighbour, target]."""
        import torch
        out = torch.empty((hi - lo, self.n_columns), dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))
        _lib.check(self._lib.b200_sim_compute_dense_device(self._h, lo, hi, out.data_ptr(),
                                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out

    def _compute_dense(self, lo, hi):
        import torch
        n = self.n_columns
        D = self.compute_dense_device(lo, hi)
        if lo != 0 or hi != n:
            full = torch.zeros((n, n), dtype=torch.float32, device=D.device)
            full[lo:hi] = D
            D = full
        if self.TopK == 0:  # pyx:597-599: dense float64 ndarray W_dense[neighbour, target]
            return D.t().contiguous().cpu().numpy().astype(np.float64)
        if self.TopK >= n:  # every non-zero similarity (EASE_R asks for topK = n_items)
            return sps.csr_matrix(D.t().contiguous().cpu().numpy())
        from .slim_bpr_epoch import dense_topk_to_sparse
        # rows of D are targets: per target keep the TopK largest over all cells, zeros dropped; transpose into W[j, i]
        return sps.csr_matrix(dense_topk_to_sparse(D, n, self.TopK, along_columns=False, mode=1).T)

    # ------------------------------------------------------------------ device-level API (multi-GPU, bench)
    def compute_topk_device(self, lo, hi, stream=None, out=None):
        """Top-K rows of the columns [lo, hi) as a device-resident TopKTable; `out` (a table of the same range from an earlier
        call) is overwritten in place instead of allocating a new one."""
        import torch
        n = hi - lo
        if out is not None:
            assert out.start_col == lo and out.end_col == hi and out.K == self.K, "out= must come from the same column range"
            idx, val, cnt = out.idx, out.val, out.cnt
        else:
            dev = torch.device("cuda", torch.cuda.current_device())
            idx = torch.empty((max(n, 1), self.K), dtype=torch.int32, device=dev)
            val = torch.empty((max(n, 1), self.K), dtype=torch.float32, device=dev)
            cnt = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream
        _lib.check(self._lib.b200_sim_compute_device(self._h, lo, hi, idx.data_ptr(), val.data_ptr(), cnt.data_ptr(),
                                                     ctypes.c_void_p(st)))
        return TopKTable(idx, val, cnt, lo, hi, self.K)

    def table_to_csr(self, tab):
        """Assemble the canonical CSR on the device (stable sort by neighbour row) and copy it out."""
        import torch
        n = self.n_columns
        if tab.start_col == 0 and tab.end_col == n:
            idx, val, cnt = tab.idx, tab.val, tab.cnt
        else:  # partial range: other columns are empty, as pyx:467 leaves them
            dev = tab.idx.device
            idx = torch.full((n, self.K), -1, dtype=torch.int32, device=dev)
            val = torch.zeros((n, self.K), dtype=torch.float32, device=dev)
            cnt = torch.zeros((n,), dtype=torch.int32, device=dev)
            m = tab.end_col - tab.start_col
            if m > 0:
                idx[tab.start_col:tab.end_col] = tab.idx[:m]
                val[tab.start_col:tab.end_col] = tab.val[:m]
                cnt[tab.start_col:tab.end_col] = tab.cnt[:m]
        return topk_table_to_csr(n, self.K, idx, val, cnt)

    def last_kernel_ms(self):
        ms = ctypes.c_float()
        _lib.check(self._lib.b200_sim_last_kernel_ms(self._h, ctypes.byref(ms)))
        return float(ms.value)

    def gathered_entries(self, lo=0, hi=None):
        hi = self.n_columns if hi is None else hi
        out = ctypes.c_int64()
        _lib.check(self._lib.b200_sim_work(self._h, lo, hi, ctypes.byref(out)))
        return int(out.value)

    def column_work(self):
        """Per-column gathered-entry counts (int64[n_columns]) -- weights for the multi-GPU partition."""
        out = np.empty(self.n_columns, np.int64)
        _lib.check(self._lib.b200_sim_col_work(self._h, _lib.ptr(out)))
        return out

    def _dealloc(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.b200_sim_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self._dealloc()
        except Exception:
            pass


class Compute_Similarity_Python(Compute_Similarity_Cython):
    """Drop-in for Base/Similarity/Compute_Similarity_Python.py:15-370 (SURVEY.md 8 a5), the reference's dense-block numpy
    implementation of the same similarities: identical constructor, `compute_similarity(start_col, end_col, block_size)`.
    Its semantics for signed similarities (zeros outrank negatives, :335-345) are the ones the CUDA kernel implements, so
    this is the same device path; `block_size` (the width of the reference's dense blocks) has no meaning here."""

    def compute_similarity(self, start_col=None, end_col=None, block_size=100):
        return super(Compute_Similarity_Python, self).compute_similarity(start_col=start_col, end_col=end_col)


_EUCLID_MODE = {"exp": 0, "lin": 1, "log": 2}


class Compute_Similarity_Euclidean(Compute_Similarity_Cython):
    """Drop-in for Base/Similarity/Compute_Similarity_Euclidean.py:14-223 (same constructor and
    `compute_similarity(start_col, end_col, block_size)` signature, same error text).  Every column has a finite
    distance to the target, so the top-K runs over ALL columns (co-rated or not), the target itself excluded
    (:149,:171); see include/b200rec.h b200_sim_create_euclidean for the formula.

    Declared deviations: `row_weights` raises NotImplementedError (the reference multiplies an n_columns vector by
    the n_rows weights, :152 -- only defined for square matrices); top-K ties resolve to the ascending neighbour
    index (binary data ties massively here: all non-co-rated columns of equal norm are equidistant)."""

    def __init__(self, dataMatrix, topK=100, shrink=0, normalize=False, normalize_avg_row=False,
                 similarity_from_distance_mode="lin", row_weights=None, **args):
        self._h = ctypes.c_void_p()
        self._lib = _lib.load()
        self.n_rows, self.n_columns = dataMatrix.shape
        self.TopK = min(topK, self.n_columns)  # :26
        self.shrink = shrink  # a Python number here (:22), not a C int
        self.normalize = bool(normalize)
        self.normalize_avg_row = bool(normalize_avg_row)
        self.similarity = "euclidean"
        if similarity_from_distance_mode not in _EUCLID_MODE:
            # same text as :44-46
            raise ValueError("Compute_Similarity_Euclidean: value for argument 'mode' not recognized."
                             " Allowed values are: 'exp', 'lin', 'log'."
                             " Passed value was '{}'".format(similarity_from_distance_mode))
        if row_weights is not None:
            if dataMatrix.shape[0] != len(row_weights):
                # :54-55
                raise ValueError("Compute_Similarity_Euclidean: provided row_weights and dataMatrix have different number of rows."
                                 "row_weights has {} rows, dataMatrix has {}.".format(len(row_weights), dataMatrix.shape[0]))
            raise NotImplementedError("Compute_Similarity_Euclidean: row_weights are not supported on the CUDA path")
        if self.TopK < 1 or self.TopK > 2048:
            raise ValueError("Compute_Similarity_Euclidean: topK must be in [1, 2048] on the CUDA path, got {}".format(topK))
        self._dense_mode = False
        X = _as_csr_f32(dataMatrix)
        self._keep = X
        _lib.check(self._lib.b200_sim_create_euclidean(
            ctypes.byref(self._h), X.shape[0], X.shape[1], X.nnz, _lib.ptr(X.indptr), _lib.ptr(X.indices),
            _lib.ptr(X.data), int(self.TopK), float(shrink), int(self.normalize), int(self.normalize_avg_row),
            _EUCLID_MODE[similarity_from_distance_mode], None))
        self._keep = None
        k = ctypes.c_int32(); nw = ctypes.c_int32(); wc = ctypes.c_int32(); bp = ctypes.c_int32(); sd = ctypes.c_int32()
        _lib.check(self._lib.b200_sim_info(self._h, ctypes.byref(k), ctypes.byref(nw), ctypes.byref(wc),
                                           ctypes.byref(bp), ctypes.byref(sd)))
        self.K, self.n_windows, self.window_cells = int(k.value), int(nw.value), int(wc.value)
        self.binary_path, self.signed_data = bool(bp.value), bool(sd.value)

    def compute_similarity(self, start_col=None, end_col=None, block_size=100):
        """:75-223; block_size (the reference's dense block width) has no meaning here and is ignored."""
        lo, hi = self._col_range(start_col, end_col)
        return self.table_to_csr(self.compute_topk_device(lo, hi))


def _pinned_empty(n, dtype):
    """numpy array of n elements backed by page-locked memory (the torch tensor that owns it stays referenced by the
    array); pageable memory if pinning fails."""
    import torch
    try:
        t = torch.empty(max(int(n), 1), dtype=torch.int32 if dtype == np.int32 else torch.float32, pin_memory=True)
    except RuntimeError:
        return np.empty(int(n), dtype)
    return t.numpy()[:int(n)]


def topk_table_to_csr(n_cols, K, idx, val, cnt):
    """[n_cols, K] device top-K table -> scipy CSR float32 (row = neighbour j, column = target), sorted indices."""
    import torch
    lib = _lib.load()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    nnz = ctypes.c_int64()
    _lib.check(lib.b200_topk_table_to_csr_count(n_cols, K, cnt.data_ptr(), ctypes.byref(nnz), st))
    nnz = int(nnz.value)
    # The three result arrays live in page-locked host memory (torch's caching host allocator: blocks are reused once a
    # previous result is garbage-collected), so the device->host copies are DMA transfers at PCIe speed; copying 320 MB
    # into fresh pageable numpy arrays costs ~0.4 s of page faults and staging at C5, 4x the kernel.
    indptr, indices, data = _pinned_empty(n_cols + 1, np.int32), _pinned_empty(nnz, np.int32), _pinned_empty(nnz, np.float32)
    _lib.check(lib.b200_topk_table_to_csr_fill(n_cols, K, idx.data_ptr(), val.data_ptr(), cnt.data_ptr(), nnz,
                                               _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), st))
    W = sps.csr_matrix((data, indices, indptr), shape=(n_cols, n_cols), dtype=np.float32)
    W.has_sorted_indices = True
    return W


class Compute_Similarity:
    """Mirror of Base/Similarity/Compute_Similarity.py:30-126: validates, then always uses the CUDA path."""

    def __init__(self, dataMatrix, use_implementation="density", similarity=None, **args):
        assert np.all(np.isfinite(dataMatrix.data)), \
            "Compute_Similarity: Data matrix contains {} non finite values".format(
                np.sum(np.logical_not(np.isfinite(dataMatrix.data))))  # Compute_Similarity.py:44
        if use_implementation not in ("density", "cython", "python"):
            raise ValueError("Compute_Similarity: value for argument 'use_implementation' not recognized")
        if similarity == "euclidean":
            # Compute_Similarity.py:52-58: the euclidean class takes the matrix as is (no 1-feature assertion)
            self.dense = False
            self.compute_similarity_object = Compute_Similarity_Euclidean(dataMatrix, **args)
            return
        assert not (dataMatrix.shape[0] == 1 and dataMatrix.nnz == dataMatrix.shape[1]), \
            "Compute_Similarity: data has only 1 feature (shape: {}) with values in all columns," \
            " cosine and set-based similarities are not able to discriminate 1-dimensional dense data," \
            " use Euclidean similarity instead.".format(dataMatrix.shape)  # Compute_Similarity.py:65
        if similarity is not None:
            args["similarity"] = similarity
        # Compute_Similarity.py:71-113: "density" picks python for ndarrays / density > 0.5, cython otherwise; both names
        # are the same device path here, the flag is kept for callers that read it
        self.dense = isinstance(dataMatrix, np.ndarray) or (
            use_implementation == "density" and sps.issparse(dataMatrix) and dataMatrix.nnz / max(1, dataMatrix.shape[0] * dataMatrix.shape[1]) > 0.5)
        cls = Compute_Similarity_Python if (use_implementation == "python" or self.dense) else Compute_Similarity_Cython
        self.compute_similarity_object = cls(dataMatrix, **args)

    def compute_similarity(self, **args):
        return self.compute_similarity_object.compute_similarity(**args)
