"""P3alpha / RP3beta item-item matrices on the K1 kernel (GraphBased/P3alphaRecommender.py:34-144,
GraphBased/RP3betaRecommender.py:31-154).

The reference computes, per 200-row block, `Piu[block] * Pui` densified, scales by `degree` (RP3beta), zeroes the
diagonal, keeps the topK of every ROW with a full argsort, optionally L1-normalises the rows and finally applies a
COLUMN top-K (`similarityMatrixTopK`).  Here the product + row top-K is one pass of the similarity kernel in its
"scale" formula (SURVEY.md Appendix A closed form): value[i, j] = (1/deg_i)^alpha * deg_j^-beta * sum_{u in item i}
(r_uj / rowsum_u)^alpha; the column top-K runs on the device over the CSC of the result.  A topK above the kernel's
candidate buffer (2048) takes the kernel's dense mode instead, one slab of targets at a time, with a dense row top-K.
Element-wise preparation of Pui (O(nnz)) stays on the host like the reference's sklearn `normalize`/`power` calls.
Ties in either top-K resolve to the ascending index (the reference's argsort order is unspecified, App. A quirk 11).
"""
import ctypes

import numpy as np
import scipy.sparse as sps

from . import _lib
from .similarity import _as_csr_f32, topk_table_to_csr

SELECT_MAX_K = 2048  # the largest topK the window kernel's candidate buffer selects
DENSE_SLAB_CELLS = 1 << 26  # topK > SELECT_MAX_K: cells of one dense slab of targets (256 MB of fp32)


def _row_l1_normalize(M):
    """sklearn.preprocessing.normalize(M, norm='l1', axis=1) for CSR (P3alphaRecommender.py:54,137-138)."""
    M = sps.csr_matrix(M, dtype=np.float32, copy=True)
    s = np.asarray(np.abs(M).sum(axis=1), dtype=np.float64).ravel()
    s[s == 0] = 1.0
    M.data = (M.data / np.repeat(s, np.diff(M.indptr))).astype(np.float32)
    return M


def sparse_column_topk(W, k):
    """similarityMatrixTopK (Base/Recommender_utils.py:55-122) for a scipy sparse matrix, on the device.  A duplicated
    entry stands for the sum of its values, as everywhere in scipy."""
    import torch
    lib = _lib.load()
    Wc = sps.csc_matrix(W, dtype=np.float32)
    if not Wc.has_canonical_format:  # the kernel reads every stored entry as a cell of its own; W stays untouched
        Wc = Wc.copy()
        Wc.sum_duplicates()
    n = Wc.shape[1]
    k = int(min(k, n))
    dev = torch.device("cuda", torch.cuda.current_device())
    ptr = torch.from_numpy(Wc.indptr.astype(np.int32)).to(dev)
    rows = torch.from_numpy(Wc.indices.astype(np.int32)).to(dev)
    vals = torch.from_numpy(Wc.data.astype(np.float32)).to(dev)
    idx = torch.empty((n, k), dtype=torch.int32, device=dev)
    val = torch.empty((n, k), dtype=torch.float32, device=dev)
    cnt = torch.empty((n,), dtype=torch.int32, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200_sparse_topk_device(n, ptr.data_ptr(), rows.data_ptr(), vals.data_ptr(), k, 0, idx.data_ptr(),
                                           val.data_ptr(), cnt.data_ptr(), st))
    return topk_table_to_csr(n, k, idx, val, cnt)  # line = column, idx = row: entries stay in place


def scaled_inputs(URM_train, alpha=1.0, beta=0.0, min_rating=0, implicit=False):
    """The arguments of b200_sim_create_scaled for p3_similarity: Pui (CSR float32, the row-normalised URM to the power
    alpha), A (float32, (1/deg_i)^alpha, 0 for an item nobody rated) and B (float32, deg_j^-beta, or 1 when beta == 0)."""
    URM = _as_csr_f32(URM_train).copy()
    if min_rating > 0:  # P3alphaRecommender.py:47-51
        URM.data[URM.data < min_rating] = 0
        URM.eliminate_zeros()
        if implicit:
            URM.data = np.ones(URM.data.size, dtype=np.float32)
    n_items = URM.shape[1]
    Pui = _row_l1_normalize(URM)
    deg = np.bincount(URM.indices, minlength=n_items).astype(np.float64)  # X_bool.sum(axis=1)
    A = np.zeros(n_items, np.float64)
    A[deg > 0] = 1.0 / deg[deg > 0]  # the constant entries of row i of Piu
    B = np.ones(n_items, np.float64)
    if beta != 0.0:  # RP3betaRecommender.py:59-65
        B = np.zeros(n_items, np.float64)
        B[deg > 0] = np.power(deg[deg > 0], -float(beta))
    if alpha != 1.0:  # :64-66
        Pui = Pui.power(alpha).astype(np.float32)
        A = np.power(A, alpha)
    return Pui, np.ascontiguousarray(A, np.float32), np.ascontiguousarray(B, np.float32)


def p3_similarity(URM_train, topK=100, alpha=1.0, beta=0.0, min_rating=0, implicit=False, normalize_similarity=False):
    """Returns W_sparse (CSR float32, row i = item i's outgoing weights) as the reference's fit() leaves it.
    beta=0 -> P3alpha, beta>0 -> RP3beta.  The recommender classes apply `min_rating` / `implicit` to their own
    URM_train first (the reference mutates it, P3alphaRecommender.py:47-51); the arguments here serve direct callers and
    work on a private copy."""
    import torch
    lib = _lib.load()
    Pui, A32, B32 = scaled_inputs(URM_train, alpha, beta, min_rating, implicit)
    n_users, n_items = Pui.shape
    K = int(min(topK, n_items)) if topK is not False else n_items
    dense = K > SELECT_MAX_K
    h = ctypes.c_void_p()
    indptr, indices, data = (np.ascontiguousarray(Pui.indptr, np.int32), np.ascontiguousarray(Pui.indices, np.int32),
                             np.ascontiguousarray(Pui.data, np.float32))
    _lib.check(lib.b200_sim_create_scaled(ctypes.byref(h), n_users, n_items, Pui.nnz, _lib.ptr(indptr), _lib.ptr(indices),
                                          _lib.ptr(data), _lib.ptr(A32), _lib.ptr(B32), 1 if dense else K, None))
    try:
        dev = torch.device("cuda", torch.cuda.current_device())
        idx = torch.empty((n_items, K), dtype=torch.int32, device=dev)
        val = torch.empty((n_items, K), dtype=torch.float32, device=dev)
        cnt = torch.empty((n_items,), dtype=torch.int32, device=dev)
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if dense:
            # topK beyond the window kernel's selection buffer: the dense mode of the same handle (the scaled values, the
            # diagonal 0) one slab of targets at a time, then per target the K largest over all cells, zeros dropped
            # (b200_dense_topk mode 1: zeros outrank negatives, ties to the ascending index, as in the window kernel)
            rows = max(1, min(n_items, DENSE_SLAB_CELLS // n_items))
            S = torch.empty((rows, n_items), dtype=torch.float32, device=dev)
            for lo in range(0, n_items, rows):
                m = min(rows, n_items - lo)
                _lib.check(lib.b200_sim_compute_dense_device(h, lo, lo + m, S.data_ptr(), st))
                _lib.check(lib.b200_dense_topk_rect_device(S.data_ptr(), m, n_items, n_items, 1, 0, K, 1, idx[lo].data_ptr(),
                                                           val[lo].data_ptr(), cnt[lo:].data_ptr(), st))
            del S
        else:
            _lib.check(lib.b200_sim_compute_device(h, 0, n_items, idx.data_ptr(), val.data_ptr(), cnt.data_ptr(), st))
        T = topk_table_to_csr(n_items, K, idx, val, cnt)  # T[j, i] = value of target i towards j
    finally:
        lib.b200_sim_destroy(h)
    # row i of W = target i: the CSR arrays of T read as CSC
    W = sps.csc_matrix((T.data, T.indices, T.indptr), shape=(n_items, n_items)).tocsr()
    if normalize_similarity:  # :137-138
        W = _row_l1_normalize(W)
    if topK is not False:  # :141-142
        W = sparse_column_topk(W, topK)
    return sps.csr_matrix(W, dtype=np.float32)
