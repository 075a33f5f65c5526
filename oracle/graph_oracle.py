"""fp64 numpy restatement of P3alpha / RP3beta (TEST INFRASTRUCTURE).  Follows GraphBased/P3alphaRecommender.py:47-144
and GraphBased/RP3betaRecommender.py:47-154 step by step (normalize -> power -> Piu*Pui -> degree -> diagonal ->
row top-K -> optional row normalise -> column top-K), with the deterministic tie rule "larger value, then ascending
index" where the reference's argsort order is unspecified.  Pinned against the reference's own classes by
tests/golden/graph_golden.npz (tests/test_oracle_graph.py).  p3_similarity_sparse restates the same steps on sparse
matrices for catalogues whose dense n x n matrix does not fit; the same test file pins it to p3_similarity."""
import numpy as np
import scipy.sparse as sps


def _row_norm(M):
    M = sps.csr_matrix(M, dtype=np.float64, copy=True)
    s = np.asarray(np.abs(M).sum(axis=1)).ravel()
    s[s == 0] = 1.0
    M.data = M.data / np.repeat(s, np.diff(M.indptr))
    return M


def p3_dense_rows(URM, alpha=1.0, beta=0.0, min_rating=0, implicit=False):
    """Dense (n_items, n_items) fp64 matrix BEFORE any top-K: row i = item i."""
    URM = sps.csr_matrix(URM, dtype=np.float32, copy=True)
    if min_rating > 0:
        URM.data[URM.data < min_rating] = 0
        URM.eliminate_zeros()
        if implicit:
            URM.data = np.ones(URM.data.size, dtype=np.float32)
    Pui = _row_norm(URM)
    Xb = sps.csr_matrix(URM.T, copy=True)
    Xb.data = np.ones(Xb.data.size)
    deg = np.asarray(Xb.sum(axis=1)).ravel()
    Piu = _row_norm(Xb)
    if alpha != 1.0:
        Pui, Piu = Pui.power(alpha), Piu.power(alpha)
    D = np.asarray((Piu @ Pui).todense())
    if beta != 0.0:
        degree = np.zeros(URM.shape[1])
        degree[deg != 0] = np.power(deg[deg != 0], -beta)
        D = D * degree[None, :]
    np.fill_diagonal(D, 0.0)
    return D


def p3_sparse_rows(URM, alpha=1.0, beta=0.0, min_rating=0, implicit=False, rows=None):
    """p3_dense_rows as a CSR fp64 matrix of its non-zero cells (sorted indices, the diagonal and every zero dropped);
    only the items `rows` (an index array: row r of the result is item rows[r]) when given."""
    URM = sps.csr_matrix(URM, dtype=np.float32, copy=True)
    if min_rating > 0:
        URM.data[URM.data < min_rating] = 0
        URM.eliminate_zeros()
        if implicit:
            URM.data = np.ones(URM.data.size, dtype=np.float32)
    Pui = _row_norm(URM)
    Xb = sps.csr_matrix(URM.T, copy=True)
    Xb.data = np.ones(Xb.data.size)
    deg = np.asarray(Xb.sum(axis=1)).ravel()
    Piu = _row_norm(Xb)
    if alpha != 1.0:
        Pui, Piu = Pui.power(alpha), Piu.power(alpha)
    P = sps.csr_matrix((Piu if rows is None else Piu[np.asarray(rows)]) @ Pui)
    if beta != 0.0:
        degree = np.zeros(URM.shape[1])
        degree[deg != 0] = np.power(deg[deg != 0], -beta)
        P = sps.csr_matrix(P @ sps.diags(degree))
    P = sps.coo_matrix(P)
    keep = (P.col != (P.row if rows is None else np.asarray(rows)[P.row])) & (P.data != 0)
    P = sps.csr_matrix((P.data[keep], (P.row[keep], P.col[keep])), shape=P.shape)
    P.sort_indices()
    return P


def _line_order(line, other, val):
    """Permutation sorting the cells by line, then value descending, then ascending index along the line; and the rank of
    every cell within its line in that order."""
    order = np.argsort(other, kind="stable")  # three stable sorts: radix sorts for the integer keys
    order = order[np.argsort(-val[order], kind="stable")]
    order = order[np.argsort(line[order], kind="stable")]
    start = np.searchsorted(line[order], line[order], side="left")
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order)) - start
    return order, rank


def sparse_row_topk(P, k):
    """Per row of the sparse P (n columns), the k largest over ALL n cells (implicit zeros included, ties to the ascending
    column), zeros then dropped: p3_similarity's row loop.  A row's negatives only survive when its positives and its
    zeros do not fill k slots."""
    P = sps.coo_matrix(P)
    n = P.shape[1]
    _, rank = _line_order(P.row, P.col, P.data)
    npos = np.bincount(P.row[P.data > 0], minlength=P.shape[0])
    nneg = np.bincount(P.row[P.data < 0], minlength=P.shape[0])
    nzero = n - npos - nneg
    r = P.row
    keep = np.where(P.data > 0, rank < k, rank - npos[r] < np.maximum(0, k - npos[r] - nzero[r]))
    W = sps.csr_matrix((P.data[keep], (P.row[keep], P.col[keep])), shape=P.shape)
    W.sort_indices()
    return W


def sparse_column_topk(W, k):
    """p3_similarity's column loop: per column the k largest of the stored non-zero values, ties to the ascending row."""
    W = sps.coo_matrix(W)
    nz = W.data != 0
    rows, cols, vals = W.row[nz], W.col[nz], W.data[nz]
    _, rank = _line_order(cols, rows, vals)
    keep = rank < k
    out = sps.csr_matrix((vals[keep], (rows[keep], cols[keep])), shape=W.shape)
    out.sort_indices()
    return out


def p3_similarity_sparse(URM, topK=100, alpha=1.0, beta=0.0, min_rating=0, implicit=False, normalize_similarity=False):
    """p3_similarity step by step on sparse fp64 matrices, for catalogues whose n x n dense matrix does not fit."""
    P = p3_sparse_rows(URM, alpha, beta, min_rating, implicit)
    n = P.shape[0]
    W = sparse_row_topk(P, min(topK, n) if topK is not False else n)
    if normalize_similarity:
        W = _row_norm(W)
    if topK is not False:
        W = sparse_column_topk(W, min(topK, n))
    return sps.csr_matrix(W, dtype=np.float32)


def p3_similarity(URM, topK=100, alpha=1.0, beta=0.0, min_rating=0, implicit=False, normalize_similarity=False):
    D = p3_dense_rows(URM, alpha, beta, min_rating, implicit)
    n = D.shape[0]
    k = min(topK, n) if topK is not False else n
    W = np.zeros_like(D)
    for i in range(n):
        order = np.lexsort((np.arange(n), -D[i]))[:k]
        order = order[D[i, order] != 0]
        W[i, order] = D[i, order]
    W = sps.csr_matrix(W)
    if normalize_similarity:
        W = _row_norm(W)
    if topK is not False:
        Wd = W.toarray()
        out = np.zeros_like(Wd)
        for c in range(n):
            col = Wd[:, c]
            nz = np.flatnonzero(col)
            keep = nz[np.lexsort((nz, -col[nz]))][:k]
            out[keep, c] = col[keep]
        W = sps.csr_matrix(out)
    return sps.csr_matrix(W, dtype=np.float32)
