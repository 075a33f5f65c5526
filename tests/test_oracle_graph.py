"""CPU: the P3alpha / RP3beta restatement (oracle/graph_oracle.py) against golden W_sparse matrices produced by the
reference's own GraphBased classes (tests/golden/make_golden.py::make_graph_golden)."""
import os
import runpy

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.graph_oracle import p3_similarity, p3_similarity_sparse
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

HERE = os.path.dirname(os.path.abspath(__file__))
GRAPH_CASES = runpy.run_path(os.path.join(HERE, "golden", "make_golden.py"), run_name="cases")["GRAPH_CASES"]
Z = np.load(os.path.join(HERE, "golden", "graph_golden.npz"))


def golden(n):
    return sps.csr_matrix((Z["g%d_data" % n], Z["g%d_indices" % n], Z["g%d_indptr" % n]), shape=(150, 150))


def case_inputs(n):
    c = dict(GRAPH_CASES[n])
    c.pop("cls")
    X = synth_urm(400, 150, 0.06, seed=17, values="continuous" if n % 2 == 0 else "ratings")
    return X, c


def close_enough(A, B, rtol=1e-4):
    """Same matrix up to top-K boundary ties: values agree where both have an entry, and the entries present in
    only one of them are at the K-th value of their row/column (tie class)."""
    A, B = A.toarray().astype(np.float64), B.toarray().astype(np.float64)
    both = (A != 0) & (B != 0)
    assert np.allclose(A[both], B[both], rtol=rtol, atol=1e-9)
    only = (A != 0) ^ (B != 0)
    return int(only.sum())


@pytest.mark.parametrize("n", range(len(GRAPH_CASES)))
def test_graph_oracle_matches_reference_golden(n):
    X, c = case_inputs(n)
    Wo = p3_similarity(X, **c)
    Wg = golden(n)
    assert Wo.shape == Wg.shape == (150, 150)
    mism = close_enough(Wo, Wg)
    if n % 2 == 0:  # continuous values: no ties, identical structure
        assert mism == 0
    else:
        assert mism <= 0.02 * Wg.nnz


def _assert_same(Ws, Wd):
    assert sps.isspmatrix_csr(Ws) and Ws.dtype == np.float32 and Ws.shape == Wd.shape
    Ws, Wd = Ws.copy(), Wd.copy()
    for W in (Ws, Wd):
        W.eliminate_zeros()
        W.sort_indices()
    assert np.array_equal(Ws.indptr, Wd.indptr) and np.array_equal(Ws.indices, Wd.indices)
    assert np.allclose(Ws.data, Wd.data, rtol=1e-12, atol=0)


def _signed_urm():
    """Ratings centred on 3 (stored zeros included): dot products of either sign, and rows whose positives plus zeros
    fall short of topK, so that negatives are kept."""
    X = synth_urm(300, 120, 0.08, seed=23, values="ratings")
    X.data -= 3.0
    return X


def _ragged_urm():
    """Users with no items, items nobody rated, a user with one item, and stored explicit zeros (counted in the degree
    and in Piu like any stored entry)."""
    X = synth_urm(200, 90, 0.05, seed=29, values="continuous").tolil()
    X[:20, :] = 0
    X[:, 40:50] = 0
    X[150, :] = 0
    X[150, 7] = 0.5
    X = sps.csr_matrix(X)
    X.eliminate_zeros()
    for u in (60, 61, 62):
        lo, hi = X.indptr[u], X.indptr[u + 1]
        assert hi > lo
        X.data[lo] = 0.0
    return X


SPARSE_CASES = ([("golden%d" % n, n, None) for n in range(len(GRAPH_CASES))]
                + [("signed", None, dict(topK=100, alpha=1.0, beta=0.0)),
                   ("signed_beta", None, dict(topK=30, alpha=1.0, beta=0.7, normalize_similarity=True)),
                   ("ragged", None, dict(topK=15, alpha=0.6, beta=1.5)),
                   ("ragged_normalized", None, dict(topK=200, alpha=1.3, beta=0.5, normalize_similarity=True))])


@pytest.mark.parametrize("name,golden_n,kw", SPARSE_CASES, ids=[c[0] for c in SPARSE_CASES])
def test_sparse_oracle_matches_dense(name, golden_n, kw):
    """p3_similarity_sparse (the restatement that scales to large catalogues) is p3_similarity: the same structure, the
    same values to 1e-12."""
    if golden_n is not None:
        X, kw = case_inputs(golden_n)
    else:
        X = _signed_urm() if name.startswith("signed") else _ragged_urm()
    Wd = p3_similarity(X, **kw)
    _assert_same(p3_similarity_sparse(X, **kw), Wd)
    assert Wd.nnz > 0 or golden_n is not None  # golden case 4 (min_rating=2 on values below 2) is empty
    if name == "signed":  # the case reaches the negatives
        assert (Wd.data < 0).any()
    if name.startswith("ragged"):
        assert (X.data == 0).any() and (np.diff(X.indptr) == 0).any() and (np.diff(X.tocsc().indptr) == 0).any()


def test_sparse_oracle_without_interactions():
    X = sps.csr_matrix((50, 40), dtype=np.float32)
    for kw in (dict(topK=5), dict(topK=5, beta=0.5, normalize_similarity=True)):
        W = p3_similarity_sparse(X, **kw)
        assert W.shape == (40, 40) and W.nnz == 0
        _assert_same(W, p3_similarity(X, **kw))
