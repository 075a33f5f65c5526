"""Parity of the CUDA similarity path (through the C ABI) against the fp64 oracle -- `-m gpu`.

Index sets must be identical where the oracle's K-th value is separated (tie-aware, see
oracle.similarity_oracle.check_topk_against_dense); values within 1e-4 relative (north_star tolerance)."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import force_k1c  # noqa: F401 (fixture)
from oracle.similarity_oracle import SimilarityOracle, check_topk_against_dense
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

RTOL = 1e-4  # north_star: "within 1e-4 relative for float similarities"


def _gpu_cls():
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    return Compute_Similarity_Cython


def _check(X, cols=None, debug_cap=None, **kw):
    sim = _gpu_cls()(X, **kw)
    if debug_cap is not None:
        from recsys2019_deeplearning_evaluation_b200 import _lib
        _lib.check(_lib.load().b200_sim_debug_set_cap(sim._h, debug_cap))
    W = sim.compute_similarity()
    assert sps.isspmatrix_csr(W) and W.dtype == np.float32 and W.shape == (X.shape[1], X.shape[1])
    assert W.has_sorted_indices or (W.sorted_indices().indices == W.indices).all()
    assert (W.data != 0).all() and W.diagonal().sum() == 0
    orc = SimilarityOracle(X, **kw)
    cols = np.arange(X.shape[1]) if cols is None else cols
    ties = check_topk_against_dense(W, orc, cols, rtol=RTOL)
    return W, sim, ties


@pytest.mark.parametrize("kind", ["cosine", "asymmetric", "jaccard", "tanimoto", "dice", "tversky", "adjusted", "pearson"])
@pytest.mark.parametrize("values", ["continuous", "binary", "ratings"])
def test_kinds_small(kind, values):
    X = synth_urm(700, 300, 0.04, seed=3, values=values)
    _check(X, topK=25, shrink=7, normalize=True, similarity=kind, asymmetric_alpha=0.3, tversky_alpha=0.7,
           tversky_beta=1.3)


@pytest.mark.parametrize("kind", ["cosine", "asymmetric", "adjusted"])
@pytest.mark.parametrize("shrink", [0, 50])
def test_no_normalize(kind, shrink):
    X = synth_urm(500, 200, 0.05, seed=5, values="continuous")
    _check(X, topK=10, shrink=shrink, normalize=False, similarity=kind)


def test_exact_index_sets_continuous_c1():
    """BASELINE.json configs[0] shape, continuous values (tie-free): index sets identical to the oracle."""
    X = synth_urm(10_000, 5_000, 0.01, seed=42, values="continuous")
    W, sim, ties = _check(X, cols=np.arange(0, 5000, 7), topK=200, shrink=100, normalize=True, similarity="cosine")
    assert ties == 0
    assert not sim.binary_path and sim.n_windows == 1
    assert W.nnz == 5000 * 200


def test_binary_c1_tie_aware():
    X = synth_urm(10_000, 5_000, 0.01, seed=42, values="binary")
    W, sim, ties = _check(X, cols=np.arange(0, 5000, 11), topK=200, shrink=100, normalize=True, similarity="cosine")
    assert sim.binary_path


def test_row_weights():
    X = synth_urm(400, 150, 0.06, seed=9, values="ratings")
    w = np.random.default_rng(0).random(400).astype(np.float32) + 0.5
    _check(X, topK=15, shrink=3, similarity="cosine", row_weights=w)
    with pytest.raises(ValueError):
        _gpu_cls()(X, topK=5, row_weights=w[:-1])


def test_topk_larger_than_candidates_and_empty_columns():
    X = synth_urm(200, 120, 0.02, seed=2, values="continuous").tolil()
    X[:, 5] = 0
    X[:, 77] = 0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    W, sim, _ = _check(X, topK=500, shrink=0, similarity="cosine")
    assert sim.K == 120
    assert W[:, 5].nnz == 0 and W[5, :].nnz == 0


def test_signed_zeros_outrank_negatives():
    """Compute_Similarity_Python.py:335-345 semantics on centred data with few positives per column."""
    X = synth_urm(3000, 400, 0.004, seed=11, values="ratings")
    for kind in ("adjusted", "pearson"):
        W, sim, _ = _check(X, topK=50, shrink=0, similarity=kind)
        assert sim.signed_data


def test_negatives_emitted_when_zeros_run_out():
    """Dense-ish signed data with K close to n_columns: negatives fill the slots zeros cannot."""
    X = synth_urm(300, 40, 0.5, seed=4, values="ratings")
    W, sim, _ = _check(X, topK=39, shrink=0, similarity="pearson")
    assert (W.data < 0).any()


def test_column_range_and_unknown_similarity():
    X = synth_urm(500, 300, 0.03, seed=6, values="continuous")
    cls = _gpu_cls()
    sim = cls(X, topK=10, shrink=2, similarity="cosine")
    Wfull = sim.compute_similarity()
    Wpart = sim.compute_similarity(start_col=100, end_col=180)
    assert abs(Wpart[:, 100:180] - Wfull[:, 100:180]).max() < 1e-7
    assert Wpart[:, :100].nnz == 0 and Wpart[:, 180:].nnz == 0
    with pytest.raises(ValueError):
        cls(X, similarity="cosin")


def test_windowed_accumulator_matches_single_window(monkeypatch):
    """More columns than one shared-memory window holds: the multi-window path (C5 layout)."""
    X = synth_urm(20_000, 120_000, 0.0004, seed=8, values="continuous")
    W, sim, ties = _check(X, cols=np.arange(0, 120_000, 997), topK=50, shrink=10, similarity="cosine")
    assert sim.n_windows >= 2
    Xb = synth_urm(20_000, 120_000, 0.0004, seed=8, values="binary")
    W, sim, ties = _check(Xb, cols=np.arange(0, 120_000, 1499), topK=50, shrink=10, similarity="cosine")
    assert sim.n_windows >= 2 and sim.binary_path


def test_popular_item_long_column():
    """Zipf popularity: a few columns far longer than the staging chunk, heavy load imbalance."""
    X = synth_urm(30_000, 2_000, 0.01, seed=13, values="ratings", popularity=1.1)
    assert np.diff(X.tocsc().indptr).max() > 4096
    _check(X, cols=np.arange(0, 2000, 13), topK=100, shrink=10, similarity="cosine")


def test_dense_control_recipe_xtx():
    """Recipe of Base/Similarity/Compute_similarity_test.py:31-56: normalize=False, shrink=0, topK=n => X^T X
    with a zero diagonal."""
    rng = np.random.default_rng(0)
    D = (rng.random((60, 25)) * (rng.random((60, 25)) < 0.4)).astype(np.float32)
    X = sps.csr_matrix(D)
    W = _gpu_cls()(X, topK=25, shrink=0, normalize=False, similarity="cosine").compute_similarity().toarray()
    G = D.astype(np.float64).T @ D.astype(np.float64)
    np.fill_diagonal(G, 0)
    assert np.allclose(W, G, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("values", ["binary", "continuous", "ratings"])
def test_candidate_buffer_overflow_path(values):
    """A tiny logical candidate buffer forces the prune-and-rescan path on every column."""
    X = synth_urm(3000, 1500, 0.03, seed=21, values=values)
    _check(X, cols=np.arange(0, 1500, 5), debug_cap=40, topK=30, shrink=5, similarity="cosine")
    _check(X, cols=np.arange(0, 1500, 7), debug_cap=33, topK=30, shrink=0, similarity="jaccard")


def test_overflow_path_multiwindow_signed():
    X = synth_urm(8000, 110_000, 0.0008, seed=22, values="ratings")
    _check(X, cols=np.arange(0, 110_000, 1999), debug_cap=64, topK=20, shrink=1, similarity="pearson")


def test_binary_counter_widths(monkeypatch):
    """Binary path: 16-bit packed counters (chosen when they reduce the window count) and the 32-bit fallback give the
    same answer, single- and multi-window, and both match the oracle."""
    from recsys2019_deeplearning_evaluation_b200 import _lib
    import ctypes
    Xs = [synth_urm(10_000, 60_000, 0.001, seed=42, values="binary"), synth_urm(20_000, 230_000, 0.0003, seed=8, values="binary")]
    for X in Xs:
        kw = dict(topK=60, shrink=20, similarity="cosine")
        cols = np.arange(0, X.shape[1], max(1, X.shape[1] // 150))
        W16, sim16, _ = _check(X, cols=cols, **kw)
        bp = ctypes.c_int32()
        _lib.check(_lib.load().b200_sim_info(sim16._h, None, None, None, ctypes.byref(bp), None))
        assert bp.value == 2
        monkeypatch.setenv("B200REC_NO_PACK", "1")
        W32, sim32, _ = _check(X, cols=cols, **kw)
        _lib.check(_lib.load().b200_sim_info(sim32._h, None, None, None, ctypes.byref(bp), None))
        assert bp.value == 1 and sim32.n_windows > sim16.n_windows
        monkeypatch.delenv("B200REC_NO_PACK")
        assert abs(W16 - W32).max() < 1e-7 if (W16 - W32).nnz else True



# ---------------------------------------------------------------------------------------------------------------------
# K1-D: the 4-bit-counter kernel of the binary path (csrc/sim_k1d.cuh).  It is chosen by itself for binary data with
# >= 32768 columns; the environment hooks route small matrices through it as well.

def _k1c_info(sim):
    import ctypes
    from recsys2019_deeplearning_evaluation_b200 import _lib
    en, ctas, nb, nw = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    _lib.check(_lib.load().b200_sim_debug_k1c(sim._h, -1, ctypes.byref(en), ctypes.byref(ctas), ctypes.byref(nb), ctypes.byref(nw)))
    return en.value, ctas.value, nb.value, nw.value



@pytest.mark.parametrize("kind", ["cosine", "asymmetric", "jaccard", "tanimoto", "dice", "tversky"])
def test_k1c_kinds_small_forced(force_k1c, kind):
    """Every formula the nibble kernel serves, on a small binary matrix whose counts reach all three levels."""
    X = synth_urm(700, 300, 0.04, seed=3, values="binary")
    W, sim, _ = _check(X, topK=25, shrink=7, normalize=True, similarity=kind, asymmetric_alpha=0.3, tversky_alpha=0.7,
                       tversky_beta=1.3)
    en, ctas, nb, nw = _k1c_info(sim)
    assert en == 1 and nb > 0 and ctas == 2


def test_k1c_not_used_for_valued_or_signed_data(force_k1c):
    for values, kind in (("ratings", "cosine"), ("continuous", "cosine"), ("binary", "adjusted"), ("binary", "pearson")):
        X = synth_urm(400, 200, 0.05, seed=4, values=values)
        W, sim, _ = _check(X, topK=10, shrink=2, similarity=kind)
        assert _k1c_info(sim)[0] == 0


def test_k1c_sparse_catalogue_auto_and_against_window_kernel(monkeypatch):
    """230 K columns, sparse counts, columns of a handful of users: chosen without hooks, all non-empty columns on the
    nibble kernel (one CTA per SM: 115 KB of counters), same W as the window kernel."""
    X = synth_urm(20_000, 230_000, 0.0003, seed=42, values="binary")
    kw = dict(topK=50, shrink=10, similarity="cosine")
    cols = np.arange(0, X.shape[1], 997)
    W1, sim1, _ = _check(X, cols=cols, **kw)
    en, ctas, nb, nw = _k1c_info(sim1)
    assert en == 1 and ctas == 1
    assert nb == int((np.diff(X.tocsc().indptr) > 0).sum()) and nb + nw == X.shape[1]  # empty columns: window kernel
    monkeypatch.setenv("B200REC_K1C", "0")
    W0, sim0, _ = _check(X, cols=cols, **kw)
    assert _k1c_info(sim0)[0] == 0
    assert abs(W1 - W0).nnz == 0  # integer counts: both kernels are exact and deterministic


def test_k1c_c1_shape_levels_and_redo(force_k1c):
    """C1 shape (counts around 1, a good share >= 3): all three levels, the chunked pushes; with the test hook every 4th
    column is handed back through the redo list to the window kernel; column ranges; ties resolved like the window kernel."""
    X = synth_urm(10_000, 5_000, 0.01, seed=42, values="binary")
    kw = dict(topK=200, shrink=100, similarity="cosine")
    cols = np.arange(0, 5000, 11)
    W1, sim1, _ = _check(X, cols=cols, **kw)
    en, ctas, nb, nw = _k1c_info(sim1)
    assert en == 1 and nb > 0
    import ctypes
    from recsys2019_deeplearning_evaluation_b200 import _lib
    _lib.check(_lib.load().b200_sim_debug_k1c(sim1._h, 4, None, None, None, None))
    W1b = sim1.compute_similarity()
    en, ctas, nb2, nw2 = _k1c_info(sim1)
    assert nw2 >= nw + nb // 4  # columns were handed back
    _lib.check(_lib.load().b200_sim_debug_k1c(sim1._h, 0, None, None, None, None))
    force_k1c.setenv("B200REC_K1C", "0")
    W0, sim0, _ = _check(X, cols=cols, **kw)
    assert abs(W1 - W0).nnz == 0 and abs(W1b - W0).nnz == 0
    force_k1c.delenv("B200REC_K1C")
    Wp = sim1.compute_similarity(start_col=1000, end_col=1800)
    assert abs(Wp[:, 1000:1800] - W0[:, 1000:1800]).nnz == 0 and Wp[:, :1000].nnz == 0 and Wp[:, 1800:].nnz == 0


def test_k1c_counter_overflow_is_detected_and_redone(force_k1c):
    """Dense co-occurrence: nearly every pair of columns shares far more than 15 users, so 4-bit counters overflow in every
    column; the nibble checksum catches it and the window kernel recomputes the column."""
    X = synth_urm(2000, 100, 0.3, seed=6, values="binary")
    W, sim, _ = _check(X, topK=20, shrink=3, similarity="cosine")
    en, ctas, nb, nw = _k1c_info(sim)
    assert en == 1 and nb == 100 and nw == 100
    # a mixed case: a few popular columns overflow, the long tail does not
    Y = synth_urm(30_000, 2_000, 0.01, seed=13, values="binary", popularity=1.1)
    W, sim, _ = _check(Y, cols=np.arange(0, 2000, 13), topK=100, shrink=10, similarity="cosine")
    en, ctas, nb, nw = _k1c_info(sim)
    assert 0 < nw < 2000


def test_k1c_long_rows_and_short_columns(force_k1c):
    """Users with long profiles (rows of several 512-byte pieces) and columns of one or two users."""
    Y = synth_urm(300, 4_000, 0.2, seed=5, values="binary")  # rows of ~800 entries
    _check(Y, cols=np.arange(0, 4000, 41), topK=40, shrink=1, similarity="jaccard")
    Z = synth_urm(500, 3_000, 0.002, seed=5, values="binary")  # columns of ~1 user, rows of ~6 entries
    _check(Z, topK=10, shrink=0, similarity="cosine")


def test_k1c_empty_columns_topk_exceeds_candidates(force_k1c):
    X = synth_urm(200, 120, 0.02, seed=2, values="binary").tolil()
    X[:, 5] = 0
    X[:, 77] = 0
    X = sps.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    W, sim, _ = _check(X, topK=100, shrink=0, similarity="cosine")
    assert W[:, 5].nnz == 0 and W[5, :].nnz == 0


def test_k1c_handle_built_later_for_fewer_columns(force_k1c):
    """Two live handles launch the same nibble and window kernels, the one built later with less shared memory (fewer
    columns): each kernel's shared-memory limit is the launching handle's, so the first handle still computes."""
    X1 = synth_urm(700, 3000, 0.01, seed=3, values="binary")
    X2 = synth_urm(700, 300, 0.04, seed=3, values="binary")
    kw = dict(topK=25, shrink=7, similarity="cosine")
    sim1 = _gpu_cls()(X1, **kw)
    sim2 = _gpu_cls()(X2, **kw)
    assert _k1c_info(sim1)[0] == 1 and _k1c_info(sim2)[0] == 1
    W1 = sim1.compute_similarity()
    check_topk_against_dense(W1, SimilarityOracle(X1, **kw), np.arange(0, 3000, 7), rtol=RTOL)
    W2 = sim2.compute_similarity()
    check_topk_against_dense(W2, SimilarityOracle(X2, **kw), np.arange(300), rtol=RTOL)
