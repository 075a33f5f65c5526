"""K1-D packed rows (csrc/sim_k1d.cuh): a 16-byte chunk holds up to seven entries of a user's doubled row, a 32-bit index
and six 16-bit gaps; gap 0 is an empty slot, and an entry 65 536 or more after its predecessor starts a new chunk.  Both
K1-D kernels decode this layout, so comparing them with each other (as test_k1d_window_gpu.py does) would pass a decoding
bug they share: here the full-range W (pair path) must also equal the window kernel's W (B200REC_K1C=0, which never reads
the layout) exactly, and agree with the fp64 oracle on chosen columns.  The pair path must decide the columns itself: a
padding slot counted as an entry, or an entry missed, breaks the nibble checksum and sends the call to the K1-D kernel,
which shows as cyc[11] == 0 -- `-m gpu`."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import _lib, _phase_cycles, force_k1c  # noqa: F401 (fixture)
from oracle.similarity_oracle import SimilarityOracle, check_topk_against_dense
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_k1d_window_gpu import _designed

pytestmark = pytest.mark.gpu

KW = dict(topK=20, shrink=1000, similarity="cosine")  # the shrink keeps sim(3, largest norm) above every count-2 / count-1 cell



def _check(X, monkeypatch, cols):
    """Full-range W on the pair path (twice on one handle), the K1-D kernel alone on two half ranges, the window kernel,
    and the oracle on `cols`."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    sim = Compute_Similarity_Cython(X, **KW)
    en = ctypes.c_int32()
    _lib().check(_lib().load().b200_sim_debug_k1c(sim._h, 0, ctypes.byref(en), None, None, None))
    assert en.value == 1
    W1, cyc = _phase_cycles(sim, sim.compute_similarity)
    assert cyc[8] > 0 and cyc[11] > 0  # upper pass and select ran; after a fallback the select emits nothing
    assert abs(sim.compute_similarity() - W1).nnz == 0  # the upper pass left its counters and deg clean
    n = X.shape[1]
    Wp = None
    for lo, hi in ((0, n // 2), (n // 2, n)):
        Wh, cyc_h = _phase_cycles(sim, lambda: sim.compute_similarity(start_col=lo, end_col=hi))
        assert cyc_h[8:12].sum() == 0 and cyc_h[1] > 0  # a sub-range runs the K1-D kernel on whole rows
        Wp = Wh if Wp is None else Wp + Wh
    assert abs(W1 - Wp).nnz == 0
    del sim
    monkeypatch.setenv("B200REC_K1C", "0")
    sim0 = Compute_Similarity_Cython(X, **KW)
    _lib().check(_lib().load().b200_sim_debug_k1c(sim0._h, 0, ctypes.byref(en), None, None, None))
    assert en.value == 0
    assert abs(W1 - sim0.compute_similarity()).nnz == 0  # integer counts: both are exact
    monkeypatch.delenv("B200REC_K1C")
    check_topk_against_dense(W1, SimilarityOracle(X, **KW), np.asarray(cols), rtol=1e-4)
    return W1


@pytest.mark.parametrize("n", [2999, 3000, 3002])
def test_short_rows_at_every_chunk_boundary(force_k1c, n):
    """Rows of ~6 entries: the doubled row of a length-L row fills 2 L mod 7 slots of its last chunk, and lengths 1, 2, 6,
    7, 8, 13, 14, 15 put the wrap and the end of the row at either end of a chunk.  Odd n, n a multiple of 8 (the first
    index past the catalogue lies inside the windows of the last columns: an empty slot must not be it) and even n
    (antipodal pairs); one designed column at each end of the norm order, the last one's window wrapping."""
    X = _designed(n, [(4, 300, 30), (9, 300, 1)])
    assert {1, 2, 6, 7, 8, 13, 14, 15} <= set(np.diff(X.indptr).tolist())
    W1 = _check(X, force_k1c, np.r_[4, 9, np.arange(0, n, 211)])
    for c in (4, 9):
        assert W1[:, c].nnz == KW["topK"]


def _with_designed_rows(n, rows_new, reps=8, seed=5):
    """A uniform background (37 K rows of ~400 entries: counts ~ Poisson(0.3), ~500 cells with count >= 3 per column) plus
    every row of rows_new `reps` times.  rows_new is in the kernels' column numbering: ascending norm term, then ascending
    index -- for cosine on binary data, a stable sort of the column counts.  Every column a designed row uses gives up as
    many background entries as it gains, so the counts, and with them the numbering, are those of the background."""
    X0 = synth_urm(37_000, n, 400.0 / n, seed=seed, values="binary").tocsc()
    counts = np.diff(X0.indptr)
    new2old = np.argsort(counts, kind="stable")
    rows_old = [new2old[np.asarray(r)] for r in rows_new]
    used, times = np.unique(np.concatenate(rows_old), return_counts=True)
    for c, t in zip(used, times * reps):
        assert counts[c] > t
        X0.data[X0.indptr[c]:X0.indptr[c] + t] = 0
    X0.eliminate_zeros()
    rep = [r for r in rows_old for _ in range(reps)]
    indptr = np.cumsum([0] + [len(r) for r in rep])
    extra = sps.csr_matrix((np.ones(indptr[-1], np.float32), np.concatenate(rep), indptr), shape=(len(rep), n))
    X = sps.csr_matrix(sps.vstack([X0.tocsr(), extra]), dtype=np.float32)
    X.sort_indices()
    assert (np.diff(X.tocsc().indptr) == counts).all()
    return X, rows_old


@pytest.mark.parametrize("n", [140_000, 140_003])
def test_gaps_around_65536(force_k1c, n):
    """Designed rows (eight users each, so that every pair in them has count >= 8 and leads its columns' top-K) in a
    catalogue wide enough for 16-bit gaps to overflow.  n a multiple of 8 and odd n; the windows of the upper half of
    the columns wrap."""
    rows_new = [
        [100, 100 + 65535, 100 + 65535 + 65536],  # gap 65 535 fits; 65 536 starts a chunk, in both copies.  Column 65 635 is
                                                  # the last entry of a chunk closed early; its window starts at a chunk base
                                                  # and ends at it (the next entry, 100 + n, lies past the window)
        [200, 200 + 65537, 200 + 65537 + 7],      # gap 65 537
        [70000, 70010, 70020],                    # the wrap (first + n - last) is the only gap that starts a chunk
        [1000, 30000, 1000 + n - 65536],          # wrap gap exactly 65 536
        [1001, 30001, 1001 + n - 65535],          # wrap gap exactly 65 535: the second copy continues the chunk
        [2000, 2000 + n - 65537],                 # two entries, wrap gap 65 537
        [90000],                                  # one entry: its second copy is a chunk of its own and nothing is counted
        [5000 + 37 * i for i in range(15)],       # 30 doubled entries: every entry is the column of one window, so the
                                                  # windows start after every slot of a chunk, its last one and its base included
    ]
    X, rows_old = _with_designed_rows(n, rows_new)
    cols = np.unique(np.concatenate(rows_old))
    W1 = _check(X, force_k1c, np.r_[cols, np.arange(0, n, 9973)])
    Wc = W1.tocsc()
    for r in rows_old:
        for c in r:
            assert np.isin(np.setdiff1d(r, [c]), Wc.indices[Wc.indptr[c]:Wc.indptr[c + 1]]).all()
