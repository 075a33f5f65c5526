"""K1-D pair path (csrc/sim_k1d.cuh): a call over the whole column range gathers every co-occurrence count once (upper
pass), exchanges the count >= 3 pairs and selects from them; a call over a sub-range runs the K1-D kernel on every column.
Counts are integers and both paths build their keys from the same counts and norm terms, so the full-range W must equal
the union of sub-range results exactly -- `-m gpu`."""
import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import _full_vs_parts, force_k1c  # noqa: F401 (fixture)
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm

pytestmark = pytest.mark.gpu

KINDS = ["cosine", "asymmetric", "jaccard", "tanimoto", "dice", "tversky"]



def test_c5_full_shape_pairs_match_subranges():
    """C5 as bench.py times it (no hooks): the pair path runs, selects nearly every column itself, and its W is the W of the
    K1-D kernel on three sub-ranges."""
    X = synth_config("C5", values="binary")
    W1, cyc = _full_vs_parts(X, topK=200, shrink=100, similarity="cosine")
    assert cyc[8] > 0 and cyc[11] > 0
    assert W1.nnz == 200 * X.shape[1] - 200 * int((np.diff(X.tocsc().indptr) == 0).sum())


def test_c5_with_an_empty_column():
    """An empty column has norm term 0, but no count-1 / count-2 cell can have it as neighbour: the pair path still
    decides the columns itself."""
    X = synth_config("C5", values="binary").tocsr(copy=True)
    X.data[X.indices == 123] = 0
    X.eliminate_zeros()
    W1, cyc = _full_vs_parts(X, topK=200, shrink=100, similarity="cosine")
    assert cyc[8] > 0 and cyc[11] > 0
    assert W1[:, 123].nnz == 0 and W1[123, :].nnz == 0


def _uniform():
    # counts ~ Poisson(0.8): ~94 cells with count >= 3 per column; ~400 users per column keep the norm terms close together
    return synth_urm(200_000, 2_000, 0.002, seed=7, values="binary")


def test_redo_list(force_k1c):
    """K close to the typical number of count >= 3 cells: some columns have fewer than K and go through the redo list to the
    K1-D kernel ([1] = its gather), the others are selected from pairs ([11])."""
    W1, cyc = _full_vs_parts(_uniform(), topK=75, shrink=5, similarity="cosine")
    assert cyc[8] > 0 and cyc[1] > 0 and cyc[11] > 0


def test_counter_overflow_falls_back_for_the_whole_call(force_k1c):
    """20 extra users share three columns: their counts overflow a 4-bit counter in the upper pass, and the call falls back
    to the K1-D kernel (and the window kernel for its overflowed columns) on every column; none is selected from pairs."""
    X = _uniform()
    extra = sps.csr_matrix((np.ones(60, np.float32), np.tile([10, 11, 12], 20), np.arange(0, 61, 3)), shape=(20, X.shape[1]))
    X = sps.csr_matrix(sps.vstack([X, extra]), dtype=np.float32)
    W1, cyc = _full_vs_parts(X, topK=50, shrink=5, similarity="cosine")
    assert cyc[8] > 0 and cyc[10] == 0 and cyc[11] == 0 and cyc[1] > 0


def test_fail_every_hook_forces_the_fallback(force_k1c):
    """The hook sets the fallback flag before the upper pass takes a column: every column goes to the K1-D kernel."""
    W1, cyc = _full_vs_parts(_uniform(), fail_every=4, topK=50, shrink=5, similarity="cosine")
    assert cyc[10] == 0 and cyc[11] == 0 and cyc[1] > 0


def test_long_tail_catalogue_keeps_the_k1d_kernel(force_k1c):
    """Zipf(1.1) popularity: most columns have a few users, so count-2 cells can reach the floor of most columns; the pair
    path would hand them back, and the handle does not take it."""
    X = synth_urm(30_000, 2_000, 0.01, seed=13, values="binary", popularity=1.1)
    W1, cyc = _full_vs_parts(X, topK=100, shrink=10, similarity="cosine")
    assert cyc[8] == 0 and cyc[1] > 0


def test_c1_shape(force_k1c):
    """C1 shape: counts ~ Poisson(1), ~400 cells with count >= 3 per column against K = 200; the pair path is taken."""
    X = synth_urm(10_000, 5_000, 0.01, seed=42, values="binary")
    W1, cyc = _full_vs_parts(X, topK=200, shrink=100, similarity="cosine")
    assert cyc[8] > 0 and cyc[11] > 0


@pytest.mark.parametrize("kind", KINDS)
def test_every_formula(force_k1c, kind):
    W1, cyc = _full_vs_parts(_uniform(), topK=50, shrink=5, similarity=kind, asymmetric_alpha=0.3, tversky_alpha=0.7,
                             tversky_beta=1.3)
    assert cyc[8] > 0 and cyc[11] > 0


def test_empty_columns(force_k1c):
    X = _uniform().tolil()
    X[:, 5] = 0
    X[:, 1500] = 0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    W1, cyc = _full_vs_parts(X, topK=50, shrink=5, similarity="cosine")
    assert cyc[8] > 0 and cyc[11] > 0
    assert W1[:, 5].nnz == 0 and W1[5, :].nnz == 0 and W1[:, 1500].nnz == 0 and W1[1500, :].nnz == 0
