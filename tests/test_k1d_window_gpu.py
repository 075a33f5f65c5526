"""K1-D pair path, cyclic half windows (csrc/sim_k1d.cuh): the upper pass of column c counts neighbour j iff
d = (j - c) mod n lies in [1, (n - 1) / 2], plus, when n is even, the antipodal d = n / 2 for c < n / 2 only, so that every
unordered pair is counted exactly once.  Rows are stored twice, back to back (the indices, then the indices + n), padded
to 16-byte chunks with an index that no window accepts.  As in test_k1d_pairs_gpu.py the full-range W must equal the sum
of the sub-range Ws (the K1-D kernel on every column, which reads only the first copy) exactly, and the pair path must
decide the columns itself: a counted pair missed or counted twice changes W, and a padding entry counted as a neighbour
breaks the nibble checksum, which sends the whole call to the K1-D kernel -- `-m gpu`."""
import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import _full_vs_parts, _phase_cycles, force_k1c  # noqa: F401 (fixture)
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_k1d_pairs_gpu import KINDS

pytestmark = pytest.mark.gpu

K = 50
KW = dict(topK=K, shrink=1000, similarity="cosine")  # the shrink keeps sim(3, largest norm) above every count-2 / count-1 cell



def _designed(n, specs, seed=11):
    """n columns, background counts ~ Poisson(0.8) (rows of ~6 entries, most not a multiple of 4), and for every (c, m, r)
    in specs: column c loses its background users and gets 3 * m / r users whose rows are c plus r of m chosen neighbours,
    every neighbour in exactly three of them, so c's candidate list (its count >= 3 cells) is exactly m long.  r = 30 gives
    c few users and puts it first in the norm order (its window is the lower half), r = 1 many users and puts it last (its
    window wraps round to the start)."""
    X = synth_urm(200_000, n, 0.002, seed=seed, values="binary").tocsr()
    cols = [c for c, _, _ in specs]
    X.data[np.isin(X.indices, cols)] = 0
    X.eliminate_zeros()
    rng = np.random.default_rng(seed)
    others = np.setdiff1d(np.arange(n), cols)
    rows = []
    for c, m, r in specs:
        nb = rng.choice(others, m, replace=False)
        for _ in range(3):
            perm = rng.permutation(nb)
            rows += [[c] + perm[b:b + r].tolist() for b in range(0, m, r)]
    indptr = np.cumsum([0] + [len(q) for q in rows])
    extra = sps.csr_matrix((np.ones(indptr[-1], np.float32), np.concatenate(rows), indptr), shape=(len(rows), n))
    X = sps.csr_matrix(sps.vstack([X, extra]), dtype=np.float32)
    X.sort_indices()
    Xc = X.tocsc()
    for c, m, _ in specs:
        cnt = (Xc[:, [c]].T @ Xc).toarray().ravel()
        cnt[c] = 0
        assert (cnt >= 3).sum() == m and cnt.max() <= 15
    return X


@pytest.mark.parametrize("n", [2999, 3000, 3002])
def test_windows_at_both_ends_of_the_norm_order(force_k1c, n):
    """Odd n, n a multiple of 8 (the first index past the catalogue, n, lies inside the windows of the last columns: the
    padding must not be it), and even n that is not (antipodal pairs).  A designed column first and one last in the norm
    order: the last one's window wraps round to the first."""
    X = _designed(n, [(4, 300, 30), (9, 300, 1)])
    assert (np.diff(X.indptr) % 4 != 0).mean() > 0.5
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[8] > 0 and cyc[11] > 0
    for c in (4, 9):
        assert W1[:, c].nnz == K


def test_stage_overflow_is_redone_without_fallback(force_k1c):
    """A column first in the norm order with 2600 candidates has about 1300 cells in its window, more than the stage: the
    cells past it reach their neighbours through the loose list, the column is redone, and the call does not fall back."""
    X = _designed(2999, [(5, 2600, 30)])
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[8] > 0 and cyc[1] > 0 and cyc[11] > 0
    assert W1[5, :].nnz > 2500  # it is in (nearly) every neighbour's top-K, so no loose cell may be lost


@pytest.mark.parametrize("kind", KINDS)
def test_every_formula_odd_n(force_k1c, kind):
    X = synth_urm(200_000, 2_999, 0.002, seed=7, values="binary")
    W1, cyc = _full_vs_parts(X, topK=50, shrink=5, similarity=kind, asymmetric_alpha=0.3, tversky_alpha=0.7,
                             tversky_beta=1.3)
    assert cyc[8] > 0 and cyc[11] > 0


def test_repeated_full_range_calls(force_k1c):
    """Full-range calls on one handle give the same W, also with a stage overflow and a wrapping window in every call."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    X = _designed(3002, [(5, 2600, 30), (9, 300, 1)])
    sim = Compute_Similarity_Cython(X, **KW)
    W1, cyc = _phase_cycles(sim, sim.compute_similarity)
    assert cyc[8] > 0 and cyc[11] > 0
    for _ in range(2):
        W = sim.compute_similarity()
        assert abs(W - W1).nnz == 0
