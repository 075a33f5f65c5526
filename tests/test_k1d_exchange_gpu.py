"""K1-D pair path, exchange and select (csrc/sim_k1d.cuh): the upper pass writes each column's count >= 3 cells as its own
list (cells past a column's shared-memory stage go to a loose list), the exchange copies them into the mirror lists of the
other end, and the select kernel decides every column from its own plus mirror list with one warp.  Designed columns put
the candidate-list lengths on the select kernel's boundaries (K, K + 1, 2048, 2049), overflow the stage, and sit at the
top of the norm order (mirror list only).  As in test_k1d_pairs_gpu.py the full-range W must equal the sum of the
sub-range Ws (the K1-D kernel on every column) exactly -- `-m gpu`."""
import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import _full_vs_parts, _phase_cycles, force_k1c  # noqa: F401 (fixture)
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

K = 50
S_CAP = 2048  # the longest candidate list the select kernel decides (= the upper pass's stage)
KW = dict(topK=K, shrink=1000, similarity="cosine")  # the shrink keeps sim(3, largest norm) above every count-2 / count-1 cell



def _designed(specs, seed=11):
    """Background counts ~ Poisson(0.8) (about 140 candidates per column), and for every (c, m, r) in specs: column c loses
    its background users and gets 3 * m / r users whose rows are c plus r of m chosen neighbours, every neighbour in exactly
    three of them.  Column c's candidate list (its count >= 3 cells) is then exactly m long, and c's norm term is set by r:
    r = 30 puts it below every background column (all its cells are its own, j > c), r = 1 above them (mirror list only)."""
    X = synth_urm(200_000, 3_000, 0.002, seed=seed, values="binary").tocsr()
    n = X.shape[1]
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
    Xc = X.tocsc()
    for c, m, _ in specs:
        cnt = (Xc[:, [c]].T @ Xc).toarray().ravel()
        cnt[c] = 0
        assert (cnt >= 3).sum() == m and cnt.max() <= 15
    return X


def test_list_length_boundaries(force_k1c):
    """Columns whose whole list is K, K + 1 (the select keeps all / cuts one), S_CAP (the longest list the select decides)
    and S_CAP + 1 (redone by the K1-D kernel).  The last one also overflows the upper pass's stage by one cell."""
    X = _designed([(3, K, 1), (7, K + 1, 1), (11, S_CAP, 30), (13, S_CAP + 1, 30)])
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[8] > 0 and cyc[10] > 0 and cyc[11] > 0
    for c in (3, 7, 11, 13):
        assert W1[:, c].nnz == K


def test_stage_overflow_keeps_the_pair_path(force_k1c):
    """A column with 2600 cells j > c overflows the stage: the cells past it reach their neighbours through the loose list
    (it is their best neighbour, so a lost cell changes their top-K), the column itself is redone, and the call does not
    fall back."""
    X = _designed([(5, 2600, 30)])
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[8] > 0 and cyc[11] > 0
    assert W1[5, :].nnz > 2500  # about 27 count >= 4 cells per column outrank it: it is in (nearly) every neighbour's top-K


def test_mirror_only_column(force_k1c):
    """A column with the largest norm term has the highest new index: every candidate comes from its mirror list."""
    X = _designed([(9, 300, 1)])
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[8] > 0 and cyc[11] > 0
    assert W1[:, 9].nnz == K


def test_repeated_full_range_calls(force_k1c):
    """The bench loop: full-range calls on one handle give the same W, so deg and the list counters are reset by every
    call -- also after a call that spilled cells to the loose list."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    X = _designed([(5, 2600, 30), (9, 300, 1)])
    sim = Compute_Similarity_Cython(X, **KW)
    W1, cyc = _phase_cycles(sim, sim.compute_similarity)
    assert cyc[8] > 0 and cyc[11] > 0
    for _ in range(2):
        W = sim.compute_similarity()
        assert abs(W - W1).nnz == 0
