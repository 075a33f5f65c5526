"""K1-D pair path, the select kernel's list bound (csrc/sim_k1d.cuh, k1d_pair_gate in csrc/sim_topk.cu): a handle's select
kernel decides lists of up to sel_cap candidates, sized at create time from the longest expected list (Poisson) plus six
standard deviations and 32, in multiples of 8; a longer list is redone by the K1-D kernel and the call keeps the pair path.
Designed columns put lists on that bound from the column's own window only and from the other ends' windows only, and
exceed it many at once.  As in test_k1d_pairs_gpu.py the full-range W must equal the sum of the sub-range Ws exactly --
`-m gpu`."""
import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import _full_vs_parts, _phase_cycles, force_k1c  # noqa: F401 (fixture)
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

K = 50
KW = dict(topK=K, shrink=1000, similarity="cosine")  # the shrink keeps sim(3, largest norm) above every count-2 / count-1 cell



def _sel_cap(X):
    """The bound: the largest expected count >= 3 cell count of a non-empty column (Poisson with the column's hits per
    neighbour) plus six standard deviations and 32, in multiples of 8, at most 2048."""
    Xc = X.tocsc()
    n = X.shape[1]
    users = np.diff(Xc.indptr)
    work = np.add.reduceat(np.diff(X.indptr)[Xc.indices].astype(np.float64), Xc.indptr[:-1])
    lam = (work[users > 0] - users[users > 0]) / n
    est = (n * np.maximum(0.0, 1.0 - np.exp(-lam) * (1.0 + lam + 0.5 * lam * lam))).max()
    return int(min(np.ceil((est + 6.0 * np.sqrt(est) + 32.0) / 8.0) * 8.0, 2048))


def _in_window(n, c, j):
    """Whether the upper pass of column c (new numbering) counts neighbour j."""
    d = (j - c) % n
    return 1 <= d <= (n - 1) // 2 or (n % 2 == 0 and d == n // 2 and c < n // 2)


def _designed(specs, seed=11):
    """Background counts ~ Poisson(0.8) (about 140 candidates per column, ~400 users per column), and for every (c, m, side)
    in specs: column c loses its background users and gets rows of c plus some of m chosen neighbours, every neighbour in
    exactly three of them, so that c has exactly m candidates.  side "own": the m columns with the fewest users, in rows of
    30, so that c has the smallest norm term and every candidate lies in c's window (own list only); "mirror": the m
    columns with the most users, in rows of 1, so that c has the largest norm term and every candidate lies in the
    neighbour's window (mirror list only); "any": m random columns in rows of 1."""
    X = synth_urm(200_000, 3_000, 0.002, seed=seed, values="binary").tocsr()
    n = X.shape[1]
    cols = [s[0] for s in specs]
    X.data[np.isin(X.indices, cols)] = 0
    X.eliminate_zeros()
    users = np.diff(X.tocsc().indptr)
    rng = np.random.default_rng(seed)
    others = np.setdiff1d(np.arange(n), cols)
    ranked = others[np.lexsort((others, users[others]))]  # the new numbering among the background columns
    rows = []
    for c, m, side in specs:
        nb = {"own": ranked[:m], "mirror": ranked[-m:], "any": rng.choice(others, m, replace=False)}[side]
        r = 30 if side == "own" else 1
        for _ in range(3):
            perm = rng.permutation(nb)
            rows += [[c] + perm[b:b + r].tolist() for b in range(0, m, r)]
    indptr = np.cumsum([0] + [len(q) for q in rows])
    extra = sps.csr_matrix((np.ones(indptr[-1], np.float32), np.concatenate(rows), indptr), shape=(len(rows), n))
    X = sps.csr_matrix(sps.vstack([X, extra]), dtype=np.float32)
    Xc = X.tocsc()
    new = np.empty(n, np.int64)
    new[np.lexsort((np.arange(n), np.diff(Xc.indptr)))] = np.arange(n)
    for c, m, side in specs:
        cnt = (Xc[:, [c]].T @ Xc).toarray().ravel()
        cnt[c] = 0
        assert (cnt >= 3).sum() == m and cnt.max() <= 15
        nb = np.flatnonzero(cnt >= 3)
        if side == "own":
            assert all(_in_window(n, new[c], new[j]) for j in nb)
        elif side == "mirror":
            assert not any(_in_window(n, new[c], new[j]) for j in nb)
    return X


CAP = 344  # _sel_cap of every matrix below (the background sets it)


@pytest.mark.parametrize("side", ["own", "mirror"])
def test_list_at_the_bound_is_selected(force_k1c, side):
    """A list of exactly sel_cap candidates is decided by the select kernel: nothing is redone ([1] stays 0)."""
    X = _designed([(5, CAP, side)])
    assert _sel_cap(X) == CAP
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[1] == 0 and cyc[8] > 0 and cyc[11] > 0
    assert W1[:, 5].nnz == K


@pytest.mark.parametrize("side", ["own", "mirror"])
def test_list_past_the_bound_is_redone(force_k1c, side):
    """One candidate more: the column is redone by the K1-D kernel ([1]), every other column is still selected ([11])."""
    X = _designed([(5, CAP + 1, side)])
    assert _sel_cap(X) == CAP
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[1] > 0 and cyc[8] > 0 and cyc[11] > 0
    assert W1[:, 5].nnz == K


def test_many_long_lists_keep_the_pair_path(force_k1c):
    """Twelve columns with 400 candidates each: they are redone, and the call does not fall back (the select kernel still
    decides the other columns)."""
    specs = [(c, 400, "any") for c in range(20, 260, 20)]
    X = _designed(specs)
    assert _sel_cap(X) == CAP
    W1, cyc = _full_vs_parts(X, **KW)
    assert cyc[1] > 0 and cyc[11] > 0
    for c, *_ in specs:
        assert W1[:, c].nnz == K


def test_repeated_calls_with_redone_columns(force_k1c):
    """Full-range calls on one handle give the same W when columns are redone for their list length.  (Both columns have
    small norm terms: with one of the largest as well, count-2 cells could reach most columns' floor and the handle would
    not take the pair path.)"""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    X = _designed([(5, 600, "own"), (9, 400, "own")])
    sim = Compute_Similarity_Cython(X, **KW)
    W1, cyc = _phase_cycles(sim, sim.compute_similarity)
    assert cyc[1] > 0 and cyc[8] > 0 and cyc[11] > 0
    for _ in range(2):
        W = sim.compute_similarity()
        assert abs(W - W1).nnz == 0


def test_fail_every_with_long_lists(force_k1c):
    """The test hook sends the whole call down the K1-D kernel, long lists or not."""
    X = _designed([(5, 600, "own"), (9, 400, "own")])
    W1, cyc = _full_vs_parts(X, fail_every=3, **KW)
    assert cyc[10] == 0 and cyc[11] == 0 and cyc[1] > 0
