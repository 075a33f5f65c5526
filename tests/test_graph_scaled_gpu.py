"""-m gpu: the scaled-product formula of the similarity kernel (P3alpha / RP3beta: b200_sim_create_scaled) against fp64,
across accumulator windows, candidate-buffer prunes and top-K sizes, and P3alpha / RP3beta end to end.

The kernel computes value[i, j] = A_i * B_j * sum over the users u that store (u, i) of X[u, j], the diagonal 0, and
keeps for every target i the K largest of its n cells (implicit zeros outrank negatives, ties to the ascending original
index), zeros dropped.  Columns are renumbered by ascending B, so this is the one formula whose pruning bounds rise with
the neighbour's norm term, and B changes inside a 4 096-cell tile when it comes from RP3beta's degrees.

The exact tests choose inputs on which fp32 is exact: stored values are multiples of 2^-3 with |x| <= 1, every column
is far shorter than 2^16 users, A and B are powers of two or 0.  Every atomic sum and every d * A_i * B_j is then exact
in any order, so each table row must equal the fp64 reference: the same indices, the same values bit for bit, the same
count, and -1 / 0.0 past the count.  The coarse value grid makes many exact ties, so the K boundary is tested hard.

Every multi-window case first asserts its route as b200_sim_info reads it (n_windows, window_cells, binary_path == 0),
and prints it (run with -s to see it)."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.graph_oracle import _line_order, _row_norm, p3_dense_rows, p3_sparse_rows, sparse_column_topk, sparse_row_topk
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
EMPTY_COLS = (5, 777)      # items nobody rated
A0_TARGET = 3              # a rated item with A = 0
B0_COLS = (1, 17, 123)     # rated items with B = 0 (an fp32 underflow of deg^-beta)
EMPTY_USERS = range(0, 10)
ONE_ITEM_USER = 10         # a user with one item: only the target's own cell


def _L():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


class Scaled:
    """A scaled handle over X (CSR float32, stored zeros kept) with A, B as given."""

    def __init__(self, X, A, B, K):
        L = _L()
        self.n = X.shape[1]
        ip, ix, dt = (np.ascontiguousarray(X.indptr, np.int32), np.ascontiguousarray(X.indices, np.int32),
                      np.ascontiguousarray(X.data, np.float32))
        A32, B32 = np.ascontiguousarray(A, np.float32), np.ascontiguousarray(B, np.float32)
        self.h = ctypes.c_void_p()
        L.check(L.load().b200_sim_create_scaled(ctypes.byref(self.h), X.shape[0], self.n, X.nnz, L.ptr(ip), L.ptr(ix),
                                                L.ptr(dt), L.ptr(A32), L.ptr(B32), K, None))
        k, nw, wc, bp, sd = (ctypes.c_int32() for _ in range(5))
        L.check(L.load().b200_sim_info(self.h, ctypes.byref(k), ctypes.byref(nw), ctypes.byref(wc), ctypes.byref(bp),
                                       ctypes.byref(sd)))
        self.K, self.route = k.value, (nw.value, wc.value, bp.value)

    def set_cap(self, cap):
        _L().check(_L().load().b200_sim_debug_set_cap(self.h, cap))

    def compute(self, lo, hi):
        """Table rows of targets [lo, hi) on the device: idx, val [hi - lo, K], cnt [hi - lo]."""
        import torch
        m = max(hi - lo, 1)
        idx = torch.full((m, self.K), 7, dtype=torch.int32, device="cuda")  # junk: every slot must be written
        val = torch.full((m, self.K), 7.0, dtype=torch.float32, device="cuda")
        cnt = torch.full((m,), -7, dtype=torch.int32, device="cuda")
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _L().check(_L().load().b200_sim_compute_device(self.h, lo, hi, idx.data_ptr(), val.data_ptr(), cnt.data_ptr(), st))
        return idx, val, cnt

    def rows(self, targets, one_by_one=False):
        """Host tables of `targets`: from one call over every column, or (one_by_one) one call per target."""
        import torch
        if one_by_one:
            parts = [self.compute(int(t), int(t) + 1) for t in targets]
            return tuple(torch.cat([p[k] for p in parts]).cpu().numpy() for k in range(3))
        idx, val, cnt = self.compute(0, self.n)
        sel = torch.as_tensor(np.asarray(targets), device="cuda")
        return idx[sel].cpu().numpy(), val[sel].cpu().numpy(), cnt[sel].cpu().numpy()

    def close(self):
        _L().load().b200_sim_destroy(self.h)


def _assert_route(route, n, label, least, most=None):
    n_win, cells, bp = route
    print("%s: n_items=%d n_windows=%d window_cells=%d binary_path=%d" % (label, n, n_win, cells, bp))
    assert bp == 0, (label, route)
    assert n_win >= least and (most is None or n_win <= most), (label, route)
    assert n_win * cells >= n and (n_win == 1) == (cells >= n), (label, route)


# ------------------------------------------------------------------------------------------------ exact inputs


def _exact_urm(n_users, n_items, density, seed, signed=False, dense_user=False):
    """Long-tail URM (the most popular column holds thousands of users) with values k / 8, k = 1..8 (negated with
    probability 0.35 when signed), users with no items, a user with one item, items nobody rated and a few stored zeros.
    dense_user: one more user rates every item that is not empty with -k / 8, so that every row is almost full and
    negatives must fill the K slots of the targets with few positives."""
    X = synth_urm(n_users, n_items, density, seed=seed, values="binary", popularity=0.8).tocoo()
    keep = ~np.isin(X.row, EMPTY_USERS) & ~np.isin(X.col, EMPTY_COLS) & ~(dense_user & (X.row == n_users - 1))
    r, c = X.row[keep], X.col[keep]
    one = np.flatnonzero(r == ONE_ITEM_USER)
    keep = np.ones(len(r), bool)
    keep[one[1:]] = False
    r, c = r[keep], c[keep]
    if not len(one):
        r, c = np.append(r, ONE_ITEM_USER), np.append(c, 4)
    rng = np.random.default_rng(seed + 1)
    v = rng.integers(1, 9, len(r)) / 8.0
    if signed:
        v[rng.random(len(r)) < 0.35] *= -1
    v[rng.choice(len(r), 40, replace=False)] = 0.0  # stored zeros: counted in the pattern like any stored value
    if dense_user:
        cols = np.setdiff1d(np.arange(n_items), EMPTY_COLS)
        r = np.append(r, np.full(len(cols), n_users - 1))
        c = np.append(c, cols)
        v = np.append(v, -rng.integers(1, 9, len(cols)) / 8.0)
    X = sps.csr_matrix((v.astype(np.float32), (r, c)), shape=(n_users, n_items))
    X.sort_indices()
    lens = np.diff(X.tocsc().indptr)
    assert lens.max() < 2 ** 16 and (lens[list(EMPTY_COLS)] == 0).all() and lens[A0_TARGET] > 0
    assert (lens[list(B0_COLS)] > 0).all() and np.diff(X.indptr)[ONE_ITEM_USER] == 1 and (X.data == 0).any()
    return X


def _exact_ab(X, bshape, seed):
    """A: 2^-k (k = 0..7), 0 on empty items and on the rated item A0_TARGET.  B: 1 everywhere ('const', P3alpha: every
    tile bound is equal) or 2^-k (k = 0..20, changing inside every tile), 0 on empty items and on the rated B0_COLS."""
    n = X.shape[1]
    rng = np.random.default_rng(seed)
    empty = np.diff(X.tocsc().indptr) == 0
    A = 2.0 ** -rng.integers(0, 8, n)
    A[empty] = 0.0
    A[A0_TARGET] = 0.0
    if bshape == "const":
        B = np.ones(n)
    else:
        B = 2.0 ** -rng.integers(0, 21, n)
        B[empty] = 0.0
        B[list(B0_COLS)] = 0.0
    return A, B


def _exact_ref(X, A, B, targets):
    """fp64 rows of the targets: A_t * (pattern(X)[:, t] . X) * B, the target's own cell and every zero dropped."""
    C = sps.csc_matrix(X, dtype=np.float64)
    Pat = C[:, targets]
    Pat.data[:] = 1.0
    R = sps.coo_matrix(sps.diags(A[targets]) @ (Pat.T @ C) @ sps.diags(B))
    keep = (R.col != np.asarray(targets)[R.row]) & (R.data != 0)
    return sps.csr_matrix((R.data[keep], (R.row[keep], R.col[keep])), shape=(len(targets), X.shape[1]))


def _targets(X, B, n_random=200, seed=0):
    """The smallest and largest B, the most popular items, the special items and a fixed random sample."""
    n = X.shape[1]
    lens = np.diff(X.tocsc().indptr)
    order_b = np.argsort(B, kind="stable")
    rng = np.random.default_rng(seed)
    t = np.concatenate([[0, 2, 4, n - 1, A0_TARGET], B0_COLS, EMPTY_COLS, np.argsort(-lens, kind="stable")[:8],
                        order_b[:8], order_b[-8:], rng.choice(n, min(n, n_random), replace=False)])
    return np.unique(t[t < n])


def _assert_rows_exact(label, got, E, targets, K):
    idx, val, cnt = got
    for r, t in enumerate(targets):
        lo, hi = E.indptr[r], E.indptr[r + 1]
        c = int(cnt[r])
        where = "%s target %d" % (label, t)
        assert c == hi - lo, "%s: %d entries, reference %d" % (where, c, hi - lo)
        o = np.argsort(idx[r, :c], kind="stable")
        gi, gv = idx[r, :c][o], val[r, :c][o]
        if not np.array_equal(gi, E.indices[lo:hi]):
            extra = np.setdiff1d(gi, E.indices[lo:hi])[:5]
            missing = np.setdiff1d(E.indices[lo:hi], gi)[:5]
            pytest.fail("%s: index sets differ: extra %s, missing %s" % (where, extra, missing))
        bad = gv.astype(np.float64) != E.data[lo:hi]
        if bad.any():
            k = int(np.argmax(bad))
            pytest.fail("%s: %d values differ, the first at %d: %r, reference %r" % (
                where, int(bad.sum()), gi[k], gv[k], E.data[lo + k]))
        assert (idx[r, c:] == -1).all() and (val[r, c:].view(np.uint32) == 0).all(), where


# name -> (n_users, n_items, density, least n_windows, most n_windows)
SHAPES = {
    "one_window": (6000, 3000, 0.01, 1, 1),
    "two_windows": (16000, 60000, 0.0008, 2, 2),
    "three_windows": (20000, 120000, 0.0004, 3, None),
}
CAP_SLACK = 64  # the small logical buffer: K + CAP_SLACK candidates, pruned again and again on the popular targets


@pytest.fixture(scope="module")
def exact_case():
    cache = {}

    def get(shape, bshape):
        if (shape, bshape) not in cache:
            nu, ni, d = SHAPES[shape][:3]
            X = _exact_urm(nu, ni, d, seed=ni % 97)
            A, B = _exact_ab(X, bshape, seed=ni % 89)
            t = _targets(X, B)
            cache[(shape, bshape)] = (X, A, B, t, _exact_ref(X, A, B, t))
        return cache[(shape, bshape)]
    return get


@pytest.mark.parametrize("K", [1, 7, 100, 2048])
@pytest.mark.parametrize("bshape", ["const", "tiles"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_exact_tables(exact_case, shape, bshape, K):
    """One, two and three windows; constant B and B over 2^-20..1; the default buffer and K + CAP_SLACK slots."""
    X, A, B, targets, R = exact_case(shape, bshape)
    n = X.shape[1]
    E = sparse_row_topk(R, K)
    h = Scaled(X, A, B, K)
    try:
        label = "%s %s K=%d" % (shape, bshape, K)
        _assert_route(h.route, n, label, *SHAPES[shape][3:])
        _assert_rows_exact(label, h.rows(targets), E, targets, K)
        if h.route[0] > 1:
            h.set_cap(K + CAP_SLACK)
            _assert_rows_exact(label + " cap=K+%d" % CAP_SLACK, h.rows(targets, one_by_one=True), E, targets, K)
    finally:
        h.close()
    cnt = np.diff(E.indptr)
    assert cnt.max() == K and (cnt[list(targets).index(A0_TARGET)] == 0)


@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("bshape", ["const", "tiles"])
def test_exact_small_catalogue_every_k(signed, bshape):
    """2 048 items, every target, K from 100 to n: the K = n - 1 and K = n tables hold every non-zero cell; on signed data
    the negatives fill what the positives and the zeros leave (B = 0 on a rated item makes a zero of a non-zero dot
    product, and that zero outranks the negatives)."""
    X = _exact_urm(4000, 2048, 0.01, seed=11, signed=signed)
    n = X.shape[1]
    A, B = _exact_ab(X, bshape, seed=12)
    targets = np.arange(n)
    R = _exact_ref(X, A, B, targets)
    emitted_neg = skipped_neg = 0
    for K in (100, 1500, n - 1, n):
        E = sparse_row_topk(R, K)
        h = Scaled(X, A, B, K)
        try:
            _assert_route(h.route, n, "small %s signed=%s K=%d" % (bshape, signed, K), 1, 1)
            _assert_rows_exact("small %s signed=%s K=%d" % (bshape, signed, K), h.rows(targets), E, targets, K)
        finally:
            h.close()
        has_neg = np.bincount(R.tocoo().row[R.data < 0], minlength=n) > 0
        kept_neg = np.bincount(E.tocoo().row[E.data < 0], minlength=n) > 0
        emitted_neg += int(kept_neg.sum())
        skipped_neg += int((has_neg & ~kept_neg).sum())
    if signed:
        assert emitted_neg > 0 and skipped_neg > 0, (emitted_neg, skipped_neg)


@pytest.mark.parametrize("K", [7, 2048])
def test_exact_signed_several_windows(K):
    """60 000 signed items and a user who rates every item negatively: rows are almost full, so a target with few
    positives emits negatives, in both windows; B = 0 on rated items; the default buffer and K + CAP_SLACK slots."""
    X = _exact_urm(6000, 60000, 0.0008, seed=31, signed=True, dense_user=True)
    n = X.shape[1]
    A, B = _exact_ab(X, "tiles", seed=32)
    lens = np.diff(X.tocsc().indptr)
    rng = np.random.default_rng(5)
    targets = np.unique(np.concatenate([[0, A0_TARGET, n - 1], B0_COLS, np.argsort(-lens, kind="stable")[:4],
                                        np.flatnonzero(lens == 1)[:6], rng.choice(n, 16, replace=False)]))
    R = _exact_ref(X, A, B, targets)
    E = sparse_row_topk(R, K)
    assert (E.data < 0).any()
    h = Scaled(X, A, B, K)
    try:
        label = "signed dense user K=%d" % K
        _assert_route(h.route, n, label, 2, 2)
        _assert_rows_exact(label, h.rows(targets), E, targets, K)
        h.set_cap(K + CAP_SLACK)
        _assert_rows_exact(label + " cap=K+%d" % CAP_SLACK, h.rows(targets, one_by_one=True), E, targets, K)
    finally:
        h.close()


def test_column_ranges_and_repeated_calls(exact_case):
    """Sub-ranges, the last column and empty ranges give the rows of the full call; a second call the same table."""
    X, A, B, _, _ = exact_case("two_windows", "tiles")
    n = X.shape[1]
    h = Scaled(X, A, B, 100)
    try:
        full = [a.cpu().numpy() for a in h.compute(0, n)]
        again = [a.cpu().numpy() for a in h.compute(0, n)]
        _assert_same_tables(full, again, 0, n, "second call")
        for lo, hi in ((0, 1), (n - 1, n), (123, 4567), (n // 2, n), (31_000, 31_001)):
            part = [a.cpu().numpy() for a in h.compute(lo, hi)]
            _assert_same_tables(full, part, lo, hi, "range [%d, %d)" % (lo, hi))
        before = _L().launch_count()
        for lo in (0, n // 2, n):
            _L().check(_L().load().b200_sim_compute_device(h.h, lo, lo, None, None, None, None))
        assert _L().launch_count() == before
    finally:
        h.close()


def _assert_same_tables(full, part, lo, hi, label):
    fi, fv, fc = (a[lo:hi] for a in full)
    pi, pv, pc = (a[:hi - lo] for a in part)
    assert np.array_equal(fc, pc), label
    for r in range(hi - lo):
        c = fc[r]
        a, b = np.argsort(fi[r, :c]), np.argsort(pi[r, :c])
        assert np.array_equal(fi[r, :c][a], pi[r, :c][b]), (label, lo + r)
        assert np.array_equal(fv[r, :c][a].view(np.uint32), pv[r, :c][b].view(np.uint32)), (label, lo + r)
        assert (pi[r, c:] == -1).all() and (pv[r, c:].view(np.uint32) == 0).all(), (label, lo + r)


def test_a_smaller_scaled_handle_built_later_does_not_break_a_larger_one(exact_case):
    """The scaled formula has a kernel instantiation of its own: a small handle built after a large one must leave the
    large one's launches (a larger accumulator window) intact."""
    Xb, Ab, Bb, tb, Rb = exact_case("three_windows", "tiles")
    Xs, As, Bs, ts, Rs = exact_case("one_window", "tiles")
    big = Scaled(Xb, Ab, Bb, 100)
    small = Scaled(Xs, As, Bs, 100)
    try:
        assert big.route[1] > small.route[1] or big.route[0] > 1
        _assert_rows_exact("big after small", big.rows(tb), sparse_row_topk(Rb, 100), tb, 100)
        _assert_rows_exact("small", small.rows(ts), sparse_row_topk(Rs, 100), ts, 100)
    finally:
        big.close()
        small.close()


def test_no_interactions():
    X = sps.csr_matrix((40, 300), dtype=np.float32)
    h = Scaled(X, np.ones(300), np.ones(300), 10)
    try:
        idx, val, cnt = h.rows(np.arange(300))
        assert (cnt == 0).all() and (idx == -1).all() and (val.view(np.uint32) == 0).all()
    finally:
        h.close()


# ------------------------------------------------------------------------------------------------ realistic inputs


def _tol(X, alpha, beta):
    """Per item i, the relative error bound of its table values: an fp32 sum of len_i non-negative terms (len_i * 2^-23,
    len_i the item's column length), the two fp32 products by A_i and B_j (2^-23), and the error of the fp32 inputs
    that graph.scaled_inputs prepares (Pui^alpha, A, B: their largest relative deviation from fp64, measured here --
    numpy's float32 power alone is off by up to ~14 * 2^-24 at alpha = 1.7)."""
    from recsys2019_deeplearning_evaluation_b200.graph import scaled_inputs
    Pui, A, B = scaled_inputs(X, alpha, beta)
    P64 = _row_norm(sps.csr_matrix(X, dtype=np.float32))
    if alpha != 1.0:
        P64 = P64.power(alpha)
    lens = np.diff(sps.csc_matrix(X).indptr).astype(np.float64)
    m = lens > 0
    A64, B64 = np.zeros_like(lens), np.ones_like(lens)
    A64[m] = (1.0 / lens[m]) ** alpha
    if beta != 0.0:
        B64[m] = lens[m] ** -beta
    assert np.array_equal(Pui.indices, P64.indices) and (A[~m] == 0).all()

    def rel(a, b):
        nz = b != 0
        return float(np.max(np.abs(a[nz] - b[nz]) / np.abs(b[nz]), initial=0.0))
    eps_in = rel(Pui.data.astype(np.float64), P64.data) + rel(A.astype(np.float64)[m], A64[m]) + rel(B.astype(np.float64)[m], B64[m])
    return lens * U + U + eps_in


def _check_rows_tol(label, got, P, targets, K, tol):
    """Row r of `got` against the fp64 row P[r]: shared indices within tol[r] relative; an index on one side only must be
    a near-tie, its fp64 value within tol[r] of the row's K-th fp64 value."""
    idx, val, cnt = got
    E = sparse_row_topk(P, K)
    n_only = 0
    for r, t in enumerate(targets):
        lo, hi = P.indptr[r], P.indptr[r + 1]
        prow = dict(zip(P.indices[lo:hi].tolist(), P.data[lo:hi].tolist()))
        ecols = E.indices[E.indptr[r]:E.indptr[r + 1]]
        c = int(cnt[r])
        gi, gv = idx[r, :c], val[r, :c].astype(np.float64)
        assert c == len(ecols), "%s target %d: %d entries, reference %d" % (label, t, c, len(ecols))
        kth = np.sort(P.data[lo:hi])[::-1][K - 1] if hi - lo >= K else None
        for j, v in zip(gi.tolist(), gv.tolist()):
            ref = prow.get(j, 0.0)
            assert abs(v - ref) <= tol[r] * ref, "%s target %d neighbour %d: %r, fp64 %r" % (label, t, j, v, ref)
        for j in np.setxor1d(gi, ecols).tolist():
            ref = prow.get(j, 0.0)
            assert kth is not None and abs(ref - kth) <= tol[r] * kth, \
                "%s target %d: neighbour %d (fp64 %r) on one side only, K-th fp64 value %r" % (label, t, j, ref, kth)
            n_only += 1
    return n_only


REALISTIC = [("continuous", 0.3, 0.0), ("continuous", 1.0, 0.5), ("continuous", 1.7, 2.0),
             ("ratings", 0.3, 2.0), ("ratings", 1.0, 0.0), ("ratings", 1.7, 0.5)]


@pytest.mark.parametrize("shape", ["one_window", "two_windows"])
@pytest.mark.parametrize("values,alpha,beta", REALISTIC)
def test_realistic_against_fp64(values, alpha, beta, shape):
    """P3alpha / RP3beta inputs as graph.py prepares them from a long-tail URM, K = 100, against fp64 on sampled targets,
    with the default buffer and with K + CAP_SLACK slots."""
    from recsys2019_deeplearning_evaluation_b200.graph import scaled_inputs
    nu, ni, d = SHAPES[shape][:3]
    X = synth_urm(nu, ni, d, seed=3, values=values, popularity=0.8)
    Pui, A, B = scaled_inputs(X, alpha, beta)
    targets = _targets(X, B, n_random=150, seed=1)
    P = p3_sparse_rows(X, alpha, beta, rows=targets)
    tol = _tol(X, alpha, beta)[targets]
    K = 100
    h = Scaled(Pui, A, B, K)
    try:
        label = "%s alpha=%g beta=%g %s" % (values, alpha, beta, shape)
        _assert_route(h.route, ni, label, *SHAPES[shape][3:])
        _check_rows_tol(label, h.rows(targets), P, targets, K, tol)
        h.set_cap(K + CAP_SLACK)
        _check_rows_tol(label + " cap=K+%d" % CAP_SLACK, h.rows(targets, one_by_one=True), P, targets, K, tol)
    finally:
        h.close()


# ------------------------------------------------------------------------------------------------ W_sparse end to end


def _kth(line, other, val, n, K):
    """Per line the K-th largest value (ties by the other index), 0 where the line holds at most K values."""
    _, rank = _line_order(line, other, val)
    kth = np.zeros(n)
    sel = rank == K - 1
    kth[line[sel]] = val[sel]
    kth[np.bincount(line, minlength=n) <= K] = 0.0
    return kth


def _check_w(label, W, P, K, normalize, tol):
    """W_sparse against the fp64 restatement built from the full rows P (row i = item i): the row top-K, the optional
    row L1 normalisation, the column top-K.  Shared entries agree within the bound of their row (doubled, plus one
    rounding, after the normalisation).  An entry on one side only must be a near-tie of its row's top-K or of its
    column's top-K, or sit in a column that lost or gained a row near-tie (which moves that column's boundary by one)."""
    if normalize:  # the quotient of two values within tol, rounded to fp32
        tol = 2 * tol + U
    R = sparse_row_topk(P, K)
    Rn = _row_norm(R) if normalize else R
    Wref = sps.csr_matrix(sparse_column_topk(Rn, K), dtype=np.float64)
    W = sps.csr_matrix(W, dtype=np.float64)
    n = W.shape[0]
    Pc, Rc = P.tocoo(), Rn.tocoo()
    row_kth, col_kth = _kth(Pc.row, Pc.col, Pc.data, n, K), _kth(Rc.col, Rc.row, Rc.data, n, K)
    both = sps.csr_matrix(W.multiply(Wref.astype(bool)))
    ref = sps.csr_matrix(Wref.multiply(W.astype(bool)))
    for M in (both, ref):
        M.sort_indices()
    assert np.array_equal(both.indptr, ref.indptr) and np.array_equal(both.indices, ref.indices)
    both, ref = both.tocoo(), ref.data
    bad = np.abs(both.data - ref) > tol[both.row] * np.abs(ref)
    if bad.any():
        k = int(np.argmax(bad))
        pytest.fail("%s: %d values off, the first at (%d, %d): %r, fp64 %r" % (
            label, int(bad.sum()), both.row[k], both.col[k], both.data[k], ref[k]))
    only = (W.astype(bool) != Wref.astype(bool)).tocoo()
    if only.nnz == 0:
        return 0
    i, j = only.row, only.col
    p = np.asarray(P[i, j]).ravel()
    rn = np.asarray(Rn[i, j]).ravel()
    row_tie = (row_kth[i] > 0) & (np.abs(p - row_kth[i]) <= tol[i] * row_kth[i])
    col_tie = (col_kth[j] > 0) & (np.abs(rn - col_kth[j]) <= 2 * tol.max() * col_kth[j])
    moved = np.isin(j, j[row_tie])
    unexplained = ~(row_tie | col_tie | moved)
    if unexplained.any():
        k = int(np.argmax(unexplained))
        pytest.fail("%s: %d entries on one side only without a near-tie, the first at (%d, %d): fp64 %r (row K-th %r)" % (
            label, int(unexplained.sum()), i[k], j[k], p[k], row_kth[i[k]]))
    return int(only.nnz)


@pytest.fixture(scope="module")
def fit_urm():
    X = synth_urm(6000, 60000, 0.0003, seed=19, values="continuous")
    return X


@pytest.mark.parametrize("cls,alpha,beta", [("P3alpha", 0.8, 0.0), ("RP3beta", 1.0, 0.6)])
@pytest.mark.parametrize("normalize", [False, True])
def test_fit_several_windows(fit_urm, cls, alpha, beta, normalize):
    """P3alphaRecommender / RP3betaRecommender.fit(topK=100) on 60 000 items (two windows of the scaled handle) against
    p3_similarity_sparse's steps in fp64."""
    from recsys2019_deeplearning_evaluation_b200 import recommenders as R
    from recsys2019_deeplearning_evaluation_b200.graph import scaled_inputs
    X = fit_urm
    n = X.shape[1]
    Pui, A, B = scaled_inputs(X, alpha, beta)
    h = Scaled(Pui, A, B, 100)
    _assert_route(h.route, n, "%s fit" % cls, 2)
    h.close()
    r = R.P3alphaRecommender(X) if cls == "P3alpha" else R.RP3betaRecommender(X)
    kw = dict(topK=100, alpha=alpha, normalize_similarity=normalize)
    if cls == "RP3beta":
        kw["beta"] = beta
    r.fit(**kw)
    W = r.W_sparse
    assert sps.isspmatrix_csr(W) and W.dtype == np.float32 and W.shape == (n, n)
    assert (np.diff(W.tocsc().indptr) <= 100).all() and W.diagonal().sum() == 0 and W.nnz > 0
    _check_w("%s normalize=%s" % (cls, normalize), W, p3_sparse_rows(X, alpha, beta), 100, normalize, _tol(X, alpha, beta))


# ------------------------------------------------------------------------------------------------ topK above 2048

N_DENSE = 3000
DENSE_CASES = [("P3alpha", "continuous", False, 2049, None), ("RP3beta", "ratings", True, 2500, 700),
               ("P3alpha", "ratings", False, N_DENSE - 1, 1500), ("RP3beta", "continuous", True, N_DENSE, None),
               ("RP3beta", "continuous", False, 10 ** 6, 1)]


@pytest.fixture(scope="module")
def dense_urm():
    cache = {}

    def get(values):
        if values not in cache:
            cache[values] = synth_urm(2500, N_DENSE, 0.04, seed=27, values=values)
        return cache[values]
    return get


@pytest.mark.parametrize("cls,values,normalize,topK,slab_rows", DENSE_CASES)
def test_topk_beyond_the_selection_buffer(dense_urm, monkeypatch, cls, values, normalize, topK, slab_rows):
    """topK > 2048 goes through the dense mode of the scaled handle, slab by slab (slab_rows targets per slab where set,
    the last slab partial), and the dense mode-1 row selection; W_sparse against the dense fp64 oracle."""
    from recsys2019_deeplearning_evaluation_b200 import graph
    from recsys2019_deeplearning_evaluation_b200 import recommenders as R
    X = dense_urm(values)
    n = X.shape[1]
    if slab_rows is not None:
        monkeypatch.setattr(graph, "DENSE_SLAB_CELLS", slab_rows * n)
    alpha, beta = (0.9, 0.0) if cls == "P3alpha" else (1.1, 0.4)
    r = R.P3alphaRecommender(X) if cls == "P3alpha" else R.RP3betaRecommender(X)
    kw = dict(topK=topK, alpha=alpha, normalize_similarity=normalize)
    if cls == "RP3beta":
        kw["beta"] = beta
    r.fit(**kw)
    W = r.W_sparse
    K = min(topK, n)
    assert sps.isspmatrix_csr(W) and W.dtype == np.float32 and W.shape == (n, n)
    assert (np.diff(W.tocsc().indptr) <= K).all() and W.diagonal().sum() == 0
    P = sps.csr_matrix(p3_dense_rows(X, alpha, beta))  # the dense oracle's rows before any top-K
    assert np.diff(P.indptr).max() > 2048  # the row selection is not trivial
    # with K = n nothing is selected: _check_w then admits no entry on one side only
    _check_w("%s %s normalize=%s topK=%d" % (cls, values, normalize, topK), W, P, K, normalize, _tol(X, alpha, beta))
