"""-m gpu: the dense mode of the similarity kernel (b200_sim_compute_dense_device) at the catalogue sizes where it runs
on packed 16-bit counters or on several accumulator windows, against fp64 references.

The in-place EASE_R fit and gram_csr_device (the sparse SLIM ElasticNet fit) build X^T X with it, EASE_GRAM_SLAB_ROWS
target columns per call, on a handle created with a token topK of 1 (a 2048-slot candidate buffer); ItemKNN with
topK > 2048 and Compute_Similarity_Cython(topK=0) take the same branch.  What the candidate buffer and the staging area
leave of the shared memory holds about 50 500 accumulator words per window, so the branch depends on the catalogue:

    binary, up to ~50 500 items                     32-bit counters, one window
    binary, ~50 500 to ~101 000 items               packed 16-bit counters, one window
    binary, beyond ~101 000 items                   packed, two or more windows
    binary, a column of 32 768 users or more        32-bit counters (a count could reach 0x8000), two or more windows
    valued, beyond ~50 500 items                    fp32 accumulators, two or more windows

Every case first asserts the route it claims to test, as b200_sim_info reads it (n_windows, window_cells and
binary_path: 2 packed, 1 32-bit, 0 valued), so that a threshold that moves fails here instead of quietly testing
another branch.  The route of each handle is printed (run with -s to see it)."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import elasticnet_oracle
from oracle.similarity_oracle import SimilarityOracle, check_topk_against_dense
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

PACKED, INT32, VALUED = 2, 1, 0
RTOL = 1e-4
SLAB = 1024  # recommenders.EASE_GRAM_SLAB_ROWS, asserted in test_gram_slabs_exact


def _set_columns(X, cols, n_users):
    """Binary X with the columns `cols` holding exactly the users 0 .. n_users - 1."""
    mask = np.ones(X.shape[1], np.float32)
    mask[cols] = 0
    X = sps.csr_matrix(X @ sps.diags(mask))
    X.eliminate_zeros()
    rows = np.tile(np.arange(n_users), len(cols))
    full = sps.csr_matrix((np.ones(len(rows), np.float32), (rows, np.repeat(cols, n_users))), shape=X.shape)
    X = sps.csr_matrix(X + full, dtype=np.float32)
    X.sort_indices()
    return X


COLD_ITEM = 12345

URMS = {
    "binary_56k": lambda: synth_urm(30_000, 56_000, 0.001, seed=42, values="binary"),
    "binary_120k": lambda: synth_urm(20_000, 120_000, 0.0004, seed=8, values="binary"),
    "ratings_120k": lambda: synth_urm(20_000, 120_000, 0.0004, seed=8, values="ratings"),
    # one column of 32 768 users: no 16-bit counter may hold its count
    "long_column_60k": lambda: _set_columns(synth_urm(40_000, 60_000, 0.0005, seed=5), [7], 32_768),
    # two columns of the same 32 767 users: their shared count is 0x7FFF, the largest a packed half-word holds
    "count_7fff_56k": lambda: _set_columns(synth_urm(33_000, 56_000, 0.0005, seed=6), [2, 1001], 32_767),
    # binary_56k with an item nobody rated
    "binary_56k_cold": lambda: _set_columns(synth_urm(30_000, 56_000, 0.001, seed=42, values="binary"), [COLD_ITEM], 0),
}

# name -> (least n_windows, most n_windows or None, binary_path) of its Gram handle
GRAM_ROUTES = {
    "binary_56k": (1, 1, PACKED),
    "binary_56k_cold": (1, 1, PACKED),
    "binary_120k": (2, None, PACKED),
    "ratings_120k": (3, None, VALUED),
    "long_column_60k": (2, None, INT32),
    "count_7fff_56k": (1, 1, PACKED),
}


class _Urm:
    def __init__(self, name):
        self.name = name
        self.X = URMS[name]()
        self.X64 = sps.csr_matrix(self.X, dtype=np.float64)
        self.C64 = self.X64.tocsc()
        self.values = "binary" if (self.X.data == 1).all() else "ratings"


@pytest.fixture(scope="module")
def urm():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _Urm(name)
        return cache[name]
    return get


def _gram_sim(X):
    """The handle recommenders.py builds for X^T X (normalize=False, shrink=0, topK = n_items > 2048: dense mode)."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    n = X.shape[1]
    return Compute_Similarity_Cython(X, shrink=0, topK=n, normalize=False, similarity="cosine")


@pytest.fixture(scope="module")
def gram_sim(urm):
    """Gram handles by URM name; pack=False sets B200REC_NO_PACK (32-bit counters on the binary path) while it is built."""
    cache = {}

    def get(name, pack=True):
        if (name, pack) not in cache:
            if not pack:
                os.environ["B200REC_NO_PACK"] = "1"
            try:
                cache[(name, pack)] = _gram_sim(urm(name).X)
            finally:
                os.environ.pop("B200REC_NO_PACK", None)
        return cache[(name, pack)]
    yield get
    for sim in cache.values():
        sim._dealloc()


def _route(sim):
    from recsys2019_deeplearning_evaluation_b200 import _lib
    bp = ctypes.c_int32()
    _lib.check(_lib.load().b200_sim_info(sim._h, None, None, None, ctypes.byref(bp), None))
    return sim.n_windows, sim.window_cells, bp.value


def _assert_route(route, n_items, label, least, most, binary_path):
    n_win, cells, bp = route
    print("%s: n_items=%d n_windows=%d window_cells=%d binary_path=%d" % (label, n_items, n_win, cells, bp))
    assert bp == binary_path, (label, route)
    assert n_win >= least and (most is None or n_win <= most), (label, route)
    assert n_win * cells >= n_items and (n_win == 1) == (cells >= n_items), (label, route)


@pytest.fixture
def created_routes(monkeypatch):
    """Routes of every Compute_Similarity_Cython handle the code under test creates (recommenders.py imports the class
    when it builds the Gram matrix)."""
    from recsys2019_deeplearning_evaluation_b200 import similarity
    routes = []

    class Spy(similarity.Compute_Similarity_Cython):
        def __init__(self, *args, **kw):
            super(Spy, self).__init__(*args, **kw)
            routes.append(_route(self))
    monkeypatch.setattr(similarity, "Compute_Similarity_Cython", Spy)
    return routes


def _slabs(n):
    """[0, SLAB), an interior slab, the last (partial) slab ending at n, and a one-column slab."""
    mid = n // 2 // SLAB * SLAB
    return [(0, SLAB), (mid, mid + SLAB), ((n - 1) // SLAB * SLAB, n), (n // 3, n // 3 + 1)]


def _assert_slab_exact(S, d, lo, hi):
    """The whole slab, zeros included: S[t, j] == (X^T X)[lo + t, j] for every neighbour j, the target's own cell 0.
    Binary and integer-rating dot products are exact in fp32 here, so the check is equality."""
    import torch
    assert S.shape == (hi - lo, d.X.shape[1]) and S.dtype == torch.float32
    nz = torch.nonzero(S)  # row-major, like a CSR with sorted indices
    got_r, got_c = nz[:, 0].cpu().numpy(), nz[:, 1].cpu().numpy()
    got_v = S[nz[:, 0], nz[:, 1]].cpu().numpy().astype(np.float64)
    R = sps.csr_matrix(d.C64[:, lo:hi].T @ d.X64)
    R.sort_indices()
    rows = np.repeat(np.arange(hi - lo), np.diff(R.indptr))
    keep = (R.indices != rows + lo) & (R.data != 0)
    ref_r, ref_c, ref_v = rows[keep], R.indices[keep], R.data[keep]
    label = "%s slab [%d, %d)" % (d.name, lo, hi)
    assert len(got_r) == len(ref_r), "%s: %d non-zero cells, reference %d" % (label, len(got_r), len(ref_r))
    moved = (got_r != ref_r) | (got_c != ref_c)
    if moved.any():
        k = int(np.argmax(moved))
        pytest.fail("%s: %d non-zero cells at the wrong place, the first at (%d, %d), reference (%d, %d)" % (
            label, int(moved.sum()), got_r[k], got_c[k], ref_r[k], ref_c[k]))
    bad = got_v != ref_v
    if bad.any():
        k = int(np.argmax(bad))
        pytest.fail("%s: %d cells differ, the first at (%d, %d): %r, reference %r" % (
            label, int(bad.sum()), got_r[k], got_c[k], got_v[k], ref_v[k]))


def _bits_equal(a, b):
    import torch
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------ Gram slabs, exact


@pytest.mark.parametrize("name", ["binary_56k", "binary_120k", "ratings_120k", "long_column_60k", "count_7fff_56k"])
def test_gram_slabs_exact(urm, gram_sim, name):
    """The slabs recommenders.py computes (normalize=False, shrink=0) against scipy's X^T X in fp64, exactly; a slab
    computed again after other slabs has the same bits (the handle caches the order of the last column range)."""
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_GRAM_SLAB_ROWS
    assert EASE_GRAM_SLAB_ROWS == SLAB
    d = urm(name)
    n = d.X.shape[1]
    sim = gram_sim(name)
    _assert_route(_route(sim), n, name, *GRAM_ROUTES[name])
    slabs = _slabs(n)
    first = sim.compute_dense_device(*slabs[0])
    _assert_slab_exact(first, d, *slabs[0])
    if name == "count_7fff_56k":
        assert float(first[2, 1001]) == float(first[1001, 2]) == 32767.0
    for lo, hi in slabs[1:]:
        _assert_slab_exact(sim.compute_dense_device(lo, hi), d, lo, hi)
    assert _bits_equal(sim.compute_dense_device(*slabs[0]), first)
    before = _lib.launch_count()
    empty = sim.compute_dense_device(n // 2, n // 2)
    assert empty.shape == (0, n) and _lib.launch_count() == before


def test_gram_slabs_unpacked_counters_match_packed(urm, gram_sim):
    """120 K binary items with 32-bit counters (B200REC_NO_PACK): three windows instead of two, the same bits."""
    d = urm("binary_120k")
    n = d.X.shape[1]
    packed, plain = gram_sim("binary_120k"), gram_sim("binary_120k", pack=False)
    _assert_route(_route(packed), n, "binary_120k", *GRAM_ROUTES["binary_120k"])
    _assert_route(_route(plain), n, "binary_120k B200REC_NO_PACK", 3, None, INT32)
    for k, (lo, hi) in enumerate(_slabs(n)):
        a = plain.compute_dense_device(lo, hi)
        if k == 0:
            _assert_slab_exact(a, d, lo, hi)
        assert _bits_equal(a, packed.compute_dense_device(lo, hi)), (lo, hi)


def test_a_smaller_handle_built_later_does_not_break_a_larger_one(urm):
    """Both handles launch the same packed kernel, the first with a larger window (60 000 cells against 56 000): the
    kernel's shared-memory limit must be this handle's at each launch, not the last built handle's."""
    big_urm, small_urm = urm("binary_120k"), urm("count_7fff_56k")
    big = _gram_sim(big_urm.X)
    small = _gram_sim(small_urm.X)
    try:
        rb, rs = _route(big), _route(small)
        _assert_route(rb, 120_000, "binary_120k", *GRAM_ROUTES["binary_120k"])
        _assert_route(rs, 56_000, "count_7fff_56k", *GRAM_ROUTES["count_7fff_56k"])
        assert rb[1] > rs[1]
        _assert_slab_exact(big.compute_dense_device(0, SLAB), big_urm, 0, SLAB)
        _assert_slab_exact(small.compute_dense_device(0, SLAB), small_urm, 0, SLAB)
    finally:
        big._dealloc()
        small._dealloc()


# ------------------------------------------------------------------------------------------------ every formula


def _row_weights(n_users):
    return np.random.default_rng(3).random(n_users).astype(np.float32) + 0.5


FORMULAS = {
    "cosine": dict(similarity="cosine", shrink=7),
    "cosine_no_normalize": dict(similarity="cosine", normalize=False, shrink=7),
    "asymmetric": dict(similarity="asymmetric", shrink=7, asymmetric_alpha=0.2),
    "jaccard": dict(similarity="jaccard", shrink=7),
    "dice": dict(similarity="dice", shrink=7),
    "tversky": dict(similarity="tversky", shrink=7, tversky_alpha=0.7, tversky_beta=1.3),
    "adjusted": dict(similarity="adjusted", shrink=7),
    "pearson": dict(similarity="pearson", shrink=7),
    "row_weights": dict(similarity="cosine", shrink=7, row_weights=True),
}
SET_FORMULAS = ("jaccard", "dice", "tversky")
CENTRED = ("adjusted", "pearson")
# centring binary data leaves every value 0: adjusted and pearson run on the ratings only
FORMULA_CASES = [("ratings_120k", f) for f in FORMULAS] + [("binary_120k", f) for f in FORMULAS if f not in CENTRED]


@pytest.mark.parametrize("name,formula", FORMULA_CASES)
def test_formulas_several_windows(urm, name, formula):
    """Every formula of the dense mode on 120 K items (two packed or three valued windows) against the fp64 oracle,
    every cell of two 128-column slabs.  Each cell is within RTOL of the oracle relative to the sum of the absolute
    terms of its dot product (normalised like the cell): that is the cell's own magnitude unless centred values
    cancel, where fp32 accumulation error is relative to the terms and not to their sum."""
    import copy
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    d = urm(name)
    n_users, n = d.X.shape
    kw = dict(FORMULAS[formula])
    if kw.pop("row_weights", False):
        kw["row_weights"] = _row_weights(n_users)
    sim = Compute_Similarity_Cython(d.X, topK=0, **kw)
    if formula in SET_FORMULAS or (d.values == "binary" and formula != "row_weights"):
        expect = (2, None, PACKED)  # set kinds binarise the data
    else:
        expect = (3, None, VALUED)
    _assert_route(_route(sim), n, "%s %s" % (name, formula), *expect)
    orc = SimilarityOracle(d.X, **kw)
    terms = None
    if formula in CENTRED:
        terms = copy.copy(orc)
        terms.X, terms.Xw_T = abs(orc.X), abs(orc.Xw_T)
    try:
        for lo, hi in ((0, 128), (n - 128, n)):
            got = sim.compute_dense_device(lo, hi).cpu().numpy().astype(np.float64)
            cols = np.arange(lo, hi)
            ref = orc.column_values(cols).T
            scale = np.abs(ref) if terms is None else terms.column_values(cols).T
            bad = np.abs(got - ref) > RTOL * scale
            if bad.any():
                t, j = np.unravel_index(int(np.argmax(bad)), bad.shape)
                pytest.fail("%s %s slab [%d, %d): %d cells off, the first at (%d, %d): %r, oracle %r" % (
                    name, formula, lo, hi, int(bad.sum()), lo + t, j, got[t, j], ref[t, j]))
            assert np.count_nonzero(ref) > 1000
    finally:
        sim._dealloc()


# ------------------------------------------------------------------------------------------------ topK beyond 2048


@pytest.fixture(scope="module")
def knn_urm():
    cache = {}

    def get(values):
        if values not in cache:
            cache[values] = synth_urm(3000, 8000, 0.02, seed=14, values=values)
        return cache[values]
    return get


TOPK_CASES = ([("continuous", "cosine", K) for K in (2048, 2049, 4000, 7999, 8000)]
              + [("continuous", "pearson", 7000), ("binary", "cosine", 2049)])


@pytest.mark.parametrize("values,kind,K", TOPK_CASES)
def test_topk_beyond_the_selection_buffer(knn_urm, values, kind, K):
    """topK = 2048 is the window kernel's top-K; above it the dense slab and b200_dense_topk_device (mode 1: zeros
    outrank negatives and are dropped) take over.  Each target has 4 400 to 6 500 neighbours among the 8 000 columns, so
    K = 4000 selects and K >= 7999 keeps every one; pearson at K = 7000 reaches past the zeros into the negatives."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    X = knn_urm(values)
    kw = dict(topK=K, shrink=10, similarity=kind)
    sim = Compute_Similarity_Cython(X, **kw)
    try:
        assert sim._dense_mode == (K > 2048) and sim.K == (1 if K > 2048 else K)
        W = sim.compute_similarity()
    finally:
        sim._dealloc()
    assert sps.isspmatrix_csr(W) and W.dtype == np.float32 and W.shape == (8000, 8000)
    assert (np.diff(W.tocsc().indptr) <= K).all() and W.diagonal().sum() == 0
    ties = check_topk_against_dense(W, SimilarityOracle(X, **kw), np.arange(0, 8000, 53), rtol=RTOL)
    if values == "continuous":
        assert ties == 0
    if kind == "pearson":
        assert (W.data < 0).any()


# ------------------------------------------------------------------------------------------------ recommenders


def test_gram_csr_several_windows(urm, created_routes):
    """gram_csr_device on 120 K binary items (two packed windows): the CSR equals scipy's X^T X without its diagonal --
    row pointers, column indices and values, exactly."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import gram_csr_device
    d = urm("binary_120k")
    n = d.X.shape[1]
    ptr, col, val = gram_csr_device(d.X)
    assert len(created_routes) == 1
    _assert_route(created_routes[0], n, "gram_csr_device binary_120k", *GRAM_ROUTES["binary_120k"])
    ptr = ptr.cpu().numpy()
    nnz = int(ptr[-1])
    col, val = col[:nnz].cpu().numpy(), val[:nnz].cpu().numpy()
    S = sps.csr_matrix(d.C64.T @ d.X64)
    S.sort_indices()
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(S.indptr))
    keep = S.indices != rows
    ref_ptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rows[keep], minlength=n), out=ref_ptr[1:])
    print("gram_csr_device binary_120k: nnz %d" % nnz)
    assert np.array_equal(ptr, ref_ptr)
    assert np.array_equal(col, S.indices[keep])
    assert np.array_equal(val.astype(np.float64), S.data[keep])


def _ease_columns(d, l2, cols):
    """fp64 columns of EASE_R's B: x solves (X^T X + l2 I) x = e_j by conjugate gradients, B[:, j] = x / -x[j] with
    B[j, j] = 0."""
    from scipy.sparse.linalg import LinearOperator, cg
    n = d.X.shape[1]
    A = LinearOperator((n, n), matvec=lambda v: d.C64.T @ (d.X64 @ v) + l2 * v, dtype=np.float64)
    out = np.zeros((n, len(cols)))
    for k, j in enumerate(cols):
        e = np.zeros(n)
        e[j] = 1.0
        x, info = cg(A, e, rtol=1e-12, maxiter=1000)
        assert info == 0 and np.linalg.norm(A @ x - e) < 1e-10, (j, info)
        out[:, k] = x / -x[j]
        out[j, k] = 0.0
    return out


@pytest.mark.parametrize("l2,topK", [(50.0, None), (1e3, 100)])
def test_ease_inplace_on_a_packed_catalogue(urm, created_routes, monkeypatch, l2, topK):
    """56 000 binary items: the default path needs about 88 GB, so fit() goes in place by itself and builds X^T X from
    packed-counter slabs.  Columns 0, n/2, n - 1, the most popular item and an item nobody rated (whose row and column
    are exactly 0) against fp64 conjugate gradients, to 1e-4 of max|B[:, j]|; with topK=None the scores of a few users
    from the dense B on the device, with topK=100 the kept entries of each column."""
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200 import recommenders as R
    d = urm("binary_56k_cold")
    X = d.X
    n = X.shape[1]
    n_pad = -(-n // 128) * 128
    ws = ctypes.c_int64()
    _lib.check(_lib.load().b200_ease_inplace_workspace_bytes(n, ctypes.byref(ws)))
    need = 4 * n_pad * n_pad + int(ws.value) + 4 * SLAB * n + R.EASE_URM_COPIES * R.ease_urm_bytes(X)
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("the in-place EASE_R fit of %d items needs %d bytes of device memory, %d are free" % (n, need, free))
    assert R.ease_inplace_for_device(n, free, R.ease_urm_bytes(X))
    captured = []
    fit_inplace = R.EASE_R_Recommender._fit_inplace

    def spy(self, *args):
        captured.append(fit_inplace(self, *args))
        return captured[-1]
    monkeypatch.setattr(R.EASE_R_Recommender, "_fit_inplace", spy)
    r = R.EASE_R_Recommender(X, verbose=False)
    r.fit(topK=topK, l2_norm=l2, verbose=False)
    assert len(captured) == 1, "the in-place path was not taken"
    assert len(created_routes) == 1
    _assert_route(created_routes[0], n, "EASE_R in place binary_56k_cold", *GRAM_ROUTES["binary_56k_cold"])
    B = captured.pop()
    cnt = np.diff(d.C64.indptr)
    assert cnt[COLD_ITEM] == 0
    cols = [0, n // 2, n - 1, int(np.argmax(cnt)), COLD_ITEM]
    ref = _ease_columns(d, l2, cols)
    got = B[:, torch.tensor(cols, device=B.device)].cpu().numpy().astype(np.float64)
    assert (got[:, -1] == 0).all() and float(B[COLD_ITEM].abs().max()) == 0.0
    for k, j in enumerate(cols[:-1]):
        err = np.abs(got[:, k] - ref[:, k]).max() / np.abs(ref[:, k]).max()
        assert got[j, k] == 0 and err < 1e-4, (j, err)
    if topK is None:
        users = np.arange(0, X.shape[0], 2999)
        sc = r._compute_item_score(users)[:, cols].astype(np.float64)
        ref_sc = d.X64[users] @ ref
        assert np.abs(sc - ref_sc).max() < 1e-4 * np.abs(ref_sc).max()
    else:
        W = r.W_sparse.tocsc()
        for k, j in enumerate(cols):  # mode 0 (similarityMatrixTopK): the topK largest non-zero values, ties by index
            b = got[:, k]
            nz = np.flatnonzero(b)
            top = np.sort(nz[np.lexsort((nz, -b[nz]))][:topK])
            assert np.array_equal(W.indices[W.indptr[j]:W.indptr[j + 1]], top), j
            assert np.array_equal(W.data[W.indptr[j]:W.indptr[j + 1]], b[top].astype(np.float32)), j
    del B


def test_slim_enet_sparse_path_several_windows(urm, created_routes, monkeypatch):
    """120 K binary items: the dense path's footprint (above 115 GB) does not fit, so fit() solves against the sparse Gram
    matrix by itself, built from two packed windows.  A few items against the fp64 oracle on their support."""
    import torch
    from recsys2019_deeplearning_evaluation_b200 import recommenders as R
    d = urm("binary_120k")
    X = d.X
    n_users, n = X.shape
    l1_ratio, alpha, topK = 0.1, 1e-4, 20
    torch.cuda.empty_cache()
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    assert R.slim_enet_dense_bytes(n, topK, sms, R.ease_urm_bytes(X)) > torch.cuda.mem_get_info()[0]
    called = []
    fit_sparse = R.SLIMElasticNetRecommender._fit_sparse

    def spy(self, *args):
        called.append(1)
        return fit_sparse(self, *args)
    monkeypatch.setattr(R.SLIMElasticNetRecommender, "_fit_sparse", spy)
    r = R.SLIMElasticNetRecommender(X, verbose=False)
    r.fit(l1_ratio=l1_ratio, alpha=alpha, positive_only=True, topK=topK)
    assert called, "the sparse path was not taken"
    assert len(created_routes) == 1
    _assert_route(created_routes[0], n, "SLIM ElasticNet sparse binary_120k", *GRAM_ROUTES["binary_120k"])
    W = r.W_sparse.tocsc()
    cnt = np.diff(d.C64.indptr)
    for j in (0, n // 2, n - 1, int(np.argmax(cnt))):
        g = np.asarray((d.C64.T @ d.C64[:, j]).todense()).ravel()
        support = np.flatnonzero(g)
        support = support[support != j]
        Xs = d.C64[:, support]
        Gs = (Xs.T @ Xs).toarray()  # the oracle on the support: the other coordinates never act
        w, _, _ = elasticnet_oracle.enet_cd_gram(Gs, g[support], g[j], alpha * l1_ratio * n_users,
                                                 alpha * (1 - l1_ratio) * n_users, True)
        full = np.zeros(n)
        full[support] = w
        rows, vals = elasticnet_oracle.select_topk(full, topK)
        ref = np.zeros(n)
        ref[rows] = vals
        got = np.asarray(W[:, j].todense()).ravel()
        assert np.count_nonzero(ref) > 0 and np.abs(got - ref).max() < 2e-5, (j, float(np.abs(got - ref).max()))


# ------------------------------------------------------------------------------------------------ argument checks


def test_dense_mode_argument_checks():
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Euclidean
    X = synth_urm(300, 500, 0.02, seed=3, values="ratings")
    eu = Compute_Similarity_Euclidean(X, topK=5)
    with pytest.raises(ValueError, match="no dense output mode"):
        eu.compute_dense_device(0, 10)
    eu._dealloc()
    sim = _gram_sim(X)
    out = torch.zeros((600, 500), dtype=torch.float32, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for lo, hi in ((-1, 4), (5, 4), (0, 501), (501, 501)):
        with pytest.raises(ValueError, match="bad column range"):
            _lib.check(_lib.load().b200_sim_compute_dense_device(sim._h, lo, hi, out.data_ptr(), stream))
    assert float(out.abs().sum()) == 0.0
    sim._dealloc()
