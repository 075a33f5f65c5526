"""The device halves of the multi-GPU paths (recsys2019_deeplearning_evaluation_b200/dist.py), run on ONE GPU: every rank is
simulated in this process, each with its own handle or buffers, and the test does the collective's work itself (the sum of
an all-reduce, the rotation of the symmetric-memory tables).  tools/mgpu_*.py run the same paths with torch.distributed on
several GPUs.

  K1  item-sharded similarity: b200_sim_compute_peers_device writes every rank's columns into every rank's table
  K2  user-sharded BPR: the replicated-delta kernels (b200_mf_delta_*) and the user-shard Philox sampler
  K4  row-sharded IALS: the half epoch on a slice of the warm rows
  K5  user-sharded EASE_R Gram: _gram_device(rows=...)
-m gpu."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from k1d_util import force_k1c  # noqa: F401 (fixture)
from oracle.similarity_oracle import EuclideanOracle, SimilarityOracle, check_topk_against_dense
from recsys2019_deeplearning_evaluation_b200.dist import balanced_ranges
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu

SENT = 0x7FC0DEAD  # int32 sentinel: neither a column index, a count, nor (as fp32 bits, a NaN) a similarity


def _L():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------------
# K1: peer tables

def _layout(n, K, gapped):
    """(idx, val, cnt offsets, total length) of one table in int32 elements: dist.SymmetricTopKTable's packed layout, or one
    with a head, sentinel gaps between the regions and a tail."""
    if not gapped:
        return 0, n * K, 2 * n * K, 2 * n * K + n
    oi = 13
    ov = oi + n * K + 7
    oc = ov + n * K + 5
    return oi, ov, oc, oc + n + 11


def _peers(sim, lo, hi, tables, off, n_tables=None):
    arr = (ctypes.c_void_p * max(1, len(tables)))(*[t if t is None else t.data_ptr() for t in tables])
    _L().check(_L().load().b200_sim_compute_peers_device(sim._h, int(lo), int(hi), len(tables) if n_tables is None else n_tables,
                                                         arr, off[0], off[1], off[2], _stream()))


def _split(buf, n, K, off):
    import torch
    oi, ov, oc, _ = off
    idx = buf[oi:oi + n * K].view(n, K)
    val = buf[ov:ov + n * K].view(torch.float32).view(n, K)
    cnt = buf[oc:oc + n]
    return idx, val, cnt


def _outside_mask(n, K, off):
    """True for every element of a table buffer that lies outside the idx / val / cnt regions."""
    oi, ov, oc, total = off
    m = np.ones(total, bool)
    m[oi:oi + n * K] = False
    m[ov:ov + n * K] = False
    m[oc:oc + n] = False
    return m


def _sorted_rows(idx, val, cnt):
    """Per row the (idx, val) pairs of slots < cnt sorted by idx (slot order is unspecified); checks slots >= cnt hold -1 / 0."""
    K = idx.shape[1]
    used = np.arange(K)[None, :] < cnt[:, None]
    assert (idx[~used] == -1).all() and (val[~used].view(np.int32) == 0).all()
    key = np.where(used, idx.astype(np.int64), np.iinfo(np.int64).max)
    order = np.argsort(key, axis=1, kind="stable")
    return np.take_along_axis(idx, order, 1), np.take_along_axis(val, order, 1)


def _reference(sim):
    tab = sim.compute_topk_device(0, sim.n_columns)
    return tab.idx.cpu().numpy(), tab.val.cpu().numpy(), tab.cnt.cpu().numpy()


def _k1c(sim, fail_every=-1):
    en, nb, nw = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    _L().check(_L().load().b200_sim_debug_k1c(sim._h, fail_every, ctypes.byref(en), None, ctypes.byref(nb), ctypes.byref(nw)))
    return en.value, nb.value, nw.value


def _phase_cycles(sim, fn):
    L = _L().load()
    _L().check(L.b200_sim_debug_phase_cycles(sim._h, 1, None))
    fn()
    out = (ctypes.c_uint64 * 16)()
    _L().check(L.b200_sim_debug_phase_cycles(sim._h, 0, out))
    return np.array(list(out), dtype=np.float64)


def _check_work(sim, X):
    """column_work() / b200_sim_work: per column the sum of the profile lengths of its users."""
    Xs = sps.csr_matrix((np.ones(X.nnz, np.int64), X.indices, X.indptr), shape=X.shape)
    work = np.asarray(Xs.T @ np.diff(X.indptr).astype(np.int64)).ravel()
    assert np.array_equal(sim.column_work(), work)
    n = X.shape[1]
    for lo, hi in ((0, n), (0, 0), (n // 3, n // 3 + 1), (n // 5, n - 1)):
        assert sim.gathered_entries(lo, hi) == int(work[lo:hi].sum())
    return work


def _run_world(sims, world, n, K, off, route_check=None):
    """Rank r of `world` calls the peers kernel on its balanced range with its own table first; returns the world's
    buffers (host int32) after every rank's call."""
    import torch
    bounds = balanced_ranges(sims[0].column_work(), world)
    assert bounds[0] == 0 and bounds[-1] == n and (np.diff(bounds) >= 0).all()
    bufs = [torch.full((off[3],), SENT, dtype=torch.int32, device="cuda") for _ in range(world)]
    for r in range(world):
        tables = [bufs[r]] + [bufs[q] for q in range(world) if q != r]
        _peers(sims[r], bounds[r], bounds[r + 1], tables, off)
        if route_check is not None and bounds[r + 1] > bounds[r]:
            route_check(sims[r])
    torch.cuda.synchronize()
    return [b.cpu().numpy() for b in bufs], bounds


def _exact(a, b):
    return np.array_equal(a.view(np.int32), b.view(np.int32))


def _check_peer_route(make, X, exact, route_check=None, oracle=None, worlds=(2, 3, 8)):
    """Every world size, both layouts: identical tables, cnt and per-row pairs of the full-range compute_device call, no
    sentinel inside, untouched gaps; then one rank alone and an empty range."""
    import torch
    sims = [make() for _ in range(max(worlds))]
    ref = make()
    _check_work(ref, X)
    n, K = ref.n_columns, ref.K
    r_idx, r_val, r_cnt = _reference(ref)
    r_si, r_sv = _sorted_rows(r_idx, r_val, r_cnt)
    for gapped in (False, True):
        off = _layout(n, K, gapped)
        outside = _outside_mask(n, K, off)
        for world in worlds:
            bufs, bounds = _run_world(sims, world, n, K, off, route_check)
            for b in bufs[1:]:
                assert np.array_equal(b, bufs[0]), "world %d: the tables differ" % world
            b = bufs[0]
            assert (b[outside] == SENT).all(), "world %d: a write outside the table" % world
            assert (b[~outside] != SENT).all(), "world %d: a row was not written" % world
            idx, val, cnt = (a.cpu().numpy() for a in _split(torch.from_numpy(b), n, K, off))
            assert np.array_equal(cnt, r_cnt)
            si, sv = _sorted_rows(idx, val, cnt)
            assert np.array_equal(si, r_si)
            if exact:
                assert _exact(sv, r_sv)
            else:  # the valued accumulators add fp32 products with shared-memory atomics: no fixed order of the sums
                assert np.allclose(sv, r_sv, rtol=1e-5, atol=1e-6), float(np.abs(sv - r_sv).max())
        # one rank alone: rows outside its range keep the sentinel
        bounds = balanced_ranges(ref.column_work(), 3)
        lo, hi = int(bounds[1]), int(bounds[2])
        assert hi > lo
        bufs = [torch.full((off[3],), SENT, dtype=torch.int32, device="cuda") for _ in range(2)]
        _peers(sims[1], lo, hi, bufs, off)
        torch.cuda.synchronize()
        for b in bufs:
            bb = b.cpu().numpy()
            idx, val, cnt = (a.cpu().numpy() for a in _split(torch.from_numpy(bb), n, K, off))
            out_rows = np.ones(n, bool)
            out_rows[lo:hi] = False
            assert (idx[out_rows] == SENT).all() and (val[out_rows].view(np.int32) == SENT).all() and (cnt[out_rows] == SENT).all()
            assert (idx[lo:hi] != SENT).all() and np.array_equal(cnt[lo:hi], r_cnt[lo:hi])
            assert (bb[outside] == SENT).all()
        # an empty range writes nothing
        bufs = [torch.full((off[3],), SENT, dtype=torch.int32, device="cuda") for _ in range(2)]
        _peers(sims[0], 5, 5, bufs, off)
        torch.cuda.synchronize()
        assert all(bool((b == SENT).all()) for b in bufs)
    if oracle is not None:
        from recsys2019_deeplearning_evaluation_b200.similarity import topk_table_to_csr
        off = _layout(n, K, False)
        bufs, _ = _run_world(sims, 3, n, K, off)
        idx, val, cnt = _split(torch.from_numpy(bufs[0]).cuda(), n, K, off)
        W = topk_table_to_csr(n, K, idx.contiguous(), val.contiguous(), cnt.contiguous())
        cols = np.unique(np.linspace(0, n - 1, 200).astype(np.int64))
        check_topk_against_dense(W, oracle, cols, rtol=1e-4)
    return sims, ref


def _sim(X, **kw):
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    return Compute_Similarity_Cython(X, **kw)


def test_peers_valued_one_window():
    X = synth_urm(3000, 1500, 0.03, seed=21, values="continuous")
    kw = dict(topK=30, shrink=5, similarity="cosine")
    sims, ref = _check_peer_route(lambda: _sim(X, **kw), X, exact=False, oracle=SimilarityOracle(X, **kw))
    assert ref.n_windows == 1 and not ref.binary_path and not ref.signed_data


def test_peers_valued_several_windows():
    X = synth_urm(20_000, 120_000, 0.0004, seed=8, values="continuous")
    kw = dict(topK=20, shrink=10, similarity="cosine")
    sims, ref = _check_peer_route(lambda: _sim(X, **kw), X, exact=False, oracle=SimilarityOracle(X, **kw), worlds=(2, 3))
    assert ref.n_windows >= 2 and not ref.binary_path


@pytest.mark.parametrize("pack", [True, False])
def test_peers_binary_counter_widths(pack, monkeypatch):
    """The window kernel's binary path, 16-bit packed counters and (B200REC_NO_PACK) 32-bit ones; the K1-D kernel is switched
    off so that every column goes through it."""
    monkeypatch.setenv("B200REC_K1C", "0")
    if not pack:
        monkeypatch.setenv("B200REC_NO_PACK", "1")
    X = synth_urm(10_000, 60_000, 0.001, seed=42, values="binary")
    kw = dict(topK=60, shrink=20, similarity="cosine")

    def route(sim):
        en, nb, _ = _k1c(sim)
        assert en == 0 and nb == 0

    sims, ref = _check_peer_route(lambda: _sim(X, **kw), X, exact=True, route_check=route, worlds=(2, 3))
    bp = ctypes.c_int32()
    _L().check(_L().load().b200_sim_info(ref._h, None, None, None, ctypes.byref(bp), None))
    assert bp.value == (2 if pack else 1)


def test_peers_signed_negatives_fill_the_slots():
    """pearson with K = n - 1 on dense-ish ratings: zeros run out and the negative pass fills the remaining slots."""
    X = synth_urm(300, 40, 0.5, seed=4, values="ratings")
    kw = dict(topK=39, shrink=0, similarity="pearson")
    sims, ref = _check_peer_route(lambda: _sim(X, **kw), X, exact=False, oracle=SimilarityOracle(X, **kw))
    assert ref.signed_data
    _, r_val, _ = _reference(ref)
    assert (r_val < 0).any()


def test_peers_candidate_overflow_rescan():
    X = synth_urm(3000, 1500, 0.03, seed=21, values="continuous")
    kw = dict(topK=30, shrink=5, similarity="cosine")

    def make():
        s = _sim(X, **kw)
        _L().check(_L().load().b200_sim_debug_set_cap(s._h, 40))
        return s

    _check_peer_route(make, X, exact=False, oracle=SimilarityOracle(X, **kw))



def test_peers_k1d_with_redo(force_k1c):
    """K1-D on every column, every 4th local column handed back to the window kernel: one peers call runs both kernels."""
    X = synth_urm(20_000, 3_000, 0.004, seed=31, values="binary")
    kw = dict(topK=50, shrink=5, similarity="cosine")

    def make():
        s = _sim(X, **kw)
        assert _k1c(s, fail_every=4)[0] == 1
        return s

    def route(sim):
        en, nb, nw = _k1c(sim)
        assert en == 1 and nb > 0 and nw > 0, (en, nb, nw)

    _check_peer_route(make, X, exact=True, route_check=route)


def test_peers_euclidean():
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Euclidean
    X = synth_urm(500, 300, 0.03, seed=12, values="continuous")
    kw = dict(topK=20, shrink=1, normalize=False, similarity_from_distance_mode="lin")
    _check_peer_route(lambda: Compute_Similarity_Euclidean(X, **kw), X, exact=False, oracle=EuclideanOracle(X, **kw))


def _uniform():
    # the pair path's shape in tests/test_k1d_pairs_gpu.py: counts ~ Poisson(0.8), ~400 users per column
    return synth_urm(200_000, 2_000, 0.002, seed=7, values="binary")


def test_peers_call_never_takes_the_pair_path(force_k1c):
    """A pair-path-eligible handle: compute_device over the full range takes the pair path; the peers call over the same range
    with two tables does not (phase counters 8..11 stay zero) and still writes the identical table into both.  With a
    single table there is nobody to write to but the caller, and the peers call may take the pair path: same table."""
    import torch
    X = _uniform()
    kw = dict(topK=50, shrink=5, similarity="cosine")
    ref = _sim(X, **kw)
    cyc = _phase_cycles(ref, lambda: _reference(ref))
    assert cyc[8] > 0 and cyc[11] > 0
    r_idx, r_val, r_cnt = _reference(ref)
    n, K = ref.n_columns, ref.K
    for n_tables in (2, 1):
        sim = _sim(X, **kw)
        off = _layout(n, K, True)
        bufs = [torch.full((off[3],), SENT, dtype=torch.int32, device="cuda") for _ in range(n_tables)]
        cyc = _phase_cycles(sim, lambda: _peers(sim, 0, n, bufs, off))
        if n_tables > 1:
            assert cyc[8:12].sum() == 0, cyc[8:12]
        for b in bufs:
            idx, val, cnt = (a.cpu().numpy() for a in _split(b, n, K, off))
            assert np.array_equal(cnt, r_cnt)
            si, sv = _sorted_rows(idx, val, cnt)
            ri, rv = _sorted_rows(r_idx, r_val, r_cnt)
            assert np.array_equal(si, ri) and _exact(sv, rv)
            assert (b.cpu().numpy()[_outside_mask(n, K, off)] == SENT).all()


def test_peers_argument_rules():
    import torch
    X = synth_urm(500, 120, 0.05, seed=3, values="continuous")
    sim = _sim(X, topK=10, similarity="cosine")
    n, K = sim.n_columns, sim.K
    off = _layout(n, K, False)
    bufs = [torch.full((off[3],), SENT, dtype=torch.int32, device="cuda") for _ in range(9)]
    with pytest.raises(ValueError):
        _peers(sim, 0, n, [], off, n_tables=0)
    with pytest.raises(ValueError):
        _peers(sim, 0, n, bufs, off)  # 9 tables
    with pytest.raises(ValueError):
        _peers(sim, 0, n, [bufs[0], None], off)
    for lo, hi in ((-1, 5), (10, 5), (0, n + 1)):
        with pytest.raises(ValueError):
            _peers(sim, lo, hi, bufs[:2], off)
    torch.cuda.synchronize()
    assert all(bool((b == SENT).all()) for b in bufs)


# ---------------------------------------------------------------------------------------------------------------------
# K2: replicated-delta exchange kernels

def _f32(t):
    return t.detach().cpu().numpy().astype(np.float32, copy=True)


@pytest.mark.parametrize("n,world", [(4, 2), (4 * 1237, 3), ((1 << 20) + 12, 2)])
def test_delta_exchange_kernels_and_overlapped_schedule(n, world):
    """Every kernel output bitwise equal to numpy's fp32 element-wise operations; over the overlapped schedule (the apply of
    exchange k runs at exchange k + 1, after the next epoch's movement; flush at the end) every replica ends at the initial
    table plus every replica's movement."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.dist import ReplicatedDeltaExchange
    rng = np.random.default_rng(n)
    V0 = rng.standard_normal(n).astype(np.float32)
    reps = [ReplicatedDeltaExchange(torch.from_numpy(V0.copy()).cuda()) for _ in range(world)]
    moved = np.zeros(n, np.float64)
    pending = False

    def apply_all():
        for x in reps:
            V, B, s, o = _f32(x.V), _f32(x.B), _f32(x.sum), _f32(x.own)
            x._apply()
            t = s - o
            assert _exact(_f32(x.V), V + t) and _exact(_f32(x.B), B + t)
            assert _exact(_f32(x.sum), s) and _exact(_f32(x.own), o)

    for step in range(4):
        for x in reps:  # this epoch's training
            m = (rng.standard_normal(n) * 10.0 ** rng.integers(-4, 0)).astype(np.float32)
            m[rng.random(n) < 0.3] = 0.0
            x.V.add_(torch.from_numpy(m).cuda())
            moved += m.astype(np.float64)
        if pending:
            apply_all()
        for x in reps:
            V, B = _f32(x.V), _f32(x.B)
            x._snapshot()
            own = V - B
            assert _exact(_f32(x.own), own) and _exact(_f32(x.sum), own) and _exact(_f32(x.B), V) and _exact(_f32(x.V), V)
        total = sum(x.sum.clone() for x in reps)  # the all-reduce
        for x in reps:
            x.sum.copy_(total)
        pending = True
    apply_all()  # flush
    ref = V0.astype(np.float64) + moved
    got = [_f32(x.V).astype(np.float64) for x in reps]
    tol = 64 * np.finfo(np.float32).eps * (np.abs(ref) + 1.0)  # a few fp32 roundings per step and replica
    for g in got:
        assert (np.abs(g - ref) <= tol).all(), float(np.abs(g - ref).max())
        assert (np.abs(g - got[0]) <= tol).all()


def test_delta_exchange_argument_rules():
    import torch
    L = _L().load()
    t = [torch.arange(8, dtype=torch.float32, device="cuda") + k for k in range(4)]
    before = [x.clone() for x in t]
    _L().check(L.b200_mf_delta_snapshot_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 0, _stream()))
    _L().check(L.b200_mf_delta_apply_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), 0, _stream()))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(t, before))
    for n in (6, 5, -4):
        with pytest.raises(ValueError):
            _L().check(L.b200_mf_delta_snapshot_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), n, _stream()))
        with pytest.raises(ValueError):
            _L().check(L.b200_mf_delta_apply_device(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), n, _stream()))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(t, before))


# ---------------------------------------------------------------------------------------------------------------------
# K2: user-shard Philox sampler

N_USERS, N_ITEMS, LO, HI = 400, 60, 100, 300


def _shard_urm():
    """Ratings; inside and outside [LO, HI) some users have an empty profile and some have every item."""
    X = synth_urm(N_USERS, N_ITEMS, 0.1, seed=17, values="ratings").tolil()
    for u in (0, 5, 120, 121, 200, 299, 350):
        X[u, :] = 0
    for u in (1, 101, 150, 298, 399):
        X[u, :] = 3.0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    X.sort_indices()
    return X


def _mf(X, algo, **kw):
    from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch
    args = dict(algorithm_name=algo, n_factors=8, batch_size=8, learning_rate=0.03, random_seed=9, sgd_mode="adagrad",
                negative_interactions_quota=0.4, sampler="philox")
    args.update(kw)
    return MatrixFactorization_Cython_Epoch(X, **args)


def _draw(g, epochs=1):
    out = []
    for _ in range(epochs):
        g.epochIteration_Cython()
        out.append(g.get_samples())
    return [np.concatenate([s[k] for s in out]) for k in range(3)]


@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_user_shard_draws_only_eligible_shard_users(algo):
    X = _shard_urm()
    lens = np.diff(X.indptr)
    dense = X.toarray()
    g = _mf(X, algo, hogwild=True)
    g.set_user_shard(LO, HI, 0, stream_id=2)
    su, si, s3 = _draw(g, epochs=12)
    assert ((su >= LO) & (su < HI)).all()
    assert ((lens[su] > 0) & (lens[su] < N_ITEMS)).all()
    eligible = np.flatnonzero((lens > 0) & (lens < N_ITEMS))
    assert set(su.tolist()) == set(eligible[(eligible >= LO) & (eligible < HI)].tolist())
    if algo == "MF_BPR":
        assert (dense[su, si] != 0).all() and (dense[su, s3] == 0).all()
    else:
        pos = s3 != 0
        assert np.array_equal(dense[su[pos], si[pos]], s3[pos].astype(np.float32)) and (dense[su[~pos], si[~pos]] == 0).all()
        assert 0.3 < pos.mean() < 0.5


@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_user_shard_epoch_length(algo):
    X = _shard_urm()
    bs = 8
    ref_len = ((N_USERS if algo == "MF_BPR" else X.nnz) // bs + 1) * bs
    for spe, want in ((0, ref_len), (5, bs), (37, 32), (64, 64), (ref_len, ref_len)):
        g = _mf(X, algo, hogwild=True, batch_size=bs)
        g.set_user_shard(LO, HI, spe, stream_id=0)
        g.epochIteration_Cython()
        assert g.samples_last_epoch() == want == max(1, (spe or ref_len) // bs) * bs


def test_user_shard_streams():
    """Same seed and stream id: the same stream; another stream id: another stream; sharding a handle twice with stream id 1
    draws stream 1, not stream 2."""
    X = _shard_urm()

    def run(*stream_ids):
        g = _mf(X, "MF_BPR", hogwild=True)
        for s in stream_ids:
            g.set_user_shard(LO, HI, 0, stream_id=s)
        return _draw(g, epochs=2)

    a, b, c = run(1), run(1), run(0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert not np.array_equal(a[0], c[0])
    twice = run(1, 1)
    assert all(np.array_equal(x, y) for x, y in zip(a, twice))
    reset = run(3, 0)
    assert all(np.array_equal(x, y) for x, y in zip(c, reset))


@pytest.mark.parametrize("dataflow", ["1", "0"])
@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_user_shard_minibatch_replays_through_the_oracle(algo, dataflow, monkeypatch):
    from oracle.sgd_oracle import MFOracle
    monkeypatch.setenv("B200REC_MF_DATAFLOW", dataflow)
    X = _shard_urm()
    # plain SGD: the adaptive modes divide by the root of a per-coordinate cache, so an fp32-rounded small gradient becomes a
    # full-size step and single coordinates drift past 1e-4 of the fp64 oracle, sharded or not
    kw = dict(n_factors=24, batch_size=16, learning_rate=0.05, random_seed=9, sgd_mode="sgd",
              user_reg=1e-3, positive_reg=1e-3, negative_reg=1e-3, negative_interactions_quota=0.4)
    g = _mf(X, algo, **kw)  # mini-batch mode
    init = (g.get_USER_factors(), g.get_ITEM_factors())
    g.set_user_shard(LO, HI, 0, stream_id=1)
    samples = _draw(g, epochs=2)
    assert ((samples[0] >= LO) & (samples[0] < HI)).all()
    o = MFOracle(X, algorithm_name=algo, init_factors=init, samples=samples, **kw)
    for _ in range(2):
        o.epochIteration_Cython()
    for name in ("get_USER_factors", "get_ITEM_factors"):
        a, b = getattr(g, name)(), getattr(o, name)()
        assert np.allclose(a, b, rtol=1e-4, atol=2e-6), "%s: max abs diff %.3e" % (name, float(np.abs(a - b).max()))
    U = g.get_USER_factors()
    assert np.array_equal(U[:LO], init[0][:LO]) and np.array_equal(U[HI:], init[0][HI:])  # rows of other shards never move


def test_user_shard_refusals():
    X = _shard_urm()
    with pytest.raises(ValueError):
        _mf(X, "MF_BPR", sampler="glibc").set_user_shard(LO, HI, 0, 0)
    g = _mf(X, "MF_BPR", hogwild=True)
    with pytest.raises(ValueError):
        g.set_user_shard(LO, HI, (N_USERS // 8 + 1) * 8 + 1, 0)
    for lo, hi in ((HI, LO), (LO, LO), (-1, 10), (0, N_USERS + 1)):
        with pytest.raises(ValueError):
            g.set_user_shard(lo, hi, 0, 0)


def _no_sampleable_user_urm():
    """Every user has an empty profile or every item: the samplers' user draw has nothing to accept."""
    D = np.zeros((6, 5), np.float32)
    D[1] = 1.0
    D[4] = 2.0
    return sps.csr_matrix(D)


def test_philox_handles_refuse_a_urm_without_sampleable_users():
    """Only handle creation is called: an epoch on such a handle would never finish its first sample."""
    from recsys2019_deeplearning_evaluation_b200.dist import ShardedSLIM_BPR
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    X = _no_sampleable_user_urm()
    for algo in ("MF_BPR", "FUNK_SVD"):
        with pytest.raises(ValueError):
            _mf(X, algo, hogwild=True)
    with pytest.raises(ValueError):
        SLIM_BPR_Cython_Epoch(X, sampler="philox", hogwild=True, symmetric=False, random_seed=1)
    with pytest.raises(ValueError):
        ShardedSLIM_BPR(X, random_seed=1, world_rank=(1, 0), batch_size=4)


def test_user_shard_without_sampleable_users_is_refused():
    """A shard made only of empty and full profiles (users 120, 121 are empty, 150 is full) is refused at set_user_shard."""
    X = _shard_urm()
    lens = np.diff(X.indptr)
    g = _mf(X, "MF_BPR", hogwild=True)
    for lo, hi in ((120, 122), (150, 151), (0, 2)):
        assert ((lens[lo:hi] == 0) | (lens[lo:hi] == N_ITEMS)).all()
        with pytest.raises(ValueError):
            g.set_user_shard(lo, hi, 0, 0)
    assert 0 < lens[122] < N_ITEMS
    g.set_user_shard(120, 123, 0, 0)  # user 122 can be drawn


# ---------------------------------------------------------------------------------------------------------------------
# K4: IALS half epoch on slices of the warm rows

def _ials(X, f, reg):
    import torch
    from recsys2019_deeplearning_evaluation_b200.recommenders import IALSRecommender, _dev_csr
    from oracle.ials_oracle import confidence
    r = IALSRecommender(X, verbose=False)
    r.num_factors, r.reg = f, reg
    C = confidence(X, "linear", 2.0)
    r._d_C = _dev_csr(C)
    r._d_work = torch.empty((f, f), dtype=torch.float64, device="cuda")
    return r, C


@pytest.mark.parametrize("f", [64, 256])
def test_ials_half_epoch_on_row_shards(f):
    """Shards of 1, 2 and an odd number of warm rows, and larger ones, each solved by its own call into one X; some warm rows
    are in no shard.  Listed rows equal the full call's (fp64 atomics in Y^T Y: rounding) and the fp64 restatement; the other
    rows keep their sentinel bit for bit."""
    import torch
    from threadpoolctl import threadpool_limits
    from oracle.ials_oracle import update_row
    nu, ni, reg = 600, 1100, 1e-2  # n_items >= 4 f: the tensor-core kernel takes f = 256
    X = synth_urm(nu, ni, 0.02, seed=f, values="ratings").tolil()
    X[[3, 50, 51, 599], :] = 0  # cold users: in no shard
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    r, C = _ials(X, f, reg)
    rng = np.random.default_rng(f)
    Y = torch.from_numpy(f ** -0.5 * rng.random((ni, f))).cuda()
    warm = np.flatnonzero(np.diff(X.indptr) > 0).astype(np.int32)
    assert len(warm) < nu
    full = torch.full((nu, f), 1234.5, dtype=torch.float64, device="cuda")
    r._half(torch.from_numpy(warm).cuda(), r._d_C, Y, full)
    sizes = [1, 2, 7, 1, 150]
    skip = 11  # warm rows between the shards that no shard lists
    Xs = torch.full((nu, f), 1234.5, dtype=torch.float64, device="cuda")
    listed = []
    pos = 0
    for k, s in enumerate(sizes):
        rows = warm[pos:pos + s]
        listed.append(rows)
        r._half(torch.from_numpy(rows.copy()).cuda(), r._d_C, Y, Xs)
        pos += s + (skip if k == 2 else 0)
    rows = warm[pos:]
    listed.append(rows)
    r._half(torch.from_numpy(rows.copy()).cuda(), r._d_C, Y, Xs)
    listed = np.concatenate(listed)
    assert len(listed) == len(warm) - skip and len(rows) > 150
    A, F = Xs.cpu().numpy(), full.cpu().numpy()
    tol = 1e-9 if f <= 128 else 1e-6
    assert np.allclose(A[listed], F[listed], rtol=tol, atol=1e-3 * tol), float(np.abs(A[listed] - F[listed]).max())
    unlisted = np.setdiff1d(np.arange(nu), listed)
    assert np.array_equal(A[unlisted].view(np.int64), np.full((len(unlisted), f), 1234.5).view(np.int64))
    Yh = Y.cpu().numpy()
    YtY = Yh.T @ Yh
    with threadpool_limits(limits=4):
        for u in listed[::4][:60]:
            s, e = C.indptr[u], C.indptr[u + 1]
            ref = update_row(C.indices[s:e], C.data[s:e].astype(np.float64), Yh, YtY, reg)
            assert np.allclose(A[u], ref, rtol=1e-4, atol=1e-8), (u, float(np.abs(A[u] - ref).max()))


# ---------------------------------------------------------------------------------------------------------------------
# K5: EASE_R Gram over user shards

@pytest.mark.parametrize("values", ["binary", "ratings", "continuous"])
@pytest.mark.parametrize("n_items", [1100, 3000])
def test_ease_gram_over_user_shards(n_items, values):
    """n_items 1100 and 3000: the two modes of _gram_device (topK 0 and topK = n_items).  Shards include a block of users
    without interactions, a one-user shard and an empty one; their sum is the full Gram."""
    import torch
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(900, n_items, 0.01, seed=n_items, values=values).tolil()
    X[300:340, :] = 0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    rec = EASE_R_Recommender(X, verbose=False)
    G = rec._gram_device().cpu().numpy()
    cuts = [0, 120, 121, 121, 300, 340, 341, 600, 900]
    S = torch.zeros((n_items, n_items), dtype=torch.float32, device="cuda")
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        part = rec._gram_device(rows=(lo, hi))
        assert part.shape == (n_items, n_items) and part.dtype == torch.float32
        if hi == lo or (lo, hi) == (300, 340):
            assert not bool(part.any())
        S += part
    S = S.cpu().numpy()
    Xd = X.toarray().astype(np.float64)
    ref = Xd.T @ Xd
    off = ~np.eye(n_items, dtype=bool)
    assert np.abs(G[off]).max() > 0
    if values == "binary":
        assert np.array_equal(S, G)
        assert np.array_equal(G[off], ref[off].astype(np.float32))
    else:
        tol = 4 * np.finfo(np.float32).eps * (np.abs(Xd).T @ np.abs(Xd))[off] + 1e-30
        assert (np.abs(S[off] - ref[off]) <= tol).all(), float(np.abs(S[off] - ref[off]).max())
        assert (np.abs(G[off] - ref[off]) <= tol).all()
        assert np.allclose(np.diag(S), np.diag(G), rtol=1e-5, atol=0)


def test_ease_gram_empty_user_slice_is_zero():
    import torch
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(50, 30, 0.2, seed=1)
    G = EASE_R_Recommender(X, verbose=False)._gram_device(rows=(5, 5))
    assert G.shape == (30, 30) and G.dtype == torch.float32 and G.is_cuda and not bool(G.any())
    assert (balanced_ranges([100, 1, 1, 1], 4)[1:] == balanced_ranges([100, 1, 1, 1], 4)[:-1]).any()  # ranks with lo == hi
