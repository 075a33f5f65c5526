"""K1-D pair path, the exchange by destination tile (csrc/sim_k1d.cuh): tiles of 2^tile_log2 columns, a bucket pass
that reserves one run per (CTA, tile), and a place pass that ranks each tile's cells per column in shared memory and
stages the tile's mirror region there (a longer region is written directly).  The width is set through
`b200_sim_debug_pair_lists`: one column per tile, tiles that hold only an empty column, a last tile that is cut short,
and one tile whose region is longer than the stage.  As in test_k1d_pairs_gpu.py, the full-range W must equal the sum
of the sub-range Ws (the K1-D kernel on every column) exactly, and the per-column mirror counts must be zero after every
call -- `-m gpu`."""
import ctypes

import numpy as np
import pytest

from k1d_util import _lib, _phase_cycles, force_k1c  # noqa: F401 (fixture)
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
from test_k1d_exchange_gpu import K, KW, S_CAP, _designed

pytestmark = pytest.mark.gpu



def _handle(X, fail_every=0, **kw):
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    sim = Compute_Similarity_Cython(X, **kw)
    en = ctypes.c_int32()
    _lib().check(_lib().load().b200_sim_debug_k1c(sim._h, fail_every, ctypes.byref(en), None, None, None))
    assert en.value == 1
    return sim


def _set_tile(sim, tile_log2):
    _lib().check(_lib().load().b200_sim_debug_pair_lists(sim._h, tile_log2, None, None, None))


def _lists(sim, n):
    """(tile width log2 of the last pair-path call, deg, mir_off), both n + 1 values"""
    tl = ctypes.c_int32()
    deg, off = np.full(n + 1, -1, np.int32), np.full(n + 1, -1, np.int32)
    _lib().check(_lib().load().b200_sim_debug_pair_lists(sim._h, -1, ctypes.byref(tl), deg.ctypes.data, off.ctypes.data))
    return tl.value, deg, off


def _full(sim, n):
    """One full-range call: its W, phase counters and mirror offsets; the mirror counts are zero after it."""
    W, cyc = _phase_cycles(sim, sim.compute_similarity)
    tl, deg, off = _lists(sim, n)
    assert (deg == 0).all()
    return W, cyc, tl, off


def _parts(sim, n, n_parts=3):
    W0 = None
    for lo, hi in zip(np.linspace(0, n, n_parts + 1).astype(int)[:-1], np.linspace(0, n, n_parts + 1).astype(int)[1:]):
        Wp, cyc = _phase_cycles(sim, lambda: sim.compute_similarity(start_col=int(lo), end_col=int(hi)))
        assert cyc[8:14].sum() == 0  # a sub-range never takes the pair path
        W0 = Wp if W0 is None else W0 + Wp
    return W0


def _check_exchange(cyc, off):
    """The pair path ran and its exchange wrote every mirror cell, in at most as many runs as cells."""
    assert cyc[8] > 0 and cyc[11] > 0
    runs, cells = cyc[12], cyc[13]
    assert 0 < runs <= cells == off[-1]


def test_tile_widths_on_one_handle(force_k1c):
    """One handle, the tile width changed between full-range calls: every width gives the sub-range W.  The designed
    columns add lists of K and 2048 / 2049 candidates (the last one past sel_cap: redone), a stage overflow in the upper
    pass (loose cells), a column at the top of the norm order and an empty column; 3 000 columns are no multiple of the
    batch or of the wider tiles, and 4 096-column tiles put the whole catalogue into one region longer than the stage."""
    X = _designed([(3, K, 1), (9, 300, 1), (11, S_CAP, 30), (13, S_CAP + 1, 30), (5, 2600, 30)])
    X.data[X.indices == 17] = 0
    X.eliminate_zeros()
    n = X.shape[1]
    sim = _handle(X, **KW)
    W0 = _parts(sim, n)
    assert (W0.data != 0).all() and W0.diagonal().sum() == 0 and W0[:, 17].nnz == 0
    sizes = {}
    for tl in (0, 1, 3, 6, 12):
        _set_tile(sim, tl)
        W1, cyc, used, off = _full(sim, n)
        assert used == tl
        assert abs(W1 - W0).nnz == 0, tl
        _check_exchange(cyc, off)
        edges = np.minimum(np.arange(0, n + (1 << tl), 1 << tl), n)
        sizes[tl] = np.diff(off[edges])
    assert (sizes[0] == 0).sum() >= 1                           # a tile of one empty column
    assert n % 64 != 0 and len(sizes[6]) == n // 64 + 1         # the last tile is cut short
    assert len(sizes[12]) == 1 and sizes[12][0] > 24576       # one region longer than the place kernel's stage


def test_fallback_and_repeated_calls(force_k1c):
    """Small tiles: repeated full-range calls give the same W and leave the mirror counts zero; a call that falls back
    (the fail_every hook) places nothing, leaves them zero too, and the next normal call is exact again."""
    X = _designed([(5, 2600, 30), (9, 300, 1)])
    n = X.shape[1]
    sim = _handle(X, **KW)
    _set_tile(sim, 2)
    W1, cyc, used, off = _full(sim, n)
    assert used == 2
    _check_exchange(cyc, off)
    for _ in range(2):
        W, cyc, _, _ = _full(sim, n)
        assert abs(W - W1).nnz == 0
        assert cyc[12] > 0
    _lib().check(_lib().load().b200_sim_debug_k1c(sim._h, 3, None, None, None, None))
    W, cyc, _, _ = _full(sim, n)
    assert cyc[11] == 0 and cyc[12] == 0 and cyc[1] > 0
    assert abs(W - W1).nnz == 0
    _lib().check(_lib().load().b200_sim_debug_k1c(sim._h, 0, None, None, None, None))
    W, cyc, _, _ = _full(sim, n)
    assert cyc[12] > 0 and abs(W - W1).nnz == 0
    assert abs(W1 - _parts(sim, n)).nnz == 0


@pytest.mark.parametrize("n_cols", [32_768, 32_769])
@pytest.mark.parametrize("tile_log2", [-1, 2])
def test_smallest_k1d_catalogues(n_cols, tile_log2):
    """32 768 columns is the smallest catalogue the create-time routing gives K1-D (no routing hook here), odd and even,
    with the default tiles (64 columns, so the last one is cut short on the odd catalogue) and with four columns per tile."""
    X = synth_urm(200_000, n_cols, 0.0015, seed=21, values="binary")
    sim = _handle(X, **KW)
    if tile_log2 >= 0:
        _set_tile(sim, tile_log2)
    W1, cyc, used, off = _full(sim, n_cols)
    _check_exchange(cyc, off)
    assert used == (6 if tile_log2 < 0 else tile_log2)
    assert abs(W1 - _parts(sim, n_cols)).nnz == 0
    assert W1.nnz == K * n_cols
