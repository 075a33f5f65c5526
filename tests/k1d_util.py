"""Helpers of the K1-D similarity tests (csrc/sim_k1d.cuh): the fixture that routes small matrices to K1-D, the per-phase
cycle counters of one call, and the full-range call checked against the union of sub-range calls."""
import ctypes

import numpy as np
import pytest


@pytest.fixture
def force_k1c(monkeypatch):
    monkeypatch.setenv("B200REC_K1C_MINCOLS", "1")
    monkeypatch.setenv("B200REC_K1C_LAMBDA", "1e9")  # every non-empty column goes to K1-D
    yield monkeypatch


def _lib():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    return _lib


def _phase_cycles(sim, fn):
    L = _lib().load()
    _lib().check(L.b200_sim_debug_phase_cycles(sim._h, 1, None))
    r = fn()
    out = (ctypes.c_uint64 * 16)()
    _lib().check(L.b200_sim_debug_phase_cycles(sim._h, 0, out))
    return r, np.array(list(out), dtype=np.float64)


def _full_vs_parts(X, n_parts=3, fail_every=0, **kw):
    """W of one full-range call and the sum of the W of n_parts sub-range calls on the same handle, plus the phase cycles
    of the full call."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    sim = Compute_Similarity_Cython(X, **kw)
    en = ctypes.c_int32()
    _lib().check(_lib().load().b200_sim_debug_k1c(sim._h, fail_every, ctypes.byref(en), None, None, None))
    assert en.value == 1
    W1, cyc = _phase_cycles(sim, sim.compute_similarity)
    n = X.shape[1]
    bounds = np.linspace(0, n, n_parts + 1).astype(int)
    W0 = None
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        Wp, cyc_p = _phase_cycles(sim, lambda: sim.compute_similarity(start_col=int(lo), end_col=int(hi)))
        assert cyc_p[8:12].sum() == 0  # a sub-range never takes the pair path
        W0 = Wp if W0 is None else W0 + Wp
    assert abs(W1 - W0).nnz == 0
    assert (W1.data != 0).all() and W1.diagonal().sum() == 0
    return W1, cyc
