"""CPU: the C-ABI library loads and exports every symbol include/b200rec.h declares; the Python binding table
matches the header; product code never imports the oracle; without a CUDA device calls fail loudly."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200rec.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[A-Za-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(lib, s), "libb200rec.so does not export %s" % s


def test_binding_table_matches_header():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    assert sorted(_lib.SIGNATURES) == header_symbols()
    lib = _lib.load()
    assert lib.b200_version() >= 100
    assert lib.b200_launch_count() >= 0


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "recsys2019_deeplearning_evaluation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "ref_loader" not in txt, f


def test_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
    X = synth_urm(50, 20, 0.2)
    with pytest.raises((_lib.B200Error, MemoryError)):
        Compute_Similarity_Cython(X, topK=5)


def test_create_scaled_rejects_columns_past_int32():
    """The column count is checked before it is narrowed to int, and before any CUDA call."""
    from recsys2019_deeplearning_evaluation_b200 import _lib
    L = _lib.load()
    h = ctypes.c_void_p(1)
    indptr = np.zeros(5, np.int32)
    A = np.ones(1, np.float32)
    B = np.ones(1, np.float32)
    rc = L.b200_sim_create_scaled(ctypes.byref(h), 4, 2**31, 0, _lib.ptr(indptr), None, None, _lib.ptr(A), _lib.ptr(B), 5, None)
    assert rc == -1
    assert h.value is None
    assert b"int32 index range exceeded" in L.b200_last_error()


def test_argument_errors_mirror_the_reference():
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython, Compute_Similarity
    from recsys2019_deeplearning_evaluation_b200.synth import synth_urm
    X = synth_urm(50, 20, 0.2)
    with pytest.raises(ValueError, match="not recognized"):
        Compute_Similarity_Cython(X, similarity="cosin")  # pyx:141-144
    with pytest.raises(ValueError, match="different number of rows"):
        Compute_Similarity_Cython(X, row_weights=np.ones(49))  # pyx:188-190
    with pytest.raises(ValueError):
        Compute_Similarity(X, use_implementation="fortran")  # Compute_Similarity.py:121
    Xbad = X.copy(); Xbad.data[0] = np.inf
    with pytest.raises(AssertionError):
        Compute_Similarity(Xbad)  # Compute_Similarity.py:44


def _sgd_create_calls():
    """Each SGD trainer's create entry point as f(out, n_users=.., sgd_mode=.., indptr=.., col_lo=.., col_hi=..) on a valid
    4 x 3 URM, so that one argument at a time can be made bad."""
    from recsys2019_deeplearning_evaluation_b200 import _lib
    L = _lib.load()
    indptr = np.array([0, 1, 2, 3, 3], np.int32)
    indices = np.array([0, 1, 2], np.int32)
    data = np.ones(3, np.float32)
    U = np.zeros((4, 2), np.float64)
    V = np.zeros((3, 2), np.float64)
    keep = (indptr, indices, data, U, V)

    def mf(out, n_users=4, sgd_mode=0, indptr=_lib.ptr(indptr), **_):
        return L.b200_mf_create(out, n_users, 3, 3, indptr, _lib.ptr(indices), _lib.ptr(data), 2, 0, 1, 0.5, 0.1, 0, 0.0, 0.0,
                                0.0, 0.0, 0.0, sgd_mode, 0.9, 0.9, 0.999, _lib.ptr(U), _lib.ptr(V), 1, 7, 1, 0)

    def slim(out, n_users=4, sgd_mode=0, indptr=_lib.ptr(indptr), **_):
        return L.b200_slim_create(out, n_users, 3, 3, indptr, _lib.ptr(indices), 0.1, 0.0, 0.0, 0, sgd_mode, 0.9, 0.9, 0.999,
                                  1, 7, 1, 0)

    def slim_sharded(out, n_users=4, sgd_mode=0, indptr=_lib.ptr(indptr), col_lo=0, col_hi=3):
        return L.b200_slim_create_sharded(out, n_users, 3, 3, indptr, _lib.ptr(indices), 0.1, 0.0, 0.0, sgd_mode, 0.9, 0.9,
                                          0.999, 7, col_lo, col_hi)

    def asysvd(out, n_users=4, sgd_mode=0, indptr=_lib.ptr(indptr), **_):
        return L.b200_asysvd_create(out, n_users, 3, 3, indptr, _lib.ptr(indices), _lib.ptr(data), 2, 0.5, 0.1, 0, 0.0, 0.0,
                                    0.0, sgd_mode, 0.9, 0.9, 0.999, _lib.ptr(V), _lib.ptr(V), 1, 7)

    calls = {"b200_mf_create": mf, "b200_slim_create": slim, "b200_slim_create_sharded": slim_sharded,
             "b200_asysvd_create": asysvd}
    return L, calls, keep


@pytest.mark.parametrize("bad", [dict(n_users=0), dict(sgd_mode=99), dict(indptr=None), dict(col_lo=2, col_hi=2)],
                         ids=["shape", "sgd_mode", "null_array", "column_range"])
def test_sgd_create_rejects_bad_arguments_before_any_cuda_call(bad):
    """Every SGD trainer's create entry point checks its arguments before it touches the device: B200_E_INVALID, *out left
    NULL, and an error text that names the entry point."""
    L, calls, keep = _sgd_create_calls()
    for fn, call in calls.items():
        if "col_lo" in bad and fn != "b200_slim_create_sharded":
            continue
        h = ctypes.c_void_p(1)
        rc = call(ctypes.byref(h), **bad)
        assert rc == -1, (fn, bad)
        assert h.value is None, (fn, bad)
        assert L.b200_last_error().decode().startswith(fn + ":"), (fn, bad, L.b200_last_error())
