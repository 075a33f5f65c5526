"""IALS: the numpy restatement against the reference's golden factors (CPU) and the CUDA half-epoch kernel against both
(-m gpu).  fp64 on both sides; tolerance 1e-4 relative (north_star), observed agreement is far tighter."""
import os
import runpy

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.ials_oracle import confidence, run_epoch
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

HERE = os.path.dirname(os.path.abspath(__file__))
IALS_CASES = runpy.run_path(os.path.join(HERE, "golden", "make_golden.py"), run_name="cases")["IALS_CASES"]
Z = np.load(os.path.join(HERE, "golden", "ials_golden.npz"))


def case_urm(n):
    X = synth_urm(500, 180, 0.05, seed=29, values=IALS_CASES[n]["values"]).tolil()
    X[7, :] = 0
    X[:, 11] = 0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    return X


@pytest.mark.parametrize("n", range(len(IALS_CASES)))
def test_oracle_matches_reference_golden(n):
    c = IALS_CASES[n]
    X = case_urm(n)
    C = confidence(X, c["confidence_scaling"], c["alpha"], c.get("epsilon", 1.0))
    U, V = np.zeros((500, c["num_factors"])), Z["ials%d_V0" % n].copy()
    for _ in range(2):
        U, V = run_epoch(C, U, V, c["reg"])
    warm_u = np.diff(X.indptr) > 0
    assert np.allclose(U[warm_u], Z["ials%d_U" % n][warm_u], rtol=1e-9, atol=1e-12)
    assert np.allclose(V, Z["ials%d_V" % n], rtol=1e-9, atol=1e-12)  # the cold item keeps its initial row in both


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(len(IALS_CASES)))
def test_cuda_matches_reference_golden(n):
    from recsys2019_deeplearning_evaluation_b200.recommenders import IALSRecommender
    c = dict(IALS_CASES[n])
    c.pop("values")
    X = case_urm(n)
    np.random.seed(100 + n)
    r = IALSRecommender(X, verbose=False)
    r.fit(epochs=2, **c)
    warm_u = np.diff(X.indptr) > 0
    assert np.allclose(r.USER_factors[warm_u], Z["ials%d_U" % n][warm_u], rtol=1e-4, atol=1e-9)
    assert np.allclose(r.ITEM_factors, Z["ials%d_V" % n], rtol=1e-4, atol=1e-9)
    assert (r.USER_factors[7] == 0).all()  # cold user untouched (np.empty garbage in the reference, zeros here)
    sc = r._compute_item_score(np.arange(20))
    assert np.allclose(sc, r.USER_factors[:20] @ r.ITEM_factors.T, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("f", [1, 17, 64, 130, 208, 209, 256])
def test_cuda_factor_sizes_against_restatement(f):
    from threadpoolctl import threadpool_limits
    from recsys2019_deeplearning_evaluation_b200.recommenders import IALSRecommender
    # the restatement inverts one f x f matrix per row in a Python loop: keep the row count small for the large systems
    # and BLAS single-threaded (on a many-core box its thread pool spins for minutes on matrices this small)
    nu = 700 if f <= 64 else 240
    X = synth_urm(nu, 260, 0.04, seed=f, values="ratings")
    np.random.seed(f)
    V0 = f ** -0.5 * np.random.random_sample((260, f))
    np.random.seed(f)
    r = IALSRecommender(X, verbose=False)
    r.fit(epochs=2, num_factors=f, alpha=3.0, reg=5e-3)
    C = confidence(X, "linear", 3.0)
    U, V = np.zeros((nu, f)), V0.copy()
    with threadpool_limits(limits=1):
        for _ in range(2):
            U, V = run_epoch(C, U, V, 5e-3)
    warm = np.diff(X.indptr) > 0
    assert np.allclose(r.USER_factors[warm], U[warm], rtol=1e-4, atol=1e-8), float(np.abs(r.USER_factors - U).max())
    assert np.allclose(r.ITEM_factors, V, rtol=1e-4, atol=1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("f", [8, 64, 100, 128, 160, 256])
def test_tensor_core_kernel_every_size_against_restatement(f, monkeypatch):
    """ials_v2.cuh (wgmma 3xTF32 Gram, blocked fp32 Cholesky, fp64 refinement) forced on for every factor count it serves
    (by default it takes over above 128 factors), on a shape with enough rows on the other side to be eligible
    (n_other >= 4 f), ratings as confidences (c - 1 varies per entry: the sqrt(c - 1) operand scaling)."""
    from threadpoolctl import threadpool_limits
    from recsys2019_deeplearning_evaluation_b200.recommenders import IALSRecommender
    monkeypatch.setenv("B200REC_IALS_V2", "1")
    nu, ni = 1100, 1056
    X = synth_urm(nu, ni, 0.03, seed=100 + f, values="ratings")
    np.random.seed(f)
    V0 = f ** -0.5 * np.random.random_sample((ni, f))
    np.random.seed(f)
    r = IALSRecommender(X, verbose=False)
    r.fit(epochs=1, num_factors=f, alpha=2.0, reg=1e-2)
    C = confidence(X, "linear", 2.0)
    with threadpool_limits(limits=4):
        U, V = run_epoch(C, np.zeros((nu, f)), V0.copy(), 1e-2)
    warm = np.diff(X.indptr) > 0
    assert np.allclose(r.USER_factors[warm], U[warm], rtol=1e-4, atol=1e-8), float(np.abs(r.USER_factors - U).max())
    assert np.allclose(r.ITEM_factors, V, rtol=1e-4, atol=1e-8), float(np.abs(r.ITEM_factors - V).max())


@pytest.mark.gpu
def test_argument_errors():
    from recsys2019_deeplearning_evaluation_b200.recommenders import IALSRecommender
    X = synth_urm(50, 20, 0.2)
    with pytest.raises(ValueError, match="confidence_scaling"):
        IALSRecommender(X, verbose=False).fit(epochs=1, confidence_scaling="sqrt")
    with pytest.raises(ValueError, match="n_factors"):
        IALSRecommender(X, verbose=False).fit(epochs=1, num_factors=257)
