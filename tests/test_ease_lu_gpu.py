"""-m gpu: the fp64 pivoted-LU inverse (csrc/lu_inverse.cu) and its FP64 tensor-core GEMM (csrc/dgemm_tc.cuh) against
float64 numpy / torch, and EASE_R on Gram matrices that are not positive definite (explicit ratings, small or negative
l2_norm), which take that path, against the fp64 restatement."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.ease_oracle import ease_B
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm

pytestmark = pytest.mark.gpu


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def _lu_inverse(A, n_pad=None):
    """b200_lu_inverse_device on A (n x n float64) padded to n_pad with an identity block; returns the n_pad x n_pad result."""
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    n = A.shape[0]
    n_pad = n_pad or n
    Ap = np.eye(n_pad)
    Ap[:n, :n] = A
    d_A = torch.from_numpy(Ap).cuda()
    work = torch.empty(2 * n_pad * n_pad, dtype=torch.float64, device="cuda")
    _lib.check(_lib.load().b200_lu_inverse_device(d_A.data_ptr(), n_pad, work.data_ptr(), _stream()))
    return d_A.cpu().numpy()


def _gram(X, l2):
    """The matrix EASE_R inverts (oracle.ease_oracle.ease_B before its inverse), fp64."""
    X = sps.csr_matrix(X, dtype=np.float32)
    G = np.asarray((X.T @ X).todense(), dtype=np.float64)
    G[np.diag_indices_from(G)] = np.diff(X.tocsc().indptr) + l2
    return G


# ---------------------------------------------------------------------------------------------- fp64 tensor-core GEMM
@pytest.mark.parametrize("kind,M,N,K,beta", [(0, 128, 128, 16, 0.0), (0, 384, 256, 1024, 1.5), (0, 256, 640, 128, 0.0),
                                             (1, 512, 128, 384, 0.0), (1, 384, 256, 128, -1.0), (2, 512, 512, 512, 0.0),
                                             (2, 1024, 1024, 1024, 0.5)])
def test_dgemm_hook_against_fp64_matmul(kind, M, N, K, beta):
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    g = torch.Generator(device="cpu").manual_seed(7 * kind + M + 3 * N + K)
    batch = M // 128 if kind == 1 else 1
    A = torch.randn((M, K), generator=g, dtype=torch.float64)
    B = torch.randn((batch * K, N), generator=g, dtype=torch.float64)
    if kind == 2:  # U^-1 L^-1: upper times lower, so dropping k < max(row block, column block) changes nothing
        A, B = torch.triu(A), torch.tril(B)
    C0 = torch.randn((M, N), generator=g, dtype=torch.float64)
    dA, dB, dC = A.cuda(), B.cuda(), C0.cuda()
    _lib.check(_lib.load().b200_debug_dgemm_device(kind, M, N, K, -0.75, dA.data_ptr(), K, dB.data_ptr(), N, beta, dC.data_ptr(), N,
                                                   _stream()))
    if kind == 1:
        ref = torch.cat([A[128 * b:128 * (b + 1)] @ B[K * b:K * (b + 1)] for b in range(batch)])
    else:
        ref = A @ B
    ref = -0.75 * ref + beta * C0
    err = (dC.cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err <= 1e-12, (kind, M, N, K, beta, err)


# ---------------------------------------------------------------------------------------------- LU inverse, C entry point
@pytest.mark.parametrize("n", [128, 256, 1152, 4096])
def test_lu_inverse_random_nonsymmetric(n):
    A = np.random.default_rng(n).standard_normal((n, n))
    assert np.linalg.cond(A) <= 1e6
    assert _rel(_lu_inverse(A), np.linalg.inv(A)) <= 1e-9


def test_lu_inverse_zero_diagonal_needs_pivoting():
    """Rows of a well-conditioned matrix in reverse order with its anti-diagonal zeroed: every diagonal entry is 0."""
    n = 512
    rng = np.random.default_rng(3)
    M = np.eye(n) + 0.3 * rng.standard_normal((n, n)) / np.sqrt(n)
    M[np.arange(n), n - 1 - np.arange(n)] = 0.0
    A = M[::-1].copy()
    assert (np.diag(A) == 0).all() and np.linalg.cond(A) <= 1e6
    assert _rel(_lu_inverse(A), np.linalg.inv(A)) <= 1e-9


def test_lu_inverse_singular_leading_block():
    """The leading 128 x 128 block (one panel) has rank 1; the whole matrix is well conditioned."""
    n = 512
    rng = np.random.default_rng(7)
    A = rng.standard_normal((n, n))
    A[:128, :128] = np.outer(rng.standard_normal(128), rng.standard_normal(128))
    assert np.linalg.matrix_rank(A[:128, :128]) == 1 and np.linalg.cond(A) <= 1e6
    assert _rel(_lu_inverse(A), np.linalg.inv(A)) <= 1e-9


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_lu_inverse_pivot_ties(seed):
    """+-1 entries: every column of the first step ties in magnitude (the lowest row wins, LAPACK's idamax)."""
    A = np.sign(np.random.default_rng(seed).standard_normal((384, 384)))
    assert np.linalg.cond(A) <= 1e6
    assert _rel(_lu_inverse(A), np.linalg.inv(A)) <= 1e-9


@pytest.mark.parametrize("n,n_pad", [(1, 128), (200, 256), (1100, 1152)])
def test_lu_inverse_padding_stays_identity(n, n_pad):
    A = np.random.default_rng(n).standard_normal((n, n)) + 2.0 * np.sqrt(n) * np.eye(n)[::-1]
    R = _lu_inverse(A, n_pad)
    assert _rel(R[:n, :n], np.linalg.inv(A)) <= 1e-9
    assert (R[n:, n:] == np.eye(n_pad - n)).all()
    assert (R[:n, n:] == 0).all() and (R[n:, :n] == 0).all()


def test_lu_inverse_zero_column_is_singular():
    n = 512
    A = np.random.default_rng(11).standard_normal((n, n))
    A[:, 300] = 0.0
    with pytest.raises(np.linalg.LinAlgError, match=r"singular matrix \(zero pivot at column 300\)"):
        _lu_inverse(A)


# ---------------------------------------------------------------------------------------------- EASE_R, indefinite Gram
def _check_ease(X, l2, users):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    with pytest.raises(np.linalg.LinAlgError):  # not positive definite: the fit takes the LU path
        np.linalg.cholesky(_gram(X, l2))
    r = EASE_R_Recommender(X, verbose=False)
    r.fit(topK=None, l2_norm=l2, verbose=False)
    B = np.asarray(r.W_sparse)
    B_ref = ease_B(X, l2)
    assert B.shape == B_ref.shape and (np.diag(B) == 0).all()
    if X.shape[1] == 1:
        assert (B == 0).all()
        return
    assert np.abs(B - B_ref).max() <= 1e-6 * np.abs(B_ref).max()
    assert _rel(r._compute_item_score(users), X[users] @ B_ref) <= 1e-5


@pytest.mark.parametrize("shape,l2", [((600, 200, 0.05), 50.0), ((5000, 1100, 0.02), 20.0), ((5000, 1100, 0.02), 200.0)])
def test_ease_indefinite_ratings(shape, l2):
    X = synth_urm(*shape, seed=23, values="ratings")
    _check_ease(X, l2, np.arange(0, shape[0], max(1, shape[0] // 40)))


def test_ease_indefinite_c2_ratings_default_l2():
    """The MovieLens-1M shape with the reference's default l2_norm = 1e3 (1 482 negative eigenvalues)."""
    X = synth_config("C2", values="ratings")
    _check_ease(X, 1e3, np.arange(0, X.shape[0], 97))


@pytest.mark.parametrize("n,l2", [(1, -40.0), (127, -5.0), (128, -5.0), (129, -5.0)])
def test_ease_indefinite_padding_edges(n, l2):
    X = synth_urm(400, n, 0.08, seed=5, values="ratings")
    _check_ease(X, l2, np.arange(0, 400, 13))


def test_ease_indefinite_topk():
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(600, 200, 0.05, seed=23, values="ratings")
    B_ref = ease_B(X, 50.0)
    r = EASE_R_Recommender(X, verbose=False)
    r.fit(topK=20, l2_norm=50.0, verbose=False)
    W = r.W_sparse.tocsc()
    assert sps.issparse(r.W_sparse) and (np.diff(W.indptr) <= 20).all()
    tol = 1e-6 * np.abs(B_ref).max()
    for j in range(200):
        ref = B_ref[:, j]
        col = W[:, j].toarray().ravel()
        kept = np.flatnonzero(col)
        top = np.argsort(-ref, kind="stable")[:20]
        t = ref[top[-1]]  # the 20th largest
        assert len(kept) == np.count_nonzero(ref[top]), j
        assert (ref[kept] >= t - tol).all(), j
        others = np.setdiff1d(np.flatnonzero(ref), kept)
        assert (ref[others] <= t + tol).all(), j
        assert np.abs(col[kept] - ref[kept]).max() <= tol, j


def test_ease_singular_gram_raises():
    """Binary data, an item nobody rated and l2_norm = 0: a zero row and column in G."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(300, 150, 0.05, seed=8, values="binary").tolil()
    X[:, 17] = 0
    X = sps.csr_matrix(X)
    X.eliminate_zeros()
    with pytest.raises(np.linalg.LinAlgError):
        ease_B(X, 0.0)
    r = EASE_R_Recommender(X, verbose=False)
    with pytest.raises(ValueError):
        r.fit(l2_norm=0.0, verbose=False)
    with pytest.raises(np.linalg.LinAlgError, match="Singular matrix"):
        r.fit(l2_norm=0.0, verbose=False)
