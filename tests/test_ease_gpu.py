"""-m gpu: EASE^R (Gram through the dense mode of the similarity kernel + blocked-Cholesky SPD inverse) against the
reference's golden B / scores and the fp64 restatement; plus the dense outputs of Compute_Similarity_Cython."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle.ease_oracle import ease_B
from oracle.similarity_oracle import SimilarityOracle
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu
Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ease_golden.npz"))


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("n,values,l2", [(0, "binary", 50.0), (1, "ratings", 500.0)])
def test_ease_matches_reference_golden(n, values, l2):
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(600, 200, 0.05, seed=23, values=values)
    r = EASE_R_Recommender(X, verbose=False)
    r.fit(topK=None, l2_norm=l2, verbose=False)
    B = np.asarray(r.W_sparse)
    assert B.shape == (200, 200) and (np.diag(B) == 0).all()
    # 1e-4 of the largest coefficient (north_star tolerance; both sides are fp32 factorisations of the same matrix)
    assert _rel(B, Z["ease%d_B" % n]) < 1e-4
    sc = r._compute_item_score(np.arange(30))
    assert _rel(sc, Z["ease%d_scores" % n]) < 1e-4
    r2 = EASE_R_Recommender(X, verbose=False)
    r2.fit(topK=20, l2_norm=l2, verbose=False)
    assert sps.issparse(r2.W_sparse) and (np.diff(r2.W_sparse.tocsc().indptr) <= 20).all()
    col = r2.W_sparse[:, 7].toarray().ravel()
    ref = Z["ease%d_B" % n][:, 7]
    keep = np.argsort(-ref, kind="stable")[:20]
    assert set(np.flatnonzero(col)) == set(keep[ref[keep] != 0])


def test_ease_multi_block_against_fp64():
    """n_items = 1100 -> padded to 1152 = 9 Cholesky blocks; l2 small enough to make the inverse non-trivial."""
    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    X = synth_urm(5000, 1100, 0.02, seed=31, values="binary")
    r = EASE_R_Recommender(X, verbose=False)
    r.fit(topK=None, l2_norm=20.0, verbose=False)
    B = ease_B(X, 20.0)
    assert _rel(np.asarray(r.W_sparse), B) < 1e-4
    users = np.arange(0, 5000, 501)
    assert _rel(r._compute_item_score(users), X[users] @ B) < 1e-4


def test_dense_similarity_outputs():
    """TopK == 0 -> dense float64 W_dense[j, i] (pyx:510-513,597-599); topK = n_columns -> every non-zero similarity."""
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    X = synth_urm(900, 2600, 0.01, seed=12, values="ratings")
    for kw in (dict(shrink=3, normalize=True, similarity="cosine"), dict(shrink=0, normalize=False, similarity="cosine"),
               dict(shrink=1, similarity="asymmetric", asymmetric_alpha=0.2)):
        orc = SimilarityOracle(X, topK=2600, **kw)
        D = orc.column_values(np.arange(2600))
        W0 = Compute_Similarity_Cython(X, topK=0, **kw).compute_similarity()
        assert isinstance(W0, np.ndarray) and W0.dtype == np.float64 and W0.shape == (2600, 2600)
        assert np.allclose(W0, D, rtol=1e-4, atol=1e-9)
        Wn = Compute_Similarity_Cython(X, topK=2600, **kw).compute_similarity()
        assert sps.issparse(Wn) and np.allclose(Wn.toarray(), D, rtol=1e-4, atol=1e-9)
    Wk = Compute_Similarity_Cython(X, topK=2100, shrink=3).compute_similarity()  # beyond the selection buffer: dense + top-K
    assert (np.diff(Wk.tocsc().indptr) <= 2100).all() and Wk.nnz > 0


def _gemm_case(version, kind, M, N, K, beta):
    import ctypes
    import torch
    from recsys2019_deeplearning_evaluation_b200 import _lib
    g = torch.Generator(device="cpu").manual_seed(1000 * kind + M + N + K)
    shape_a = (M, K) if kind in (0, 1) else (K, M)
    shape_b = (N, K) if kind == 0 else (K, N)
    A = torch.randn(shape_a, generator=g, dtype=torch.float32).cuda()
    B = torch.randn(shape_b, generator=g, dtype=torch.float32).cuda()
    if kind == 2:  # the L^T L product: operands are lower triangular, so dropping k < max(row, col block) changes nothing
        A, B = torch.tril(A), torch.tril(B)
    C0 = torch.randn((M, N), generator=g, dtype=torch.float32).cuda()
    C = C0.clone()
    _lib.check(_lib.load().b200_debug_gemm_device(version, kind, M, N, K, 0.75, A.data_ptr(), A.shape[1], B.data_ptr(), B.shape[1],
                                                  beta, C.data_ptr(), N, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    Ad, Bd = A.double(), B.double()
    ref = 0.75 * (Ad @ Bd.t() if kind == 0 else (Ad @ Bd if kind == 1 else Ad.t() @ Bd)) + beta * C0.double()
    err = (C.double() - ref).abs().max().item() / ref.abs().max().item()
    # 3xTF32: fp32-level accuracy (a single TF32 pass gives ~3e-4).  The tensor core accumulates with truncation, so the
    # error grows linearly with the number of K = 8 steps.
    assert err < 1e-5 * max(1.0, K / 512.0), (version, kind, M, N, K, beta, err)


GEMM_SHAPES = [(0, 384, 128, 128, 0.0), (0, 256, 256, 128, 1.0), (1, 128, 128, 640, 0.0), (2, 512, 512, 512, 0.0)]


@pytest.mark.parametrize("kind,M,N,K,beta", GEMM_SHAPES)
def test_tensor_core_gemm_v1(kind, M, N, K, beta):
    """The three GEMM shapes of the blocked inverse through the first wgmma kernel (B200REC_GEMM=1), against fp64."""
    _gemm_case(1, kind, M, N, K, beta)


@pytest.mark.parametrize("kind,M,N,K,beta", GEMM_SHAPES + [(0, 1024, 1024, 128, 1.0), (2, 2048, 2048, 2048, 0.0)])
def test_tensor_core_gemm_v2(kind, M, N, K, beta):
    """The default kernel (pre-packed hi/lo TF32 operands, cp.async.bulk producer, mbarrier ring)."""
    _gemm_case(2, kind, M, N, K, beta)
