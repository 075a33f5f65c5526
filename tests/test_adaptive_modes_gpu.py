"""-m gpu: the adaptive optimisers (adagrad, rmsprop, adam) on the hogwild trainers and on MF's barrier kernel, against the
C oracle.

An epoch is deterministic when it holds one sample: MF with batch_size 1 and a user shard of one sample per epoch, SLIM on
a URM with one user.  Over many such epochs the trainers must follow the oracle replayed on the same stream, which also
checks how the Adam powers carry from one epoch to the next (advanced on the host after a hogwild epoch, read back from
the device after a barrier epoch)."""
import numpy as np
import pytest

from oracle.sgd_oracle import MFOracle, SLIMOracle
from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 2e-6
MODES = ["adagrad", "rmsprop", "adam"]


@pytest.mark.parametrize("kernel", ["hogwild", "barrier"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_mf_one_sample_epochs_follow_the_oracle(algo, mode, kernel, monkeypatch):
    """FunkSVD carries bias terms; with them the mini-batch semantics always run on the barrier kernel (mf_epoch_kernel),
    and B200REC_MF_DATAFLOW=0 puts MF_BPR there too."""
    from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch
    monkeypatch.setenv("B200REC_MF_DATAFLOW", "0")
    X = synth_urm(20, 40, 0.1, seed=5, values="ratings")
    bias = algo == "FUNK_SVD"
    kw = dict(algorithm_name=algo, n_factors=12, batch_size=1, learning_rate=0.05, random_seed=11, sgd_mode=mode,
              user_reg=1e-3, positive_reg=2e-3, negative_reg=3e-3, use_bias=bias, bias_reg=1e-3,
              negative_interactions_quota=0.4)
    g = MatrixFactorization_Cython_Epoch(X, sampler="philox", hogwild=kernel == "hogwild", **kw)
    init = (g.get_USER_factors(), g.get_ITEM_factors())
    g.set_user_shard(0, X.shape[0], 1, stream_id=0)
    # the oracle's one epoch at batch size 1: n_users + 1 samples (BPR) or nnz + 1 (FunkSVD)
    n = (X.shape[0] if algo == "MF_BPR" else X.nnz) + 1
    drawn = []
    for _ in range(n):
        g.epochIteration_Cython()
        assert g.samples_last_epoch() == 1
        drawn.append(g.get_samples())
    samples = [np.concatenate([s[k] for s in drawn]) for k in range(3)]
    o = MFOracle(X, init_factors=init, samples=samples, **kw)
    o.epochIteration_Cython()
    names = ("get_USER_factors", "get_ITEM_factors") + (("get_USER_bias", "get_ITEM_bias", "get_GLOBAL_bias") if bias else ())
    for name in names:
        a, b = getattr(g, name)(), getattr(o, name)()
        assert np.allclose(a, b, rtol=RTOL, atol=ATOL), "%s: max abs diff %.3e" % (name, float(np.abs(a - b).max()))
    assert not np.allclose(g.get_ITEM_factors(), init[1])


@pytest.mark.parametrize("symmetric", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_slim_hogwild_one_user_follows_the_oracle(mode, symmetric):
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    X = synth_urm(1, 30, 0.3, seed=2)
    assert 0 < X.nnz < 30
    kw = dict(learning_rate=0.05, li_reg=1e-3, lj_reg=2e-3, topK=30, symmetric=symmetric, random_seed=6, sgd_mode=mode)
    g = SLIM_BPR_Cython_Epoch(X, sampler="philox", hogwild=True, **kw)
    epochs = 25
    drawn = []
    for _ in range(epochs):
        g.epochIteration_Cython()
        drawn.append(g.get_samples())
    samples = tuple(np.concatenate([s[k] for s in drawn]) for k in range(3))
    o = SLIMOracle(X, samples=samples, **kw)
    for _ in range(epochs):
        o.epochIteration_Cython()
    S = g.get_S_dense().astype(np.float64)
    R = o.S_full()
    np.fill_diagonal(R, 0)
    assert np.abs(R).max() > 0
    assert np.allclose(S, R, rtol=RTOL, atol=ATOL), float(np.abs(S - R).max())
