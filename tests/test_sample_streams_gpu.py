"""The SGD trainers' sample streams, value for value.

Every trainer (BPR-MF / FunkSVD, SLIM-BPR, AsySVD) draws its samples with the rule of the reference's sampleBPR_Cython /
sampleMSE_Cython (MatrixFactorization_Cython_Epoch.pyx:881-987, SLIM_BPR_Cython_Epoch.pyx:436-480):
  1. redraw the user until 0 < profile length < n_items;
  2. FunkSVD with a non-zero quota: one draw chooses positive (uniform <= quota) or negative;
  3. a positive is a draw of a position in the profile;
  4. a negative is redrawn until it is not in the profile.
The draws come from glibc's rand() (the reference's own stream, replayed on the host or resolved on the device) or from
Philox4x32-10 on the device.  The glibc streams are compared with the C oracle's sampler (oracle/sgd_oracle.c); the Philox
streams with the restatement below, which is checked against the Random123 known answers without a GPU."""
import numpy as np
import pytest
import scipy.sparse as sps

from recsys2019_deeplearning_evaluation_b200.synth import synth_urm

M32 = 0xFFFFFFFF
MF_C3, SLIM_C3 = 0x9E3779B9, 0x243F6A88  # fourth counter word of the MF and the SLIM streams


def philox4x32_10(ctr, key):
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c3 ^ k1) & M32, p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def philox_draws(g, seed, epoch, c3):
    """Sample g's draws: counter (g low word, g high word, draw block, C3), key (seed, epoch), words taken x, y, z, w."""
    blk = 0
    while True:
        yield from philox4x32_10((g & M32, g >> 32, blk, c3), (seed, epoch))
        blk += 1


def philox_uniform_le(x, quota):
    """The device's fp32 test: the draw's top 24 bits as a uniform in [0, 1)."""
    return np.float32(x >> 8) * np.float32(2.0 ** -24) <= np.float32(quota)


def draw_sample(draws, uniform_le, X, user_lo, n_users, bpr, quota):
    """(u, i, j) for BPR, (u, i, r) for MSE; every modulo is unsigned 32-bit."""
    n_items = X.shape[1]
    while True:
        u = user_lo + next(draws) % n_users
        s, e = int(X.indptr[u]), int(X.indptr[u + 1])
        if 0 < e - s < n_items:
            break
    profile = X.indices[s:e]
    positive = True
    if not bpr and quota != 0:
        positive = uniform_le(next(draws), quota)
    if bpr or positive:
        k = s + next(draws) % (e - s)
        item, r = int(X.indices[k]), np.float32(X.data[k])
    if bpr or not positive:
        while True:
            neg = next(draws) % n_items
            if neg not in profile:
                break
        if bpr:
            return u, item, neg
        return u, neg, np.float32(0)
    return u, item, r


def philox_stream(X, n, seed, epoch, c3, bpr=True, quota=0.0, user_lo=0, n_users=None):
    n_users = X.shape[0] if n_users is None else n_users
    out = [draw_sample(philox_draws(g, seed, epoch, c3), philox_uniform_le, X, user_lo, n_users, bpr, quota) for g in range(n)]
    return [np.array(col) for col in zip(*out)]


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((M32,) * 4, (M32, M32), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_restatement_reproduces_the_random123_known_answers(ctr, key, want):
    assert philox4x32_10(ctr, key) == want


def test_sampling_rule_restatement_on_scripted_draws():
    """Users 0 (empty) and 1 (full) are redrawn; item 4 of user 2's profile {1, 4} is redrawn as a negative."""
    D = np.zeros((3, 5), np.float32)
    D[1] = 1.0
    D[2, 1], D[2, 4] = 2.0, 5.0
    X = sps.csr_matrix(D)
    draws = iter([3, 4, 5, 7, 9, 13])  # users 0, 1, 2; position 7 % 2 = 1 (item 4); negatives 4 (rejected), 3
    assert draw_sample(draws, None, X, 0, 3, True, 0.0) == (2, 4, 3)
    draws = iter([2, 0xFFFFFF00, 8])  # user 2; not <= 0.5: a negative; 8 % 5 = 3
    assert draw_sample(draws, philox_uniform_le, X, 0, 3, False, 0.5) == (2, 3, 0.0)
    draws = iter([5, 0x7FFFFF00, 6])  # user 2; 0.49999994 <= 0.5: a positive at position 0 (item 1, rating 2)
    assert draw_sample(draws, philox_uniform_le, X, 0, 3, False, 0.5) == (2, 1, 2.0)


# ---------------------------------------------------------------------------------------------------------------------
# streams on the device

N_USERS, N_ITEMS, LO, HI = 400, 60, 100, 300


def _shard_urm():
    """Ratings; inside and outside [LO, HI) some users have an empty profile (user redraws) and some have every item; the
    rest are dense enough that negative draws are often rejected."""
    X = synth_urm(N_USERS, N_ITEMS, 0.3, seed=17, values="ratings").tolil()
    for u in (0, 5, 120, 121, 200, 299, 350):
        X[u, :] = 0
    for u in (1, 101, 150, 298, 399):
        X[u, :] = 3.0
    X = sps.csr_matrix(X.tocsr(), dtype=np.float32)
    X.eliminate_zeros()
    X.sort_indices()
    return X


def _glibc_urm(shape):
    """The shapes under which the device replay of the glibc stream extends its buffer and carries its unread tail."""
    if shape == "sparse":
        return synth_urm(3000, 900, 0.01, seed=21, values="ratings")
    if shape == "dense_profiles":
        return synth_urm(200, 40, 0.7, seed=22, values="ratings")   # most negative draws are rejected
    if shape == "cold_users":
        return synth_urm(500, 200, 0.004, seed=23, values="ratings")  # most users have an empty profile
    return _shard_urm()


def _mf(X, algo, **kw):
    from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch
    args = dict(algorithm_name=algo, n_factors=8, batch_size=8, learning_rate=0.01, random_seed=9, sgd_mode="sgd")
    args.update(kw)
    return MatrixFactorization_Cython_Epoch(X, **args)


def _slim(X, **kw):
    from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch
    return SLIM_BPR_Cython_Epoch(X, learning_rate=0.01, symmetric=False, sgd_mode="sgd", random_seed=5, **kw)


def _assert_stream(got, want):
    assert len(got[0]) == len(want[0]) > 0
    for a, b in zip(got, want):
        assert np.array_equal(a, b), int(np.flatnonzero(a != b)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("algo,quota", [("MF_BPR", 0.5), ("FUNK_SVD", 0.0), ("FUNK_SVD", 0.4)])
def test_mf_philox_stream(algo, quota):
    X = _shard_urm()
    g = _mf(X, algo, sampler="philox", negative_interactions_quota=quota)
    for epoch in range(3):
        g.epochIteration_Cython()
        want = philox_stream(X, g.samples_last_epoch(), 9, epoch, MF_C3, algo == "MF_BPR", quota)
        _assert_stream(g.get_samples(), want)
    if algo == "FUNK_SVD":
        u, i, r = want
        assert np.array_equal(r, X.toarray()[u, i])  # the rating of a positive, 0 for a negative
        assert (quota == 0) == (r != 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("stream_id", [0, 1])
@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_mf_user_shard_philox_stream(algo, stream_id):
    X = _shard_urm()
    g = _mf(X, algo, sampler="philox", hogwild=True, negative_interactions_quota=0.4, random_seed=0xFFFFFFF0)
    g.set_user_shard(LO, HI, 203, stream_id=stream_id)
    seed = (0xFFFFFFF0 + 0x9E3779B9 * stream_id) & M32
    for epoch in range(3):
        g.epochIteration_Cython()
        assert g.samples_last_epoch() == 200  # 203 samples per epoch, whole batches of 8
        _assert_stream(g.get_samples(), philox_stream(X, 200, seed, epoch, MF_C3, algo == "MF_BPR", 0.4, LO, HI - LO))


@pytest.mark.gpu
@pytest.mark.parametrize("hogwild", [False, True])
def test_slim_philox_stream(hogwild):
    X = _shard_urm()
    g = _slim(X, sampler="philox", hogwild=hogwild)
    for epoch in range(3):
        g.epochIteration_Cython()
        _assert_stream(g.get_samples(), philox_stream(X, N_USERS, 5, epoch, SLIM_C3))


@pytest.mark.gpu
def test_slim_column_sharded_philox_stream():
    from recsys2019_deeplearning_evaluation_b200 import _lib
    from recsys2019_deeplearning_evaluation_b200.dist import ShardedSLIM_BPR
    X = _shard_urm()
    s = ShardedSLIM_BPR(X, batch_size=64, learning_rate=0.01, sgd_mode="sgd", random_seed=11, col_range=(10, 40),
                        world_rank=(1, 0))
    for epoch in range(3):
        s.epochIteration_Cython()  # a world of one: the shard's partial sums are the whole sums
        got = [np.empty(N_USERS, np.int32) for _ in range(3)]
        _lib.check(_lib.load().b200_slim_get_samples(s._h, *(_lib.ptr(a) for a in got)))
        _assert_stream(got, philox_stream(X, N_USERS, 11, epoch, SLIM_C3))


GLIBC_SHAPES = ["sparse", "dense_profiles", "cold_users", "shard"]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GLIBC_SHAPES)
@pytest.mark.parametrize("host", ["1", "0"])
@pytest.mark.parametrize("algo", ["MF_BPR", "FUNK_SVD"])
def test_mf_glibc_stream_is_the_oracles(algo, host, shape, monkeypatch):
    """B200REC_GLIBC_HOST=1: the sequential host replay; =0: the stream resolved on the device."""
    from oracle.sgd_oracle import MFOracle
    X = _glibc_urm(shape)
    kw = dict(n_factors=8, batch_size=50, learning_rate=0.01, random_seed=77, sgd_mode="sgd", negative_interactions_quota=0.35)
    monkeypatch.setenv("B200REC_GLIBC_HOST", host)
    g = _mf(X, algo, **kw)
    n = ((X.shape[0] if algo == "MF_BPR" else X.nnz) // 50 + 1) * 50
    o = MFOracle(X, algorithm_name=algo, record=2 * n, **kw)
    dense = X.toarray()
    for epoch in range(2):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
        assert g.samples_last_epoch() == n
        u, i, third = g.get_samples()
        ou, oi, oj = (a[epoch * n:(epoch + 1) * n] for a in o.recorded())
        _assert_stream((u, i), (ou, oi))
        if algo == "MF_BPR":
            assert np.array_equal(third, oj)
        else:
            assert np.array_equal(third, dense[u, i])  # the rating of a positive, 0 for a negative


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GLIBC_SHAPES)
def test_slim_glibc_stream_is_the_oracles(shape):
    from oracle.sgd_oracle import SLIMOracle
    X = _glibc_urm(shape)
    n = X.shape[0]
    g = _slim(X)
    o = SLIMOracle(X, learning_rate=0.01, symmetric=False, sgd_mode="sgd", random_seed=5, record=2 * n)
    for epoch in range(2):
        g.epochIteration_Cython()
        o.epochIteration_Cython()
        _assert_stream(g.get_samples(), [a[epoch * n:(epoch + 1) * n] for a in o.recorded()])
