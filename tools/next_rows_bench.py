"""Timings of the SURVEY.md 8(f).4 trainers at BASELINE shapes, one JSON object per line, with the CPU side timed beside them
on a bounded sample (the oracle port for the SGD trainers, scikit-learn's ElasticNet -- what the reference calls -- for SLIM
ElasticNet).
    python tools/next_rows_bench.py [--no-c4] [--no-c5] [--only-slim-tree]
--only-slim-tree runs the SLIM-BPR tree-mode legs alone (C2, then the C5 shape unless --no-c5).
"""
import json, os, sys, time, warnings
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.sparse as sps
import torch

from recsys2019_deeplearning_evaluation_b200.synth import synth_config
from recsys2019_deeplearning_evaluation_b200 import recommenders as R
from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch
from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch


def emit(**kw):
    print(json.dumps(kw), flush=True)


def sync():
    torch.cuda.synchronize()


X2 = synth_config("C2", values="ratings")
nu, ni = X2.shape
emit(bench="URM C2", shape=list(X2.shape), nnz=int(X2.nnz))

only_asy = "--only-asy" in sys.argv
only_tree = "--only-slim-tree" in sys.argv


def gpu_info():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa
        return repr(ex)


def slim_tree_c2():
    # ---- SLIM-BPR tree mode, C2 (adagrad, topK 200: the reference's configs[1] hyper-parameters, sparse-weights mode)
    kws = dict(train_with_sparse_weights=True, learning_rate=1e-4, li_reg=0.0, lj_reg=0.0, topK=200, sgd_mode="adagrad", random_seed=42)
    g = SLIM_BPR_Cython_Epoch(sps.csr_matrix(X2), **kws)
    g.epochIteration_Cython(); sync()
    ts = []
    for _ in range(5):
        t = time.perf_counter(); g.epochIteration_Cython(); sync(); ts.append(time.perf_counter() - t)
    t = time.perf_counter(); S = g.get_S(); t_get = time.perf_counter() - t
    emit(bench="SLIM-BPR tree mode epoch C2", samples=nu, seconds_median=float(np.median(ts)), samples_per_s=nu / float(np.median(ts)), get_S_s=t_get,
         nnz=int(S.nnz), cuts_per_epoch=4, epochs_s=ts, gpu=gpu_info())
    g._dealloc()


def slim_tree_c5():
    # ---- SLIM-BPR tree mode at the C5 shape (1 M users x 200 K items, K = 200, adagrad): the dense S would be 160 GB.  One
    # epoch timed plain, one under torch.profiler for the split: structure build (key emission, sort, unique, rowptr, value
    # carry, slot map) / the sequential kernel / the cuts
    X5 = synth_config("C5", values="ratings")
    kws = dict(train_with_sparse_weights=True, learning_rate=1e-4, topK=200, sgd_mode="adagrad", random_seed=42)
    g = SLIM_BPR_Cython_Epoch(sps.csr_matrix(X5), **kws)
    sync(); t = time.perf_counter(); g.epochIteration_Cython(); sync(); t_epoch = time.perf_counter() - t
    cells_epoch = g.tree_cells()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t = time.perf_counter(); g.epochIteration_Cython(); sync(); t_prof = time.perf_counter() - t
    split = {"build": 0.0, "sequential": 0.0, "cut": 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if us <= 0:
            continue
        key = "sequential" if "slim_sequential_kernel" in ev.key else ("cut" if "slim_tree_cut" in ev.key else "build")
        split[key] += us * 1e-6
    t = time.perf_counter(); S = g.get_S(); t_get = time.perf_counter() - t
    emit(bench="SLIM-BPR tree mode epoch C5 shape", shape=list(X5.shape), nnz_urm=int(X5.nnz), samples=int(X5.shape[0]), epoch_s=t_epoch,
         epoch_profiled_s=t_prof, device_s_build=split["build"], device_s_sequential=split["sequential"], device_s_cut=split["cut"],
         get_S_s=t_get, cells_after_epoch=cells_epoch, cells_after_get_S=g.tree_cells(), structure_bytes_after_epoch=12 * cells_epoch,
         nnz=int(S.nnz), gpu=gpu_info())
    g._dealloc()


if only_tree:
    slim_tree_c2()
    if "--no-c5" not in sys.argv:
        slim_tree_c5()
    sys.exit(0)
if only_asy:
    for mode in ("sgd", "adagrad", "adam"):
        for f in (32, 128):
            g = MatrixFactorization_Cython_Epoch(X2, n_factors=f, algorithm_name="ASY_SVD", batch_size=1, learning_rate=1e-3, random_seed=42,
                                                 sgd_mode=mode, use_bias=True, negative_interactions_quota=0.2, user_reg=1e-3, item_reg=1e-3)
            g.epochIteration_Cython(); sync()
            ms = g.last_epoch_ms()
            emit(bench="AsySVD epoch C2 f=%d %s" % (f, mode), samples=int(X2.nnz + 1), kernel_s=ms * 1e-3, samples_per_s=(X2.nnz + 1) / (ms * 1e-3),
                 us_per_sample=ms * 1e3 / (X2.nnz + 1), mean_profile=float(X2.nnz / nu))
            g._dealloc()
    sys.exit(0)

# ---- SLIM ElasticNet, C2 (the MovieLens-1M shape the reference's own sweep runs it on)
kw = dict(l1_ratio=0.1, alpha=1e-3, positive_only=True, topK=100)
rec = R.SLIMElasticNetRecommender(X2, verbose=False)
rec.fit(**kw); sync()
t = time.perf_counter(); rec.fit(**kw); sync(); dt = time.perf_counter() - t
it = rec._n_iter.cpu().numpy()
emit(bench="SLIM ElasticNet fit C2", seconds=dt, items_per_s=ni / dt, nnz=int(rec.W_sparse.nnz), passes_mean=float(it.mean()), passes_max=int(it.max()), **kw)
W_gpu = rec.W_sparse.tocsc()
try:  # what the reference runs per item (SLIMElasticNetRecommender.py:49-93), on a sample of items
    from sklearn.linear_model import ElasticNet
    Xc = sps.csc_matrix(X2, dtype=np.float32)
    cols = list(range(0, ni, ni // 16))[:16]
    m = ElasticNet(alpha=kw["alpha"], l1_ratio=kw["l1_ratio"], positive=True, fit_intercept=False, copy_X=False, precompute=True,
                   selection="random", max_iter=100, tol=1e-4)
    t = time.perf_counter(); worst = 0.0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for j in cols:
            y = Xc[:, j].toarray()
            s, e = Xc.indptr[j], Xc.indptr[j + 1]
            keep = Xc.data[s:e].copy(); Xc.data[s:e] = 0.0
            m.fit(Xc, y)
            Xc.data[s:e] = keep
            coef = np.asarray(m.coef_).ravel()
            got = np.asarray(W_gpu[:, j].todense()).ravel()
            nzg = got != 0
            worst = max(worst, float(np.abs(coef[nzg] - got[nzg]).max()) if nzg.any() else 0.0)
    dt_cpu = time.perf_counter() - t
    emit(bench="SLIM ElasticNet sklearn per item C2 (CPU, the reference's call)", items=len(cols), seconds=dt_cpu, items_per_s=len(cols) / dt_cpu,
         full_fit_estimate_s=dt_cpu / len(cols) * ni, max_abs_diff_to_gpu_on_kept_entries=worst)
except Exception as ex:  # noqa
    emit(bench="sklearn leg failed", error=repr(ex))
del rec

# ---- AsySVD, C2: one epoch = nnz + 1 strictly sequential samples
for mode in ("sgd", "adagrad"):
    g = MatrixFactorization_Cython_Epoch(X2, n_factors=32, algorithm_name="ASY_SVD", batch_size=1, learning_rate=1e-3, random_seed=42,
                                         sgd_mode=mode, use_bias=True, negative_interactions_quota=0.2, user_reg=1e-3, item_reg=1e-3)
    t = time.perf_counter(); g.epochIteration_Cython(); sync(); wall = time.perf_counter() - t
    ms = g.last_epoch_ms()
    emit(bench="AsySVD epoch C2 f=32 %s" % mode, samples=int(X2.nnz + 1), kernel_s=ms * 1e-3, wall_s=wall, samples_per_s=(X2.nnz + 1) / (ms * 1e-3),
         us_per_sample=ms * 1e3 / (X2.nnz + 1), mean_profile=float(X2.nnz / nu))
    g._dealloc()
from oracle.sgd_oracle import MFOracle  # CPU side: the C port of the reference's loop, on a slice of the epoch
Xs = X2[:600]
o = MFOracle(Xs, n_factors=32, algorithm_name="ASY_SVD", batch_size=1, learning_rate=1e-3, random_seed=42, sgd_mode="adagrad", use_bias=True,
             negative_interactions_quota=0.2, user_reg=1e-3, item_reg=1e-3)
t = time.perf_counter(); n = o.epochIteration_Cython(); dt = time.perf_counter() - t
emit(bench="AsySVD C port of the reference loop (CPU, 1 thread), 600 users of C2", samples=int(n), seconds=dt, samples_per_s=n / dt)

slim_tree_c2()
if "--no-c5" not in sys.argv:
    slim_tree_c5()

# ---- SLIM ElasticNet, C4 (480 K x 17.7 K): the Gram matrix is the EASE_R one; 3 * n * 4 bytes = 208 KB of shared memory per CTA
if "--no-c4" not in sys.argv:
    X4 = synth_config("C4", values="binary")
    rec = R.SLIMElasticNetRecommender(X4, verbose=False)
    kw4 = dict(l1_ratio=0.1, alpha=1e-4, positive_only=True, topK=100)
    sync(); t = time.perf_counter(); rec.fit(**kw4); sync(); dt = time.perf_counter() - t
    it = rec._n_iter.cpu().numpy()
    emit(bench="SLIM ElasticNet fit C4", seconds=dt, items_per_s=X4.shape[1] / dt, nnz=int(rec.W_sparse.nnz), passes_mean=float(it.mean()),
         passes_max=int(it.max()), **kw4)
