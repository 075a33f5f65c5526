"""Epoch timings of the SGD trainers where their sample streams are drawn, for A/B runs of two checkouts in one session:
    python tools/dev_sampler_bench.py [--root CHECKOUT] [--steps K]
bpr:    bench.py's BPR-MF leg at C5 (device ms per epoch of every mode, the C3 rows); the Philox sample kernel is inside the
        timed region of the Philox modes, the device-resolved glibc stream inside the wall time of the glibc mode; the
        device time of the kernels that resolve the glibc stream from a torch.profiler run of its own.
slim:   host wall time of one SLIM-BPR sequential epoch on the glibc stream at C2 (host replay + upload + kernel).
asysvd: host wall time of one AsySVD epoch on a C2-shaped URM at 0.5 % density (host replay + upload + kernel).
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="checkout to import")
ap.add_argument("--steps", type=int, default=5)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import bench  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.mf_epoch import MatrixFactorization_Cython_Epoch  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.slim_bpr_epoch import SLIM_BPR_Cython_Epoch  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm  # noqa: E402


def wall_ms(m, steps):
    m.epochIteration_Cython()
    torch.cuda.synchronize()
    out = []
    for _ in range(steps):
        t = time.perf_counter()
        m.epochIteration_Cython()
        torch.cuda.synchronize()
        out.append(1e3 * (time.perf_counter() - t))
    m._dealloc()
    return {"median_ms": float(np.median(out)), "min_ms": float(min(out))}


def glibc_replay_kernels_ms(X, steps):
    """Device time per epoch of the kernels that resolve the glibc stream (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    m = MatrixFactorization_Cython_Epoch(X, n_factors=128, algorithm_name="MF_BPR", batch_size=1000, learning_rate=1e-3,
                                         random_seed=42, sgd_mode="sgd")
    m.epochIteration_Cython()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            m.epochIteration_Cython()
        torch.cuda.synchronize()
    m._dealloc()
    out = {}
    for e in prof.key_averages():
        for k in ("glibc_len_kernel", "glibc_double_kernel", "glibc_emit_kernel"):
            if k in e.key:
                out[k] = round(out.get(k, 0.0) + e.device_time_total / 1e3 / steps, 4)
    return out


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()[0]
res = {"root": os.path.abspath(args.root), "card": card}
X5 = synth_config("C5")
bpr = bench.bpr_leg(argparse.Namespace(steps=args.steps, workload="C5", no_cpu_baseline=True), X5)
res["bpr"] = {k: round(v["device_ms_per_epoch"], 3) for k, v in bpr["modes"].items()}
res["bpr"]["glibc_e2e_ms"] = round(1e3 * bpr["modes"]["minibatch_bs1000_glibc_stream"]["samples_per_epoch"]
                                   / bpr["modes"]["minibatch_bs1000_glibc_stream"]["e2e_value"], 3)
res["bpr"].update({"c3_" + k: round(v["device_ms_per_epoch"], 3) for k, v in bpr["c3"].items() if isinstance(v, dict)})
res["glibc_replay_kernels_ms"] = glibc_replay_kernels_ms(X5, args.steps)
res["slim_glibc_c2"] = wall_ms(SLIM_BPR_Cython_Epoch(synth_config("C2"), topK=200, symmetric=True, sgd_mode="adagrad",
                                                     learning_rate=1e-4, random_seed=42), args.steps)
res["asysvd_glibc"] = wall_ms(MatrixFactorization_Cython_Epoch(synth_urm(6040, 3706, 0.005, seed=42, values="ratings"),
                                                               algorithm_name="ASY_SVD", n_factors=32, batch_size=1,
                                                               learning_rate=1e-3, random_seed=42, sgd_mode="adagrad"), args.steps)
print(json.dumps(res), flush=True)
