"""Development timing of the fp64 LU path of EASE_R on one GPU:
    python tools/dev_ease_lu_bench.py [--out FILE.json]
1. the FP64 tensor-core GEMM (b200_debug_dgemm_device kind 0) at 8192^3, TFLOP/s against the 67 TFLOP/s FP64 tensor-core
   figure of the H100 SXM data sheet;
2. b200_lu_inverse_device alone at n_pad = 3712 and 17792 on a seeded non-symmetric well-conditioned matrix, as 2 n^3 / t;
3. EASE_R_Recommender.fit() on synth_config("C2", values="ratings") at l2_norm = 1e3 (indefinite Gram: Cholesky attempt,
   then the LU path), best of several fits after a warm-up.
The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from recsys2019_deeplearning_evaluation_b200 import _lib

FP64_TC_DATASHEET_TFLOPS = 67.0


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = _lib.load()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {"card": card()}
    print("card: %s" % res["card"], flush=True)

    n = 8192
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn((n, n), generator=g, device="cuda", dtype=torch.float64)
    B = torch.randn((n, n), generator=g, device="cuda", dtype=torch.float64)
    C = torch.empty((n, n), device="cuda", dtype=torch.float64)
    ms = timed(lambda: _lib.check(L.b200_debug_dgemm_device(0, n, n, n, 1.0, A.data_ptr(), n, B.data_ptr(), n, 0.0, C.data_ptr(), n, st)), 5)
    best = min(ms[1:])
    tf = 2.0 * n ** 3 / best / 1e9
    res["dgemm_8192"] = {"ms_all": ms, "ms": best, "tflops": tf, "frac_of_datasheet_fp64_tc": tf / FP64_TC_DATASHEET_TFLOPS}
    print("DMMA GEMM 8192^3: %.2f ms, %.1f TFLOP/s (%.0f%% of the %.0f TFLOP/s data-sheet figure)" % (
        best, tf, 100 * tf / FP64_TC_DATASHEET_TFLOPS, FP64_TC_DATASHEET_TFLOPS), flush=True)
    del A, B, C

    for n_pad in (3712, 17792):
        rng = np.random.default_rng(n_pad)
        M0 = torch.from_numpy(rng.standard_normal((n_pad, n_pad))).cuda()
        M0 += 2.0 * np.sqrt(n_pad) * torch.eye(n_pad, dtype=torch.float64, device="cuda").flip(0)  # well conditioned, needs pivots
        Aw = torch.empty_like(M0)
        W = torch.empty(2 * n_pad * n_pad, dtype=torch.float64, device="cuda")
        ms = []
        for _ in range(4):  # the first is the warm-up
            Aw.copy_(M0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(L.b200_lu_inverse_device(Aw.data_ptr(), n_pad, W.data_ptr(), st))
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        # residual of the last inverse: max |A X - I| (the check runs on the device in fp64)
        resid = (M0 @ Aw - torch.eye(n_pad, dtype=torch.float64, device="cuda")).abs().max().item()
        best = min(ms[1:])
        tf = 2.0 * n_pad ** 3 / best / 1e9
        res["lu_inverse_%d" % n_pad] = {"ms_all": ms, "ms": best, "tflops_2n3": tf, "max_abs_AX_minus_I": resid}
        print("b200_lu_inverse_device n_pad=%d: %.1f ms, %.1f TFLOP/s (2n^3/t), max|AX-I| = %.2e" % (n_pad, best, tf, resid), flush=True)
        del M0, Aw, W
        torch.cuda.empty_cache()

    from recsys2019_deeplearning_evaluation_b200.recommenders import EASE_R_Recommender
    from recsys2019_deeplearning_evaluation_b200.synth import synth_config
    X = synth_config("C2", values="ratings")
    r = EASE_R_Recommender(X, verbose=False)
    secs = []
    for _ in range(5):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r.fit(topK=None, l2_norm=1e3, verbose=False)
        torch.cuda.synchronize()
        secs.append(time.perf_counter() - t)
    res["ease_c2_ratings_fit"] = {"s_all": secs, "s": min(secs[1:]), "shape": list(X.shape), "nnz": int(X.nnz)}
    print("EASE_R fit, C2 ratings %dx%d, l2_norm=1e3: best %.1f ms of %s (first = warm-up)" % (
        X.shape[0], X.shape[1], 1e3 * min(secs[1:]), ["%.1f" % (1e3 * s) for s in secs]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
