"""Development timing of PureSVDRecommender.fit (csrc/puresvd.cu) on one GPU against scikit-learn on the CPU:
    python tools/dev_puresvd_bench.py [--cases C2:100,C2:350,...] [--sklearn C2,C3] [--out FILE.json]
For each synthetic config and number of factors (default C2, C3 and C4 at 100 and 350 factors, C5 at 100; seed 1):
  - GPU: a whole fit() by the host clock (sketch draw, upload, transpose, SVD, download; fit ends in a synchronise), the best
    of three after a warm-up fit;
  - device time per phase, from one more fit under torch.profiler (CUDA activities), by kernel name: transpose (the CSR
    transpose and its radix sort), spmm, gram + orth (Gram partials and sums, SVQB's small kernels), eigensolve (Jacobi
    rounds, convergence checks, sort), products (tall x small, signs);
  - the algorithmic SpMM rate: (2 n_iter + 2) SpMMs, each reading nnz * 8 bytes of column ids and values and gathering
    nnz * 4 * n_random bytes of the dense operand, over the spmm kernels' device time;
  - scikit-learn's float32 randomized_svd on the same URM and the same host (configs in --sklearn, default C2 and C3).
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from recsys2019_deeplearning_evaluation_b200.recommenders import PureSVDRecommender
from recsys2019_deeplearning_evaluation_b200.synth import synth_config

PHASES = [("transpose", ("transpose", "row_of", "count_cols", "RadixSort", "DeviceScan")), ("spmm", ("spmm_kernel",)),
          ("gram+orth", ("gram_partial", "sum_splits", "svqb_", "identity_kernel")),
          ("eigensolve", ("jacobi_round", "offnorm", "sort_desc")),
          ("products", ("tall_small", "final_coef", "flip_sign", "scale_cols"))]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def phase_ms(X, k):
    from torch.profiler import ProfilerActivity, profile
    r = PureSVDRecommender(X, verbose=False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r.fit(num_factors=k, random_seed=1)
        torch.cuda.synchronize()
    out = {name: 0.0 for name, _ in PHASES}
    out["other"] = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if not t or ev.key.startswith(("Memcpy", "Memset", "cudaMemcpy", "cudaMemset")):
            continue
        name = next((n for n, keys in PHASES if any(s in ev.key for s in keys)), "other")
        out[name] += t / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="C2:100,C2:350,C3:100,C3:350,C4:100,C4:350,C5:100")
    ap.add_argument("--sklearn", default="C2,C3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = {"card": card()}
    print(json.dumps(info), flush=True)
    rows = []
    for case in a.cases.split(","):
        cfg, k = case.split(":")
        k = int(k)
        X = synth_config(cfg)
        n_random = k + 10
        n_iter = 7 if k < 0.1 * min(X.shape) else 4
        r = PureSVDRecommender(X, verbose=False)
        r.fit(num_factors=k, random_seed=1)  # warm-up
        walls = []
        for _ in range(3):
            r = PureSVDRecommender(X, verbose=False)
            torch.cuda.synchronize()
            t = time.perf_counter()
            r.fit(num_factors=k, random_seed=1)
            walls.append(time.perf_counter() - t)
        ph = phase_ms(X, k)
        spmm_bytes = (2 * n_iter + 2) * X.nnz * (4 * n_random + 8)
        row = {"config": cfg, "shape": list(X.shape), "nnz": int(X.nnz), "factors": k, "n_iter": n_iter, "fit_s": min(walls),
               "fit_s_all": walls, "phase_ms": ph, "spmm_GB": spmm_bytes / 1e9,
               "spmm_GBps": spmm_bytes / 1e9 / (ph["spmm"] / 1e3) if ph["spmm"] > 0 else None}
        if cfg in a.sklearn.split(","):
            from oracle.puresvd_oracle import puresvd_reference
            t = time.perf_counter()
            puresvd_reference(X, k, random_seed=1, dtype=np.float32)
            row["sklearn_f32_s"] = time.perf_counter() - t
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"info": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
