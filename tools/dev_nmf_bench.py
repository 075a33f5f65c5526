"""Development timing of NMFRecommender's device solves (csrc/nmf.cu) on one GPU against scikit-learn on the CPU:
    python tools/dev_nmf_bench.py [--configs C2,C3] [--factors 100,350] [--out FILE.json]
For each synthetic config, number of factors and (solver, loss) in (mu, Frobenius), (mu, KL), (cd, Frobenius):
  - GPU: the fit solve and the transform solve of NMFRecommender.fit (tol 1e-4, max_iter 200) from the random init of seed 7,
    after a warm-up solve of 2 iterations.  The URM, X^T and the factors are uploaded first; then the C call alone is timed,
    by the host clock (the call ends in a stream synchronise) and by CUDA events (device time, divided by the iterations).
    Then a whole NMFRecommender.fit() is timed by the host clock (init, uploads, both solves, downloads).  Algorithmic bytes
    per fit iteration come from the shapes (below);
  - scikit-learn, float32, on the same URM: at C2 with 100 factors the full fit + transform for the two Frobenius cases;
    everywhere else a fixed number of fit and of transform iterations (tol 0), extrapolated to the GPU's iteration counts
    and labelled so.
Bytes per fit iteration: each of the two SpMMs (X H^T and X^T W; for KL the fused SDDMM + SpMM) gathers nnz * f * 4 bytes of
the other factor and reads nnz * 8 bytes of indices and values; each factor is read by its Gram or column sum and read and
written by its update, with X H^T read back once: 5 * (n_users + n_items) * f * 4.
The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.sparse as sps
import torch

from recsys2019_deeplearning_evaluation_b200.recommenders import NMFRecommender, _dev_csr, nmf_random_init
from recsys2019_deeplearning_evaluation_b200.synth import synth_config

CASES = [("multiplicative_update", "frobenius"), ("multiplicative_update", "kullback-leibler"), ("coordinate_descent", "frobenius")]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def gpu_solve(r, W, Ht, d_xt, update_h, max_iter=None, tol=None):
    """Uploads W and Ht, then times the C call alone: (n_iter, wall seconds of the call, device ms from CUDA events)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    r._urm_device()
    r._d_nmf_W = torch.from_numpy(np.ascontiguousarray(W, np.float32)).to(dev)
    r._d_nmf_Ht = torch.from_numpy(np.ascontiguousarray(Ht, np.float32)).to(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    e0.record()
    n_iter, _ = r._solve_device(d_xt, update_h, max_iter=max_iter, tol=tol)
    e1.record()
    torch.cuda.synchronize()
    return n_iter, time.perf_counter() - t, e0.elapsed_time(e1)


def sklearn_iters(X, W, H, solver, beta_loss, k, update_h):
    from sklearn.decomposition._nmf import _fit_coordinate_descent, _fit_multiplicative_update
    W, H = W.copy(), H.copy()
    t = time.perf_counter()
    if solver == "coordinate_descent":
        _fit_coordinate_descent(X, W, H, tol=0, max_iter=k, update_H=update_h)
    else:
        _fit_multiplicative_update(X, W, H, beta_loss=beta_loss, max_iter=k, tol=0, update_H=update_h)
    return (time.perf_counter() - t) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C3")
    ap.add_argument("--factors", default="100,350")
    ap.add_argument("--sk-iters", type=int, default=3,
                    help="iterations scikit-learn is timed on where it is extrapolated; 0 skips scikit-learn")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = {"card": card(), "rows": []}
    print("card:", out["card"], flush=True)
    for cfg in args.configs.split(","):
        X = sps.csr_matrix(synth_config(cfg), dtype=np.float32)
        n_u, n_i, nnz = X.shape[0], X.shape[1], X.nnz
        for f in (int(v) for v in args.factors.split(",")):
            W0, H0 = nmf_random_init(X, f, 7)
            for solver, beta_loss in CASES:
                r = NMFRecommender(X, verbose=False)
                r.solver, r.beta_loss = solver, beta_loss
                d_xt = _dev_csr(X.T)
                gpu_solve(r, W0, H0.T, d_xt, True, max_iter=2, tol=0.0)  # warm-up
                n_fit, t_fit, ms_fit = gpu_solve(r, W0, H0.T, d_xt, True)
                Ht = r._d_nmf_Ht.cpu().numpy()
                Wt0 = (np.full((n_u, f), np.sqrt(X.mean() / f), np.float32) if solver == "multiplicative_update"
                       else np.zeros((n_u, f), np.float32))
                n_tr, t_tr, ms_tr = gpu_solve(r, Wt0, Ht, None, False)
                del d_xt
                torch.cuda.synchronize()
                t = time.perf_counter()
                r.fit(num_factors=f, solver=solver, beta_loss=beta_loss, random_seed=7)
                fit_wall = time.perf_counter() - t
                bytes_it = 2 * nnz * (f * 4 + 8) + 5 * (n_u + n_i) * f * 4
                row = dict(config=cfg, f=f, solver=solver, beta_loss=beta_loss, n_iter_fit=n_fit, n_iter_transform=n_tr,
                           gpu_fit_call_s=t_fit, gpu_transform_call_s=t_tr, recommender_fit_wall_s=fit_wall,
                           device_ms_per_fit_iter=ms_fit / n_fit, device_ms_per_transform_iter=ms_tr / n_tr,
                           bytes_per_fit_iter=bytes_it, gbps_fit=bytes_it / (ms_fit / n_fit) / 1e6)
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    if args.sk_iters == 0:
                        row.update(sklearn_fit_transform_s=None)  # not measured
                    elif cfg == "C2" and f == 100 and beta_loss == "frobenius":
                        from oracle.nmf_oracle import nmf_reference
                        t = time.perf_counter()
                        _, _, sn, st = nmf_reference(X, f, solver=solver, beta_loss=beta_loss, random_seed=7)
                        row.update(sklearn_fit_transform_s=time.perf_counter() - t, sklearn_n_iter=(sn, st), sklearn_extrapolated=False)
                    else:
                        s_it = sklearn_iters(X, W0, H0, solver, beta_loss, args.sk_iters, True)
                        s_tr = sklearn_iters(X, Wt0, np.ascontiguousarray(Ht.T), solver, beta_loss, args.sk_iters, False)
                        row.update(sklearn_s_per_fit_iter=s_it, sklearn_s_per_transform_iter=s_tr,
                                   sklearn_fit_transform_s=s_it * n_fit + s_tr * n_tr, sklearn_extrapolated=True)
                if row["sklearn_fit_transform_s"] is not None:
                    row["speedup_vs_fit_wall"] = row["sklearn_fit_transform_s"] / fit_wall
                out["rows"].append(row)
                print(json.dumps(row), flush=True)
                del r
                torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
