"""SLIM ElasticNet against a sparse Gram matrix (gram_csr_device + b200_slim_enet_sparse_device), on the GPU.

  python tools/dev_enet_sparse_bench.py [--reps 2] [--large-users 1000000] [--large-items 150000] [--per-user 20]
                                        [--popularity 0.8] [--configs C2,C4] [--paths dense,sparse]

First a long-tailed catalogue that only the sparse path fits (Zipf item popularity, about --per-user interactions per
user, ratings): wall time of the fit, its Gram and solve phases, nnz of X^T X, and the device-memory high-water (polled
mem_get_info) against the dense path's computed footprint.  Then the --configs shapes with both paths alternated in one
process (the sparse one forced through the free-memory query): fit time of each, the first round's included (--reps 0
runs that round alone: a dense C4 fit takes minutes), and max |W_dense - W_sparse|.  Prints
the card name and power limit of the same run, one JSON line at the end."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from recsys2019_deeplearning_evaluation_b200 import recommenders as R  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm  # noqa: E402

FIT = dict(l1_ratio=0.1, alpha=1e-3, positive_only=True, topK=100)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def n_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


class FreePoll:
    """Lowest free device memory seen while the block runs (mem_get_info every 5 ms from a second thread)."""

    def __enter__(self):
        self.low, self.stop = torch.cuda.mem_get_info()[0], False

        def run():
            torch.cuda.set_device(torch.cuda.current_device())
            while not self.stop:
                self.low = min(self.low, torch.cuda.mem_get_info()[0])
                time.sleep(0.005)
        self.t = threading.Thread(target=run, daemon=True)
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop = True
        self.t.join()


class Phases:
    """Wall time of gram_csr_device inside the fit (the rest of _fit_sparse is the solve and the table's assembly)."""

    def __enter__(self):
        self.real, self.gram_s, self.nnz = R.gram_csr_device, None, None

        def timed(URM):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = self.real(URM)
            torch.cuda.synchronize()
            self.gram_s, self.nnz = time.perf_counter() - t, int(out[0][-1])
            return out
        R.gram_csr_device = timed
        return self

    def __exit__(self, *a):
        R.gram_csr_device = self.real


def fit_timed(X, sparse):
    real = torch.cuda.mem_get_info
    if sparse:  # a free-memory figure just below the dense path's footprint routes the fit to the sparse Gram
        dense = R.slim_enet_dense_bytes(X.shape[1], FIT["topK"], n_sms(), R.ease_urm_bytes(X))
        torch.cuda.mem_get_info = lambda *a: (dense - 1, real()[1])
    try:
        r = R.SLIMElasticNetRecommender(X, verbose=False)
        torch.cuda.synchronize()
        t = time.perf_counter()
        r.fit(**FIT)
        torch.cuda.synchronize()
        return r, time.perf_counter() - t
    finally:
        torch.cuda.mem_get_info = real


def large(n_users, n_items, per_user, popularity):
    X = synth_urm(n_users, n_items, per_user / n_items, seed=7, values="ratings", popularity=popularity)
    torch.cuda.empty_cache()
    free0, total = torch.cuda.mem_get_info()
    dense = R.slim_enet_dense_bytes(n_items, FIT["topK"], n_sms(), R.ease_urm_bytes(X))
    assert R.slim_enet_sparse_for_device(n_items, free0, True, True, FIT["topK"], n_sms(), R.ease_urm_bytes(X)), (free0, dense)
    with FreePoll() as poll, Phases() as ph:
        r, t = fit_timed(X, False)
    it = r._n_iter.cpu().numpy()
    return {"n_users": n_users, "n_items": n_items, "urm_nnz": int(X.nnz), "gram_nnz_offdiag": ph.nnz, "fit_s": t,
            "gram_s": ph.gram_s, "solve_and_table_s": t - ph.gram_s, "free_before": int(free0), "total": int(total),
            "high_water_bytes": int(free0 - poll.low), "dense_footprint_bytes": int(dense), "W_nnz": int(r.W_sparse.nnz),
            "passes_mean": float(it.mean()), "passes_max": int(it.max())}


def paired(name, reps, paths):
    X = synth_config(name, values="ratings")
    times = {path: [] for path in paths}
    W, nnz = {}, None
    for rep in range(reps + 1):  # the first round warms both paths up: the first time of each list
        for path in paths:
            with Phases() as ph:
                r, t = fit_timed(X, path == "sparse")
            if path == "sparse":
                nnz = ph.nnz
            times[path].append(t)
            W[path] = r.W_sparse.tocsc()
            W[path].sort_indices()
            print("%s %-6s fit %.3f s" % (name, path, t), flush=True)
    out = {"shape": list(X.shape), "gram_nnz_offdiag": nnz, "times_s": times}
    if len(W) == 2:
        d = W["dense"] - W["sparse"]
        out.update(max_abs_dW=float(np.abs(d.data).max()) if d.nnz else 0.0, max_abs_W=float(np.abs(W["dense"].data).max()),
                   same_pattern=bool(np.array_equal(W["dense"].indptr, W["sparse"].indptr)
                                     and np.array_equal(W["dense"].indices, W["sparse"].indices)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--large-users", type=int, default=1_000_000)
    ap.add_argument("--large-items", type=int, default=150_000)  # 0 skips the large catalogue
    ap.add_argument("--per-user", type=float, default=20.0)
    ap.add_argument("--popularity", type=float, default=0.8)
    ap.add_argument("--configs", default="C2,C4")
    ap.add_argument("--paths", default="dense,sparse")  # one of them alone when a call has room for only one C4 fit
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    out = {"card": card()}
    print(out["card"], flush=True)
    if a.large_items > 0:
        out["large"] = large(a.large_users, a.large_items, a.per_user, a.popularity)
        print(json.dumps(out["large"]), flush=True)
    for name in filter(None, a.configs.split(",")):
        out[name] = paired(name, a.reps, a.paths.split(","))
        print(json.dumps(out[name]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
