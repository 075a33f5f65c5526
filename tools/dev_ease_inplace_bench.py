"""The in-place EASE_R fit (b200_ease_inplace_device) against the default path, on the GPU.

  python tools/dev_ease_inplace_bench.py [--reps 2] [--large-users 1000000] [--large-items 100000] [--large-density 0.0005]

C4 (480 K x 17.7 K): the two paths alternate (the in-place one forced through the free-memory query), fit time of each
and max |B_default - B_inplace|.  Then one binary catalogue above the default path's limit, fitted with topK=100 (the
dense B is never copied to the host): wall time, device-memory high-water (polled mem_get_info) against the computed
bound, and (G + D)(e_j - B[:, j]) on 20 sampled columns, computed in fp64 on the host as X^T (X v) with the diagonal
corrected, which must vanish off entry j.  Prints the card name and power limit of the same run, one JSON line at the end."""
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
from recsys2019_deeplearning_evaluation_b200 import slim_bpr_epoch  # noqa: E402
from recsys2019_deeplearning_evaluation_b200.synth import synth_config, synth_urm  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def fit_timed(X, inplace, **kw):
    real = torch.cuda.mem_get_info
    if inplace:  # a free-memory figure just below the default path's peak routes the fit in place
        n = X.shape[1]
        n_pad = -(-n // 128) * 128
        torch.cuda.mem_get_info = lambda *a: (4 * (2 * n * n + 5 * n_pad * n_pad) - 1, real()[1])
    try:
        r = R.EASE_R_Recommender(X, verbose=False)
        torch.cuda.synchronize()
        t = time.perf_counter()
        r.fit(verbose=False, **kw)
        torch.cuda.synchronize()
        return r, time.perf_counter() - t
    finally:
        torch.cuda.mem_get_info = real


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


def c4(reps):
    X = synth_config("C4")
    times = {"default": [], "inplace": []}
    B = {}
    for rep in range(reps + 1):  # the first round warms both paths up
        for name in ("default", "inplace"):
            r, t = fit_timed(X, name == "inplace", topK=None, l2_norm=1e3)
            if rep > 0:
                times[name].append(t)
            B[name] = r._d_B
            print("C4 %-8s fit %.3f s" % (name, t), flush=True)
    d = float((B["default"] - B["inplace"]).abs().max())
    scale = float(B["default"].abs().max())
    return {"times_s": times, "max_abs_dB": d, "max_abs_B": scale}


def large(n_users, n_items, density, n_cols=20):
    X = synth_urm(n_users, n_items, density, seed=7, values="binary")
    n = n_items
    n_pad = -(-n // 128) * 128
    torch.cuda.empty_cache()
    free0, total = torch.cuda.mem_get_info()
    default_peak = 4 * (2 * n * n + 5 * n_pad * n_pad)
    ws = R.ctypes.c_int64()
    R._lib.check(R._lib.load().b200_ease_inplace_workspace_bytes(n, R.ctypes.byref(ws)))
    urm = R.ease_urm_bytes(X)
    bound = 4 * n_pad * n_pad + int(ws.value) + 4 * min(n, R.EASE_GRAM_SLAB_ROWS) * n + R.EASE_URM_COPIES * urm
    assert R.ease_inplace_for_device(n, free0, urm), (free0, default_peak, bound)
    cols = np.sort(np.random.default_rng(3).choice(n, n_cols, replace=False))
    captured = {}
    real_topk = slim_bpr_epoch.dense_topk_to_sparse

    def capture(B, *a, **k):  # the dense B the fit hands to its top-K: keep the sampled columns
        captured["cols"] = B[:, torch.from_numpy(cols).to(B.device)].double().cpu().numpy()
        return real_topk(B, *a, **k)
    slim_bpr_epoch.dense_topk_to_sparse = capture
    try:
        with FreePoll() as poll:
            r, t = fit_timed(X, False, topK=100, l2_norm=1e3)
    finally:
        slim_bpr_epoch.dense_topk_to_sparse = real_topk
    high_water = free0 - poll.low
    # residual (G + D)(e_j - B[:, j]) in fp64: G = X^T X with diag(G) replaced by popularity + l2
    Xd = X.astype(np.float64).tocsr()
    XT = Xd.T.tocsr()
    sq = np.asarray(Xd.multiply(Xd).sum(axis=0)).ravel()
    diag = np.diff(X.tocsc().indptr) + 1e3
    worst = 0.0
    for k, j in enumerate(cols):
        v = -captured["cols"][:, k]
        v[j] += 1.0
        res = XT @ (Xd @ v) - sq * v + diag * v
        off = np.abs(np.delete(res, j)).max()
        worst = max(worst, float(off / abs(res[j])))
    return {"n_users": n_users, "n_items": n_items, "nnz": int(X.nnz), "fit_s": t, "free_before": int(free0),
            "total": int(total), "high_water_bytes": int(high_water), "bound_bytes": int(bound),
            "default_peak_bytes": int(default_peak), "max_offdiag_residual_rel": worst, "W_nnz": int(r.W_sparse.nnz)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--large-users", type=int, default=1_000_000)
    ap.add_argument("--large-items", type=int, default=100_000)
    ap.add_argument("--large-density", type=float, default=0.0005)
    ap.add_argument("--skip-c4", action="store_true")  # --large-items 0 skips the large catalogue
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    out = {"card": card()}
    print(out["card"], flush=True)
    # the large catalogue first: C4's default path leaves its packed-operand workspaces grown (2 n_pad^2 floats)
    if a.large_items > 0:
        out["large"] = large(a.large_users, a.large_items, a.large_density)
        print(json.dumps(out["large"]), flush=True)
    if not a.skip_c4:
        out["C4"] = c4(a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
