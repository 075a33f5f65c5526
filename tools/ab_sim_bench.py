"""Development A/B timing of libb200rec variants on one GPU (one URM generation, one subprocess per library):
    python tools/ab_sim_bench.py C5 binary default ub4 ...
`default` = the in-tree libb200rec.so, any other name = recsys2019_deeplearning_evaluation_b200/_variants/libb200rec_<name>.so"""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

if sys.argv[1] == "--child":
    import ctypes
    import scipy.sparse as sps
    import torch
    from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython
    from recsys2019_deeplearning_evaluation_b200 import _lib
    z = np.load(sys.argv[2])
    X = sps.csr_matrix((z["data"], z["indices"], z["indptr"]), shape=tuple(z["shape"]))
    t0 = time.time()
    sim = Compute_Similarity_Cython(X, topK=200, shrink=100, similarity="cosine")
    torch.cuda.synchronize()
    create_s = time.time() - t0  # uploads, relabelling, row layouts: the first create of a process also loads the library
    n = X.shape[1]
    ms = []
    for r in range(4):
        tab = sim.compute_topk_device(0, n)
        torch.cuda.synchronize()
        ms.append(sim.last_kernel_ms())
    chk = int(tab.cnt.sum().item()), float(tab.val.double().sum().item())
    # the range as two half-range calls: the K1-D kernel alone on every column (a sub-range never takes the pair path)
    halves = []
    for r in range(3):
        t = 0.0
        for lo, hi in ((0, n // 2), (n // 2, n)):
            sim.compute_topk_device(lo, hi)
            torch.cuda.synchronize()
            t += sim.last_kernel_ms()
        halves.append(t)
    print("%-10s create %.3f s  two half-range calls, kernel ms %s" % (sys.argv[3], create_s, " ".join("%.2f" % m for m in halves)),
          flush=True)
    L = _lib.load()
    _lib.check(L.b200_sim_debug_phase_cycles(sim._h, 1, None))
    sim.compute_topk_device(0, n); torch.cuda.synchronize()
    out = (ctypes.c_uint64 * 16)()
    _lib.check(L.b200_sim_debug_phase_cycles(sim._h, 0, out))
    cyc = np.array(list(out), dtype=np.float64) / n
    print("%-10s kernel ms %s  checksum %s  cycles/col stage=%.0f mac=%.0f boot=%.0f scan=%.0f eval=%.0f select=%.0f emit=%.0f"
          "  pair path: upper-gather=%.0f upper-sweep=%.0f sel-keys=%.0f sel-emit=%.0f" % (
              sys.argv[3], " ".join("%.2f" % m for m in ms), chk, *cyc[:7], *cyc[8:12]), flush=True)
    if cyc[12] > 0:
        print("%-10s exchange: %d runs for %d cells, mean run %.1f cells" % (sys.argv[3], cyc[12] * n, cyc[13] * n, cyc[13] / cyc[12]),
              flush=True)
    # device time per kernel of one call (a profiled run of its own): the gather / exchange / select split
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sim.compute_topk_device(0, n); torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            key = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("b200::sim::", "")
            per[key] = per.get(key, 0.0) + e.device_time_total / 1e3
    print("%-10s kernel split ms: %s" % (sys.argv[3], ", ".join("%s %.2f" % kv for kv in sorted(per.items(), key=lambda kv: -kv[1]))),
          flush=True)
    sys.exit(0)

from recsys2019_deeplearning_evaluation_b200.synth import synth_config
cfg, values, names = sys.argv[1], sys.argv[2], sys.argv[3:]
t = time.time()
X = synth_config(cfg, values=values)
path = "/dev/shm/ab_%s_%s.npz" % (cfg, values)
np.savez(path, data=X.data, indices=X.indices, indptr=X.indptr, shape=np.array(X.shape))
print("generated %s %s nnz=%d in %.1fs" % (cfg, X.shape, X.nnz, time.time() - t), flush=True)
for name in names:
    env = dict(os.environ)
    if name != "default":
        env["B200REC_LIB"] = os.path.join(ROOT, "recsys2019_deeplearning_evaluation_b200", "_variants", "libb200rec_%s.so" % name)
    subprocess.call([sys.executable, os.path.abspath(__file__), "--child", path, name], env=env)
os.remove(path)
