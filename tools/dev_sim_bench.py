"""Development timing of the similarity path on one GPU: python tools/dev_sim_bench.py C5 [binary|continuous] [reps]"""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from recsys2019_deeplearning_evaluation_b200.synth import synth_config
from recsys2019_deeplearning_evaluation_b200.similarity import Compute_Similarity_Cython

cfg = sys.argv[1] if len(sys.argv) > 1 else "C1"
values = sys.argv[2] if len(sys.argv) > 2 else "binary"
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
t = time.time(); X = synth_config(cfg, values=values); print("gen %s %s nnz=%d %.1fs" % (cfg, X.shape, X.nnz, time.time() - t), flush=True)
torch.cuda.init()
t = time.time(); sim = Compute_Similarity_Cython(X, topK=200, shrink=100, similarity="cosine"); torch.cuda.synchronize()
print("create %.3fs windows=%d cells=%d binary=%s" % (time.time() - t, sim.n_windows, sim.window_cells, sim.binary_path), flush=True)
ent = sim.gathered_entries()
bpe = 4 if sim.binary_path else 8
alg = bpe * ent + (8 if not sim.binary_path else 4) * 2 * X.nnz + 8 * sim.K * X.shape[1]
for r in range(reps):
    t = time.time(); tab = sim.compute_topk_device(0, X.shape[1]); torch.cuda.synchronize(); dt = time.time() - t
    ms = sim.last_kernel_ms()
    print("rep %d: wall %.3fs kernel %.3f ms  %.3e cols/s  alg %.2f GB -> %.1f GB/s" % (r, dt, ms, X.shape[1] / (ms * 1e-3), alg / 1e9, alg / 1e9 / (ms * 1e-3)), flush=True)
import ctypes
from recsys2019_deeplearning_evaluation_b200 import _lib
L = _lib.load()
_lib.check(L.b200_sim_debug_phase_cycles(sim._h, 1, None))
tab = sim.compute_topk_device(0, X.shape[1]); torch.cuda.synchronize()
out = (ctypes.c_uint64 * 16)()
_lib.check(L.b200_sim_debug_phase_cycles(sim._h, 0, out))
cyc = np.array(list(out), dtype=np.float64)
en, tb, nb, nw = (ctypes.c_int32() for _ in range(4))
_lib.check(L.b200_sim_debug_k1c(sim._h, -1, ctypes.byref(en), ctypes.byref(tb), ctypes.byref(nb), ctypes.byref(nw)))
print("nibble kernel: enabled=%d ctas/SM=%d its cols=%d window cols (dense + redo)=%d" % (en.value, tb.value, nb.value, nw.value), flush=True)
names = ["stage", "mac|gather", "bootstrap|sweep", "scan|lvl3", "eval|lvl2", "select|lvl1", "emit|select+emit", "-"]
print("phase cycles per column: " + "  ".join("%s=%.0f" % (n, c / X.shape[1]) for n, c in zip(names, cyc)) + "  total=%.0f (kernel %.3f ms)" % (cyc.sum() / X.shape[1], sim.last_kernel_ms()), flush=True)
t = time.time(); W = sim.table_to_csr(tab); print("to_csr %.3fs nnz=%d" % (time.time() - t, W.nnz), flush=True)
