"""Development timing of the tensor-core GEMM on one GPU, on the shapes of the blocked SPD inverse at C4 size:
    python tools/dev_gemm_bench.py [n=17792]
kind 0: trailing update (n-128) x (n-128) x 128; kind 1: factor-inverse block 128 x 128 x (n/2); kind 2: Linv^T Linv, n^3/3."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from recsys2019_deeplearning_evaluation_b200 import _lib

n = int(sys.argv[1]) if len(sys.argv) > 1 else 17792
L = _lib.load()
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
shapes = [(0, n - 128, n - 128, 128), (1, 128, 128, (n // 2) // 32 * 32), (2, n, n, n)]
for kind, M, N, K in shapes:
    A = torch.randn((M, K) if kind < 2 else (K, M), device="cuda")
    B = torch.randn((N, K) if kind == 0 else (K, N), device="cuda")
    if kind == 2:
        A, B = torch.tril(A), torch.tril(B)
    C = torch.zeros((M, N), device="cuda")
    flops = 2.0 * M * N * K * (1.0 / 3.0 if kind == 2 else 1.0)
    ms = []
    for rep in range(4):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(L.b200_debug_gemm_device(kind, M, N, K, 1.0, A.data_ptr(), A.shape[1], B.data_ptr(), B.shape[1], 0.0,
                                            C.data_ptr(), N, st))
        e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    best = min(ms[1:])
    print("kind %d  %6d x %6d x %6d  %8.3f ms  %7.1f TFLOP/s (useful fp32-equivalent; x3 on the tensor pipe)" % (
        kind, M, N, K, best, flops / best / 1e9), flush=True)
