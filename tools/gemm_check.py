"""GPU: speed of the tensor-core 3xTF32 GEMM (gemm_tc3.cu) in both call patterns -- "gen2" the default (grouped
launches, pre-split weight planes), "gen1" gib_tc_debug bit 0 (per-problem launches).  Accuracy against float64 lives
in tests/test_gpu_gemm_patterns.py.

    python tools/gemm_check.py                # forward / dX and weight-gradient timing table
"""
import ctypes
import sys

import torch

sys.path.insert(0, ".")
from graphinvent_b200._lib import check, lib  # noqa: E402

P = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)
st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def planes(W):
    hi, lo = torch.empty_like(W), torch.empty_like(W)
    check(lib.gib_split_planes(P(W), P(hi), P(lo), W.numel(), st()), "split")
    return hi, lo


def nt(X, Whl, b, Y, M, N, K, act, gen):
    lib.gib_tc_debug({1: 1, 2: 0}[gen])
    check(lib.gib_linear_fwd_tc_planes(P(X), X.shape[1], P(Whl[0]), P(Whl[1]), K, P(b), P(Y), Y.shape[1], M, N, K, act,
                                       None, None, st()), f"linear gen{gen}")
    lib.gib_tc_debug(0)


def dw(G, X, M, N, K, gen, dW, db, sc):
    lib.gib_tc_debug({1: 1, 2: 0}[gen])
    check(lib.gib_linear_bwd_dw(P(G), G.shape[1], N, P(X), X.shape[1], K, M, P(dW), P(db), N, K, P(sc), None, None,
                                st()), f"dw gen{gen}")
    lib.gib_tc_debug(0)


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


# ---- forward / dX shapes of the model ----------------------------------------------------------------------------------
for (M, N, K) in [(128, 128, 32), (100, 48, 16), (1000, 256, 256), (23808, 256, 256), (23808, 128, 256),
                  (23808, 256, 128), (13312, 512, 512), (13312, 384, 128), (4096, 48, 512), (5000, 608, 512),
                  (13312, 256, 144), (1024, 500, 688), (155648, 256, 256)]:
    torch.manual_seed(M + N + K)
    X = torch.randn(M, K, device="cuda")
    Whl = planes(torch.randn(N, K, device="cuda") / K ** 0.5)
    b = torch.randn(N, device="cuda")
    Y = torch.empty(M, N, device="cuda")
    t2 = timeit(lambda: nt(X, Whl, b, Y, M, N, K, 1, 2))
    t1 = timeit(lambda: nt(X, Whl, b, Y, M, N, K, 1, 1))
    fl = 2.0 * M * N * K
    print(f"NT M={M:6d} N={N:4d} K={K:4d}: gen2 {t2*1e3:8.1f} us ({fl/t2/1e9:7.1f} TF/s)   "
          f"gen1 {t1*1e3:8.1f} us ({fl/t1/1e9:6.1f} TF/s)", flush=True)

# ---- weight gradients --------------------------------------------------------------------------------------------------
for (M, N, K) in [(2048, 128, 128), (4100, 256, 256), (23808, 256, 256), (23808, 256, 128), (13312, 512, 512),
                  (13312, 384, 128), (13312, 48, 512), (13312, 256, 144), (20000, 608, 512), (155648, 256, 256)]:
    torch.manual_seed(M + N)
    G = torch.randn(M, N, device="cuda"); X = torch.randn(M, K, device="cuda")
    dW = torch.zeros(N, K, device="cuda"); db = torch.zeros(N, device="cuda")
    sc = torch.empty(lib.gib_dw_scratch_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    line = f"TN M={M:6d} N={N:4d} K={K:4d}:"
    for gen in (2, 1):
        t = timeit(lambda: dw(G, X, M, N, K, gen, dW, db, sc), 10)
        line += f" gen{gen} {t*1e3:7.1f} us ({2.0*M*N*K/t/1e9:5.1f} TF/s)"
    print(line, flush=True)
