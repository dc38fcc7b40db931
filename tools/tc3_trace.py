"""GPU: per-tile timeline of CTA 0 of the tensor-core GEMM (gib_tc_trace): when does it start a work item, when has
its last wgmma retired, when are its results handed to the store warps (specialised epilogues) and when are its
stores issued (and the chain counter released), or, with the register epilogue, when is the tile stored.
    python tools/tc3_trace.py [MxNxK] [tiles] [tn] [dselu] [chain]
      tn:    the weight-gradient mode too, one line per work item
      dselu: also the dX epilogue C = acc * selu'(aux) (gib_test_gemm_nt)
      chain: also a 5-layer chain of MxNxK SELU layers (K = N), the message-MLP forward pattern"""
import ctypes
import sys

import torch

sys.path.insert(0, ".")
from graphinvent_b200._lib import check, lib  # noqa: E402

P = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)
st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
M, N, K = (int(v) for v in (sys.argv[1] if len(sys.argv) > 1 else "155648x256x256").split("x"))
tiles = int(sys.argv[2]) if len(sys.argv) > 2 else 12
X = torch.randn(M, K, device="cuda"); W = torch.randn(N, K, device="cuda") / K ** 0.5; b = torch.randn(N, device="cuda")
hi, lo = torch.empty_like(W), torch.empty_like(W)
check(lib.gib_split_planes(P(W), P(hi), P(lo), W.numel(), st()), "split")
Y = torch.empty(M, N, device="cuda")


def trace(run, title):
    buf = torch.zeros(tiles, 16, dtype=torch.int64, device="cuda")
    for _ in range(2):
        run()
    lib.gib_tc_trace(P(buf), tiles)
    run()
    torch.cuda.synchronize()
    lib.gib_tc_trace(None, 0)
    t = buf.cpu()
    t0 = int(t[0, 0])
    print(f"== {title}: cycles relative to the first start of CTA 0 (0: not stamped by this kernel)")
    print("item     start   mma end    handed    stored  end(reg)  main loop  outside")
    rel = lambda v: int(v) - t0 if int(v) else 0
    for i in range(tiles):
        r = t[i]
        if int(r[0]) == 0:
            break
        nxt = int(t[i + 1, 0]) if i + 1 < tiles and int(t[i + 1, 0]) else 0
        outside = nxt - int(r[1]) if nxt and int(r[1]) else 0
        print(f"{i:4d} {rel(r[0]):9d} {rel(r[1]):9d} {rel(r[2]):9d} {rel(r[3]):9d} {rel(r[6]):9d} "
              f"{int(r[1]) - int(r[0]) if int(r[1]) else 0:10d} {outside:8d}")


def test_nt(ps, dep=None):
    """gib_test_gemm_nt on ctypes GemmProblem structs"""
    from graphinvent_b200 import _lib
    arr = (_lib.GemmProblem * len(ps))(*ps)
    flags, dp = None, None
    if dep is not None:
        nb = lib.gib_test_chain_flag_bytes(arr, len(ps))
        flags = torch.empty(max(nb // 4, 1), dtype=torch.int32, device="cuda")
        dp = (ctypes.c_int * len(ps))(*dep)
    return lambda: check(lib.gib_test_gemm_nt(arr, len(ps), dp, P(flags), st()), "test_gemm_nt")


def problem(A, hi, lo, C, N, K, mode, act, bias=None, aux=None):
    from graphinvent_b200 import _lib
    s = _lib.GemmProblem()
    s.A, s.lda, s.W, s.ldw, s.W_hi, s.W_lo = A.data_ptr(), A.shape[1], hi.data_ptr(), K, hi.data_ptr(), lo.data_ptr()
    s.C, s.ldc, s.M, s.N, s.K = C.data_ptr(), C.shape[1], A.shape[0], N, K
    s.bias, s.act, s.mode = (bias.data_ptr() if bias is not None else 0), act, mode
    s.aux, s.ldaux = (aux.data_ptr() if aux is not None else 0), (aux.shape[1] if aux is not None else 0)
    s.n_store, s.n_valid, s.m_dev, s.base_dev = N, N, 0, 0
    return s


trace(lambda: check(lib.gib_linear_fwd_tc_planes(P(X), K, P(hi), P(lo), K, P(b), P(Y), N, M, N, K, 1, None, None, st()),
                    "nt"), f"NT {M}x{N}x{K}")
if "dselu" in sys.argv[1:]:
    Yf = torch.selu(torch.randn(M, N, device="cuda"))
    trace(test_nt([problem(X, hi, lo, Y, N, K, 1, 1, aux=Yf)]), f"NT dselu {M}x{N}x{K}")
if "chain" in sys.argv[1:]:
    Ws = []   # keeps the weights alive
    bufs = [X] + [torch.empty(M, N, device="cuda") for _ in range(5)]
    ps = []
    for l in range(5):
        Wl = torch.randn(N, bufs[l].shape[1], device="cuda") / bufs[l].shape[1] ** 0.5
        h, o = torch.empty_like(Wl), torch.empty_like(Wl)
        check(lib.gib_split_planes(P(Wl), P(h), P(o), Wl.numel(), st()), "split")
        Ws.append((Wl, h, o))
        ps.append(problem(bufs[l], h, o, bufs[l + 1], N, bufs[l].shape[1], 0, 1, bias=b))
    trace(test_nt(ps, [-1, 0, 1, 2, 3]), f"NT chain 5 x {M}x{N}x{K}")
if "tn" in sys.argv[1:]:
    G = torch.randn(M, N, device="cuda")
    sc = torch.empty(lib.gib_dw_scratch_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    dW = torch.zeros(N, K, device="cuda"); db = torch.zeros(N, device="cuda")
    trace(lambda: check(lib.gib_linear_bwd_dw(P(G), N, N, P(X), K, K, M, P(dW), P(db), N, K, P(sc), None, None, st()),
                        "dw"), f"TN {M}x{N}x{K}")
