"""GPU: the specialised epilogues of tc3_wgmma_kernel (SELU, LINEAR, DSELU, ADD), which stage a tile's aux block or
bias slice and its results in shared memory and store them from warpgroup 2.

Every output goes to a guarded, poisoned buffer (tests/guarded.py) with 4 spare columns past n_store and spare rows
around the live range.  Each case checks that:
- the live block [base, base + M) x [0, n_store) agrees with float64 within the 3xTF32 bound of
  test_gpu_gemm_patterns.py;
- every other byte of the buffer still holds what it held before, and both guard bands are intact;
- grouped and chained launches give the same bits as the same problems launched one at a time.
"""
import ctypes

import pytest
import torch

from tests.guarded import Guarded
from tests.test_gpu_gemm_patterns import (ACT_SLACK, DACT_SLACK, EPI_ACT, EPI_ADD, EPI_MUL_DACT, SLOPE, TC_NT, _act64,
                                          _dact64, _dev_int, _lib, _p, _planes, _profiled, _st, _within)

pytestmark = pytest.mark.gpu

EPIS = {"selu": (EPI_ACT, 1), "linear": (EPI_ACT, 0), "dselu": (EPI_MUL_DACT, 1), "add": (EPI_ADD, 0)}
SPARE_COLS, SPARE_ROWS = 4, 37


class Prob:
    """one NT problem on guarded buffers.  dyn: the row count and base are device ints, the buffers hold
    base + M + SPARE_ROWS rows; else the buffers hold exactly M rows."""

    def __init__(self, M, n_store, epi, dyn, base=0, alias=False, seed=0, A=None, K=None):
        torch.manual_seed(seed * 7919 + M * 31 + n_store * 7 + (1 + base))
        self.mode, self.act = EPIS[epi]
        self.M, self.N, self.n_store, self.dyn = M, n_store, n_store, dyn
        self.K = K or (48 if M < 1000 else 256)
        self.lo = base if dyn else 0
        self.hi = self.lo + M
        self.rows = self.hi + SPARE_ROWS if dyn else M
        self.ldc = n_store + SPARE_COLS
        if A is None:
            A = torch.full((self.rows, self.K), float("nan"), device="cuda")
            A[self.lo:self.hi] = torch.randn(M, self.K, device="cuda")
        self.A = A
        self.W = torch.randn(self.N, self.K, device="cuda") / self.K ** 0.5
        self.hl = _planes(self.W)
        with_bias = epi == "selu" or (epi == "linear" and n_store != 144)
        self.bias = torch.randn(self.N, device="cuda") if with_bias else None
        self.gC = Guarded(self.rows * self.ldc * 4)
        self.C = self.gC.view(torch.float32, (self.rows, self.ldc))
        self.aux = None
        if self.mode != EPI_ACT:
            if alias:
                self.aux = self.C
            else:
                self.gaux = Guarded(self.rows * self.ldc * 4)
                self.aux = self.gaux.view(torch.float32, (self.rows, self.ldc))
            x = torch.randn(M, n_store, device="cuda") * 2
            self.aux[self.lo:self.hi, :n_store] = torch.selu(x) if self.mode == EPI_MUL_DACT else x
        self.C0 = self.C.clone()
        self.aux0 = None if self.aux is None else self.aux.clone()
        self.m_dev = _dev_int(M) if dyn else None
        self.base_dev = _dev_int(base) if dyn else None

    def struct(self):
        s = _lib().GemmProblem()
        s.A, s.lda = _p(self.A), self.A.shape[1]
        s.W, s.ldw = _p(self.W), self.K
        s.W_hi, s.W_lo = _p(self.hl[0]), _p(self.hl[1])
        s.C, s.ldc = _p(self.C), self.ldc
        s.M, s.N, s.K = self.rows, self.N, self.K
        s.bias, s.act, s.mode = _p(self.bias), self.act, self.mode
        s.aux, s.ldaux = _p(self.aux), (self.ldc if self.aux is not None else 0)
        s.n_store, s.n_valid = self.n_store, self.n_store
        s.m_dev, s.base_dev = _p(self.m_dev), _p(self.base_dev)
        return s

    def check(self, what):
        lo, hi, ns = self.lo, self.hi, self.n_store
        A64, W64 = self.A[lo:hi, :self.K].double(), self.W.double()
        pre, mag = A64 @ W64.t(), A64.abs() @ W64.abs().t()
        slack = 0.0
        if self.mode == EPI_ACT:
            if self.bias is not None:
                pre, mag = pre + self.bias.double(), mag + self.bias.double().abs()
            ref, mag = _act64(pre, self.act), mag * SLOPE[self.act]
            slack = ACT_SLACK if self.act else 0.0
        elif self.mode == EPI_MUL_DACT:
            d = _dact64(self.aux0[lo:hi, :ns].double(), self.act)
            ref, mag, slack = pre * d, mag * d.abs(), mag * DACT_SLACK
        else:
            x = self.aux0[lo:hi, :ns].double()
            ref, mag = pre + x, mag + x.abs()
        _within("tc", self.C[lo:hi, :ns], ref, mag, what, slack)
        outside = torch.ones(self.rows, self.ldc, dtype=torch.bool, device="cuda")
        outside[lo:hi, :ns] = False
        assert torch.equal(self.C.view(torch.int32)[outside], self.C0.view(torch.int32)[outside]), \
            f"{what}: a cell outside the live block changed"
        assert self.gC.intact(), f"{what}: guard band written at {self.gC.damage()}"
        if self.aux is not None and self.aux is not self.C:
            assert torch.equal(self.aux.view(torch.int32), self.aux0.view(torch.int32)), f"{what}: aux changed"
            assert self.gaux.intact(), f"{what}: aux guard band written"


def _run(ps, dep=None):
    L = _lib()
    arr = (L.GemmProblem * len(ps))(*[p.struct() for p in ps])
    flags = None
    if dep is not None:
        nb = L.lib.gib_test_chain_flag_bytes(arr, len(ps))
        flags = torch.full((max(nb // 4, 1),), 12345, dtype=torch.int32, device="cuda")
        dep = (ctypes.c_int * len(ps))(*dep)
    rc, cls = _profiled(lambda: L.lib.gib_test_gemm_nt(arr, len(ps), dep, _p(flags), _st()))
    assert rc == 0, L.lib.gib_last_error().decode()
    assert cls == [TC_NT], f"one tensor-core launch expected, got {cls}"


def _bits(t):
    return t.view(torch.int32).clone()


@pytest.mark.parametrize("n_store", [48, 128, 144, 256, 608])
@pytest.mark.parametrize("M", [1, 127, 128, 129, 16001])
@pytest.mark.parametrize("epi", list(EPIS))
def test_epilogue_device_rows(epi, M, n_store):
    """device-side row count and base: one problem alone, then the same problem as member 2 of a group of 3"""
    base = 3 if M < 1000 else 130
    p = Prob(M, n_store, epi, dyn=True, base=base)
    _run([p])
    p.check(f"{epi} M={M} n_store={n_store} device rows")
    alone = _bits(p.C)
    q = Prob(M, n_store, epi, dyn=True, base=base)
    others = [Prob(M + 5, n_store, epi, dyn=True, base=base, seed=s) for s in (1, 2)]
    _run([others[0], q, others[1]])
    assert torch.equal(_bits(q.C), alone), "grouped launch differs from the launch alone"
    for o in others:
        o.check(f"{epi} M={M} n_store={n_store} device rows, group member")


@pytest.mark.parametrize("n_store", [48, 128, 144, 256, 608])
@pytest.mark.parametrize("M", [1, 127, 128, 129, 16001])
@pytest.mark.parametrize("epi", list(EPIS))
def test_epilogue_host_rows(epi, M, n_store):
    """host-side row counts in a group of 4 (so that small problems take the tensor cores), against the same problems
    launched alone on device-side counts"""
    ps = [Prob(M, n_store, epi, dyn=False, seed=s) for s in range(4)]
    _run(ps)
    for i, p in enumerate(ps):
        p.check(f"{epi} M={M} n_store={n_store} host rows, member {i}")
        q = Prob(M, n_store, epi, dyn=True, base=0, seed=i)
        _run([q])
        assert torch.equal(_bits(q.C[:M, :n_store]), _bits(p.C[:M, :n_store])), \
            f"member {i}: grouped launch differs from the launch alone"


@pytest.mark.parametrize("M", [129, 16001])
@pytest.mark.parametrize("n_store", [144, 608])
@pytest.mark.parametrize("dyn", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("epi", ["add", "dselu"])
def test_epilogue_aux_aliases_c(epi, dyn, n_store, M):
    """aux is C itself (in-place dh += ...): each tile reads its aux before its results are stored"""
    ps = [Prob(M, n_store, epi, dyn=dyn, base=65 if dyn else 0, alias=True, seed=s) for s in range(4)]
    _run(ps)
    for i, p in enumerate(ps):
        p.check(f"{epi} aliased M={M} n_store={n_store} member {i}")


@pytest.mark.parametrize("M", [1, 129, 16001])
def test_epilogue_dselu_chain(M):
    """a 3-layer x 2-member dX chain on device-side rows: the same bits as its layers launched one at a time"""
    widths = [256, 128, 144, 608]

    def build():
        ps, dep, last = [], [], [None, None]
        for l in range(1, len(widths)):
            for i in range(2):
                a = last[i].C if last[i] is not None else None
                p = Prob(M, widths[l], "dselu", dyn=True, base=70, seed=10 * l + i, A=a, K=widths[l - 1])
                if a is not None:
                    p.m_dev, p.base_dev = last[i].m_dev, last[i].base_dev
                ps.append(p)
                dep.append(len(ps) - 3 if l > 1 else -1)
                last[i] = p
        return ps, dep

    chain, dep = build()
    _run(chain, dep)
    for k, p in enumerate(chain):
        p.check(f"chain M={M} problem {k}")
    single, _ = build()
    for p in single:
        _run([p])
    for k, (a, b) in enumerate(zip(chain, single)):
        assert torch.equal(_bits(a.C), _bits(b.C)), f"chain problem {k} differs from its launch alone"
