"""GPU: every call pattern the model runs on the GEMM kernels (csrc/gemm_tc3.cu, csrc/gemm_simt.cu), one at a time
against float64, through the C-ABI test hooks (gib_test_gemm_nt, gib_test_dw_groups).

Bound, per element:  |C - C64| <= eps[path] * (|A| |W|^T)_ij   (+ the magnitudes of bias / aux / the accumulated dW that
enter the element), scaled by the activation's slope, with one eps per path: "tc" (3xTF32 on the tensor cores) and
"simt" (fp32 FMA).  Activations evaluated in the epilogue add a fixed 1e-6 (SELU through ex2.approx, tanhf), derivatives act'(aux)
2^-21 * (|A| |W|^T)_ij (their fp32 evaluation).
Cells outside a problem's range start as sentinels and must come back bit-identical; pad columns must be exact zeros.
The kernel class of every launch (gib_profile_records) is checked too: a case meant for the tensor cores fails if it
lands on the SIMT kernels, and the reverse.
"""
import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

# 4 x (rounded down) the worst |C - C64| / magnitude over the whole sweep, measured on an H100 80GB HBM3 (SXM):
#   tc 8.27e-7 (the group of 16 weight gradients), simt 3.51e-7 (M=4097 N=608 K=688, C + aux aliasing C)
EPS = {"tc": 3.2e-6, "simt": 1.4e-6}
ACT_SLACK = 1e-6
DACT_SLACK = 2.0 ** -21
SLOPE = {0: 1.0, 1: 1.7581, 2: 1.0}         # max |act'|: none, SELU, tanh
TC_NT, TC_DW, SIMT_NT, SIMT_DW = 0, 1, 3, 4   # profile classes (include/gib200.h)
EPI_ACT, EPI_MUL_DACT, EPI_ADD = 0, 1, 2
NAN = float("nan")
WORST = {}


def _lib():
    from graphinvent_b200 import _lib
    return _lib


def _p(t):
    return t.data_ptr() if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev_int(v):
    return torch.tensor([v], dtype=torch.int32, device="cuda")


def pad16(x):
    return (x + 15) // 16 * 16


def cdiv(a, b):
    return -(-a // b)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst error / magnitude per path:", {k: f"{v[0]:.3g} ({v[1]})" for k, v in sorted(WORST.items())})


@contextlib.contextmanager
def _mode(tc=1, debug=0):
    L = _lib().lib
    L.gib_set_tensor_cores(tc)
    L.gib_tc_debug(debug)
    try:
        yield
    finally:
        L.gib_set_tensor_cores(1)
        L.gib_tc_debug(0)


def _profiled(fn):
    """run fn() with the per-launch profile on: (its return code, sorted kernel classes of its launches)"""
    L = _lib().lib
    torch.cuda.synchronize()
    L.gib_profile_enable(1)
    try:
        rc = fn()
        torch.cuda.synchronize()
        cap = 256
        ms, work, cls = (ctypes.c_double * cap)(), (ctypes.c_double * cap)(), (ctypes.c_int * cap)()
        n = L.gib_profile_records(ms, work, cls, cap)
    finally:
        L.gib_profile_enable(0)
    assert 0 <= n <= cap
    return rc, sorted(cls[:n])


def _within(path, got, ref, mag, what, slack=0.0):
    """|got - ref| <= EPS[path] * mag + slack elementwise (NaN fails); records the worst (err - slack) / mag"""
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (mag + 1e-300)).max().item() if err.numel() else 0.0
    if ratio >= WORST.get(path, (0.0, ""))[0]:
        WORST[path] = (ratio, what)
    assert ratio <= EPS[path], f"{what}: error / magnitude {ratio:.3g} > eps {EPS[path]:.1e} ({path})"


def _same_bits(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), f"{what}: sentinels changed"


def _act64(x, act):
    return {0: x, 1: torch.selu(x), 2: torch.tanh(x)}[act]


def _dact64(y, act):
    if act == 1:
        return torch.where(y > 0, torch.full_like(y, 1.0507009873554805), y + 1.0507009873554805 * 1.6732632423543772)
    if act == 2:
        return 1 - y * y
    return torch.ones_like(y)


def _planes(W):
    L = _lib()
    hi, lo = torch.empty_like(W), torch.empty_like(W)
    L.check(L.lib.gib_split_planes(_p(W), _p(hi), _p(lo), W.numel(), _st()), "split_planes")
    return hi, lo


# ----------------------------------------------------------------------------------------------------------------------
# NT problems
# ----------------------------------------------------------------------------------------------------------------------
class NT:
    """one NT problem with its operands, sentinel-filled output and float64 check.  cap: the buffers hold `cap` rows and
    the problem covers rows [base, base + M) of them through device-side counts (m_dev may exceed cap - base: clamped)"""

    def __init__(self, M, N, K, mode=EPI_ACT, act=0, bias=True, n_store=None, n_valid=None, ldc=None, lda=None,
                 alias=False, planes=True, cap=None, base=0, seed=0, A=None):
        torch.manual_seed(seed * 7919 + M * 31 + N * 7 + K)
        self.N, self.K, self.mode, self.act, self.alias = N, K, mode, act, alias
        self.n_store = N if n_store is None else n_store
        self.n_valid = self.n_store if n_valid is None else n_valid
        self.ldc = ldc or self.n_store
        self.dyn = cap is not None
        rows = cap if self.dyn else M
        self.rows, self.M = rows, M
        self.lo = base if self.dyn else 0
        self.hi = min(base + M, cap) if self.dyn else M
        if A is None:
            lda = lda or K
            A = torch.full((rows, lda), NAN, device="cuda")   # rows outside the range and columns >= K: never read
            A[self.lo:self.hi, :K] = torch.randn(self.hi - self.lo, K, device="cuda")
        self.A = A
        self.W = torch.randn(N, K, device="cuda") / K ** 0.5
        self.hl = _planes(self.W) if planes else (None, None)
        self.bias = torch.randn(N, device="cuda") if (bias and mode == EPI_ACT) else None
        if alias:
            self.C = torch.randn(rows, self.ldc, device="cuda")
            self.aux = self.C
        else:
            self.C = torch.full((rows, self.ldc), NAN, device="cuda")
            self.aux = None
            if mode == EPI_MUL_DACT:
                self.aux = _act_t(torch.randn(rows, self.ldc, device="cuda") * 2, act)
            elif mode == EPI_ADD:
                self.aux = torch.randn(rows, self.ldc, device="cuda")
        self.C0 = self.C.clone()
        self.aux0 = None if self.aux is None else self.aux.clone()
        self.m_dev = _dev_int(M) if self.dyn else None
        self.base_dev = _dev_int(base) if self.dyn else None

    def struct(self):
        s = _lib().GemmProblem()
        s.A, s.lda = _p(self.A), self.A.shape[1]
        s.W, s.ldw = _p(self.W), self.K
        s.W_hi, s.W_lo = _p(self.hl[0]), _p(self.hl[1])
        s.C, s.ldc = _p(self.C), self.ldc
        s.M, s.N, s.K = self.rows if self.dyn else self.M, self.N, self.K
        s.bias, s.act, s.mode = _p(self.bias), self.act, self.mode
        s.aux, s.ldaux = _p(self.aux), (self.ldc if self.aux is not None else 0)
        s.n_store, s.n_valid = self.n_store, self.n_valid
        s.m_dev, s.base_dev = _p(self.m_dev), _p(self.base_dev)
        return s

    def check(self, path, what):
        lo, hi, ns, nv = self.lo, self.hi, self.n_store, self.n_valid
        A64 = self.A[lo:hi, :self.K].double()
        Wp = torch.zeros(max(self.N, ns), self.K, dtype=torch.float64, device="cuda")
        Wp[:self.N] = self.W.double()
        pre, mag = A64 @ Wp[:ns].t(), A64.abs() @ Wp[:ns].abs().t()
        slack = 0.0
        if self.mode == EPI_ACT:
            if self.bias is not None:
                b = torch.zeros(max(self.N, ns), dtype=torch.float64, device="cuda")
                b[:self.N] = self.bias.double()
                pre, mag = pre + b[:ns], mag + b[:ns].abs()
            ref, mag = _act64(pre, self.act), mag * SLOPE[self.act]
            slack = ACT_SLACK if self.act else 0.0
        elif self.mode == EPI_MUL_DACT:
            d = _dact64(self.aux0[lo:hi, :ns].double(), self.act)
            # the epilogue evaluates act'(aux) in fp32: <= 2^-21 absolute (SELU: aux + 1.758, tanh: 1 - aux^2)
            ref, mag, slack = pre * d, mag * d.abs(), mag * DACT_SLACK
        else:
            x = self.aux0[lo:hi, :ns].double()
            ref, mag = pre + x, mag + x.abs()
        out = self.C[lo:hi]
        _within(path, out[:, :nv], ref[:, :nv], mag[:, :nv], what, slack)
        assert (out[:, nv:ns] == 0).all() and not torch.signbit(out[:, nv:ns]).any(), f"{what}: pad columns not +0"
        _same_bits(out[:, ns:], self.C0[lo:hi, ns:], what + " columns >= n_store")
        _same_bits(self.C[:lo], self.C0[:lo], what + " rows before the range")
        _same_bits(self.C[hi:], self.C0[hi:], what + " rows after the range")

    def untouched(self, what):
        _same_bits(self.C, self.C0, what)


def _act_t(x, act):
    return {0: x, 1: torch.selu(x), 2: torch.tanh(x)}[act]


def _run_nt(nts, dep=None):
    L = _lib()
    arr = (L.GemmProblem * len(nts))(*[t.struct() for t in nts])
    flags = None
    if dep is not None:
        nb = L.lib.gib_test_chain_flag_bytes(arr, len(nts))
        flags = torch.full((max(nb // 4, 1),), 12345, dtype=torch.int32, device="cuda")   # zeroed by the launch
        dep = (ctypes.c_int * len(nts))(*dep)
    return _profiled(lambda: L.lib.gib_test_gemm_nt(arr, len(nts), dep, _p(flags), _st()))


def _expect_single(t, tc, debug):
    """kernel class the single-problem dispatcher picks (csrc/gemm_simt.cu: gemm_nt)"""
    if t.M <= 0:
        return []
    if t.dyn:
        return [TC_NT]
    if tc and t.N >= 48 and t.K >= 32:
        if not debug & 1 and t.M >= 256 and t.hl[0] is not None:
            return [TC_NT]
        if t.M >= 1024:
            return [TC_NT]
    return [SIMT_NT]


def _expect_group(nts, tc, debug):
    """kernel classes the grouped dispatcher produces (csrc/gemm_simt.cu: gemm_nt_group)"""
    if len(nts) == 1:
        return _expect_single(nts[0], tc, debug)
    ok = bool(tc) and len(nts) <= 4
    ok3, dyn, tiles = ok and not debug & 1, False, 0
    for t in nts:
        if not ok:
            break
        dyn = dyn or t.dyn
        if t.M <= 0:
            continue
        ok = t.K >= 32 and t.N >= 48
        ok3 = ok3 and ok and t.hl[0] is not None
        tiles += cdiv(t.M, 128) * cdiv(t.N, 128)
    if ok3 and (tiles >= 4 or dyn):
        return [TC_NT]
    if ok and not dyn and tiles >= 16:
        return [TC_NT]
    return sorted(c for t in nts for c in _expect_single(t, tc, debug))


def _path(classes):
    return "tc" if any(c in (TC_NT, TC_DW) for c in classes) else "simt"


def _epilogues(N):
    """(label, kwargs) of every epilogue the model uses on one shape"""
    return [("act none", dict(mode=EPI_ACT, act=0)),
            ("act selu", dict(mode=EPI_ACT, act=1)),
            ("act tanh", dict(mode=EPI_ACT, act=2)),
            ("mul_dact selu", dict(mode=EPI_MUL_DACT, act=1)),
            ("mul_dact tanh", dict(mode=EPI_MUL_DACT, act=2)),
            ("add", dict(mode=EPI_ADD)),
            ("add aliasing C", dict(mode=EPI_ADD, alias=True)),
            # n_valid < N < n_store < ldc, a bias of N entries, A with NaN pad columns past K
            ("generic", dict(mode=EPI_ACT, act=1, n_store=N + 8, n_valid=N - 3, ldc=N + 21, lda_pad=16))]


@pytest.mark.parametrize("M", [1, 64, 65, 127, 128, 129, 4097])
@pytest.mark.parametrize("N", [48, 64, 65, 128, 129, 200, 256, 608])
def test_nt_shapes_and_epilogues(M, N):
    """every epilogue at every shape: the dispatcher's own choice, the tensor-core kernel forced through a device-side
    row count (any M), and tensor cores off.  The wgmma tile is 128 x 128, split between two 64-row consumer
    warpgroups: M = 64 / 65 fill one warpgroup / spill one row into the second, N = 129 / 200 leave one / 72 live
    columns in a second column tile; K = 32 and 160 end on a full k-block (K = 160: five k-blocks, one more than the
    ring has stages), the other K on a half-empty one"""
    for K in (16, 32, 48, 144, 160, 688):
        for label, kw in _epilogues(N):
            kw = dict(kw)
            lda = K + kw.pop("lda_pad", 0)
            for run in ("dispatch", "tc", "simt"):
                what = f"M={M} N={N} K={K} {label} [{run}]"
                dyn = dict(cap=M + 5, base=3) if run == "tc" else {}
                t = NT(M, N, K, lda=lda, **kw, **dyn)
                tc = 0 if run == "simt" else 1
                with _mode(tc=tc):
                    rc, cls = _run_nt([t])
                assert rc == 0, what + ": " + _lib().lib.gib_last_error().decode()
                assert cls == _expect_single(t, tc, 0), f"{what}: kernel classes {cls}"
                t.check(_path(cls), what)


def test_nt_device_rows_refused_without_tensor_cores():
    """device-side row counts exist only on the tensor-core path: refused before any launch otherwise"""
    t = NT(300, 64, 48, cap=512, base=128)
    for tc, debug in ((0, 0), (1, 1)):
        with _mode(tc=tc, debug=debug):
            rc, cls = _run_nt([t])
        assert rc < 0 and cls == []
        t.untouched("refused problem")


def test_nt_identity_weight_reproduces_the_input():
    """W = I: every element of A must come back at its own place (a swizzle / fragment / column mix-up is a
    permutation, far outside the 3xTF32 rounding of the lo part)"""
    for M, K in ((128, 32), (128, 64), (256, 128), (300, 144), (4097, 48)):
        t = NT(M, K, K, bias=False, cap=M, base=0, seed=1)
        t.W.copy_(torch.eye(K, device="cuda"))
        t.hl = _planes(t.W)
        rc, cls = _run_nt([t])
        assert rc == 0 and cls == [TC_NT]
        X = t.A[:, :K]
        assert ((t.C - X).abs() <= 2.0 ** -20 * X.abs()).all(), f"identity M={M} K={K}"


def test_nt_large_row_count():
    """the largest GEMM row count of the C4 shape (155648 rows)"""
    t = NT(155648, 256, 256, act=1)
    rc, cls = _run_nt([t])
    assert rc == 0 and cls == [TC_NT]
    t.check("tc", "M=155648")


def _group_cases():
    return {
        "shared selu": lambda: [NT(1000, 256, 144, act=1), NT(129, 64, 48, act=1), NT(300, 608, 688, act=1)],
        "mixed + empty member": lambda: [
            NT(300, 65, 48, act=2, n_store=72, n_valid=70, ldc=84), NT(513, 256, 144, mode=EPI_MUL_DACT, act=1),
            NT(129, 128, 64, mode=EPI_ADD, alias=True), NT(0, 64, 32, act=1)],
        "k16 member": lambda: [NT(1000, 256, 16, act=1), NT(2000, 128, 64, act=0), NT(127, 48, 48, mode=EPI_ADD)],
        "device rows": lambda: [NT(1000, 256, 144, act=1, cap=2048, base=256),
                                NT(700, 64, 48, mode=EPI_MUL_DACT, act=1, cap=2048, base=1900)],
    }


@pytest.mark.parametrize("case", list(_group_cases()))
@pytest.mark.parametrize("tc,debug", [(1, 0), (0, 0), (1, 1)])
def test_nt_groups(case, tc, debug):
    """2-4 independent problems of different shapes in one call of the grouped dispatcher"""
    nts = _group_cases()[case]()
    if debug:      # the per-problem call pattern splits raw W in the kernel
        for t in nts:
            t.hl = (None, None)
    with _mode(tc=tc, debug=debug):
        rc, cls = _run_nt(nts)
    if case == "device rows" and (not tc or debug):
        assert rc < 0 and cls == []
        for t in nts:
            t.untouched(case)
        return
    assert rc == 0, _lib().lib.gib_last_error().decode()
    assert cls == _expect_group(nts, tc, debug), f"{case}: kernel classes {cls}"
    if case in ("shared selu", "mixed + empty member", "device rows") and tc and not debug:
        assert cls == [TC_NT], f"{case}: expected one tensor-core launch, got {cls}"
    for i, t in enumerate(nts):
        t.check(_path(cls), f"{case} member {i}")


def test_nt_raw_weights_grouped_under_debug():
    """gib_tc_debug(1): a group of raw-W problems big enough for one tensor-core launch (W split in the kernel)"""
    nts = [NT(2000, 256, 144, act=1, planes=False), NT(1500, 128, 48, mode=EPI_ADD, planes=False)]
    with _mode(debug=1):
        rc, cls = _run_nt(nts)
    assert rc == 0 and cls == [TC_NT]
    for i, t in enumerate(nts):
        t.check("tc", f"raw member {i}")


# ----------------------------------------------------------------------------------------------------------------------
# dependent chains (mlp_forward_multi / mlp_backward_multi)
# ----------------------------------------------------------------------------------------------------------------------
def _chain(M, widths, members, mode, cap=None, base=0, seed=0, last_linear=False):
    """members x (len(widths) - 1) layers, layer-major like the model; each layer reads what the layer below stores"""
    depth = len(widths) - 1
    nts, dep, last = [], [], [-1] * members
    ins = [None] * members
    rows = (_dev_int(M), _dev_int(base)) if cap is not None else (None, None)   # siblings share one row range
    for l in range(1, depth + 1):
        for i in range(members):
            act = 0 if (last_linear and l == depth and mode == EPI_ACT) else 1
            kw = dict(mode=mode, act=act, seed=seed + 100 * l + i)
            if cap is not None:
                kw.update(cap=cap, base=base)
            if ins[i] is not None:
                kw["A"] = ins[i].C
            # widths that are not a multiple of 16 are stored with +0 pad columns up to the next one, which the
            # layer above reads as its K (the model's padded layout)
            t = NT(M, widths[l], pad16(widths[l - 1]), n_store=pad16(widths[l]), n_valid=widths[l], **kw)
            t.C.fill_(7.0)
            t.C0 = t.C.clone()
            t.m_dev, t.base_dev = rows
            nts.append(t)
            dep.append(last[i])
            last[i] = len(nts) - 1
            ins[i] = t
    return nts, dep


def _chain_cases():
    return {
        "2x1 M=1000": dict(M=1000, widths=[144, 256, 128], members=1, mode=EPI_ACT),
        "5x3 M=4097 widths vary": dict(M=4097, widths=[64, 48, 112, 96, 256, 80], members=3, mode=EPI_ACT,
                                       last_linear=True),
        "4x2 dX chain": dict(M=2000, widths=[96, 128, 48, 64, 256], members=2, mode=EPI_MUL_DACT),
        "3x2 device rows": dict(M=2500, widths=[64, 128, 256, 48], members=2, mode=EPI_ACT, cap=4096, base=384),
        "2x3 device rows dX": dict(M=1111, widths=[48, 112, 64], members=3, mode=EPI_MUL_DACT, cap=2048, base=640),
        "3x2 partial column tile": dict(M=3000, widths=[96, 200, 256, 200], members=2, mode=EPI_ACT),
        "3x1 device rows clamped": dict(M=1000, widths=[64, 64, 64, 64], members=1, mode=EPI_ACT, cap=4096,
                                        base=3968),
        "2x2 live count 0": dict(M=0, widths=[64, 96, 48], members=2, mode=EPI_ACT, cap=1024, base=0),
    }


@pytest.mark.parametrize("case", list(_chain_cases()))
def test_nt_chains(case):
    nts, dep = _chain(**_chain_cases()[case])
    rc, cls = _run_nt(nts, dep)
    assert rc == 0, _lib().lib.gib_last_error().decode()
    assert cls == [TC_NT], f"{case}: one chain launch expected, got {cls}"
    for k, t in enumerate(nts):
        t.check("tc", f"{case} problem {k} (depends on {dep[k]})")


def test_nt_chain_refusals():
    """the host refuses a chain that does not qualify, before any launch: too few tiles, K < 32, tensor cores off"""
    for kw, tc in ((dict(M=300, widths=[64, 64, 64], members=1, mode=EPI_ACT), 1),
                   (dict(M=4097, widths=[16, 64, 64], members=1, mode=EPI_ACT), 1),
                   (dict(M=4097, widths=[64, 128, 64], members=1, mode=EPI_ACT), 0)):
        nts, dep = _chain(**kw)
        with _mode(tc=tc):
            rc, cls = _run_nt(nts, dep)
        assert rc < 0 and cls == []
        for t in nts:
            t.untouched("refused chain")


# ----------------------------------------------------------------------------------------------------------------------
# weight gradients
# ----------------------------------------------------------------------------------------------------------------------
class DW:
    """one weight-gradient problem: dW[r*rs + c*cs] += sum_m G[m, prow(r)] X[m, c] (+ bias) over its live rows"""

    def __init__(self, G, X, M, dW, R, C, dbias=None, Rb=None, Rbp=None, rs=None, cs=1, rows=None):
        self.G, self.X, self.M, self.dW, self.dbias = G, X, M, dW, dbias
        self.R, self.C, self.rs, self.cs = R, C, C if rs is None else rs, cs
        self.Rb, self.Rbp = (R, G.shape[1]) if Rb is None else (Rb, Rbp)
        self.rows = rows                       # (m_dev, base_dev, lo, hi) for device-side counts
        self.Nn, self.Kk = G.shape[1], X.shape[1]

    def struct(self):
        q = _lib().DwProblem()
        q.G, q.ldg, q.Nn, q.X, q.ldx, q.Kk = _p(self.G), self.G.shape[1], self.Nn, _p(self.X), self.X.shape[1], self.Kk
        q.M, q.dW, q.dbias = self.M, _p(self.dW), _p(self.dbias)
        q.R, q.C, q.Rb, q.Rbp, q.rs, q.cs = self.R, self.C, self.Rb, self.Rbp, self.rs, self.cs
        if self.rows:
            q.m_dev, q.base_dev = _p(self.rows[0]), _p(self.rows[1])
        return q

    def live(self):
        return (self.rows[2], self.rows[3]) if self.rows else (0, self.M)

    def contribution(self):
        """(index of each dW element in the flat destination, fp64 sum, magnitude) and the same for the bias"""
        lo, hi = self.live()
        r = torch.arange(self.R, device="cuda")
        prow = (r // self.Rb) * self.Rbp + r % self.Rb
        G = self.G[lo:hi].double()[:, prow]
        X = self.X[lo:hi, :self.C].double()
        c = torch.arange(self.C, device="cuda")
        idx = r[:, None] * self.rs + c[None, :] * self.cs
        return idx, G.t() @ X, G.abs().t() @ X.abs(), G.sum(0), G.abs().sum(0)


def _operands(M, Nn, Kk, R, C, seed):
    """G [M, Nn] / X [M, Kk] with exact-zero pad columns (the layout contract)"""
    torch.manual_seed(seed)
    G = torch.zeros(M, Nn, device="cuda")
    X = torch.zeros(M, Kk, device="cuda")
    G[:, :R] = torch.randn(M, R, device="cuda")
    X[:, :C] = torch.randn(M, C, device="cuda")
    return G, X


def _dw_expect(groups, tc, debug):
    """kernel classes of the weight-gradient dispatchers (csrc/gemm_simt.cu: gemm_dw_group / gemm_dw)"""
    tc3 = bool(tc) and not debug & 1

    def elig(q):
        return q.Nn >= 32 and q.Kk >= 32

    def single(q):
        if q.M <= 0:
            return []
        if q.rows or (tc3 and q.M >= 2048 and elig(q)):
            return [TC_DW]
        return [TC_DW] if (tc and q.M >= 2048 and elig(q)) else [SIMT_DW]

    out = []
    for grp in groups:
        if len(grp) == 1:
            out += single(grp[0])
            continue
        live = [q for q in grp if q.M > 0 and tc3 and elig(q)]
        rest = [q for q in grp if q.M > 0 and q not in live]
        dyn = any(q.rows for q in grp if q.M > 0)
        if live and not dyn and sum(q.M for q in live) < 2048:
            rest, live = rest + live, []
        for q in rest:
            out += single(q)
        out += [TC_DW] if live else []
    return sorted(out)


def _run_dw(groups, plan_rows=0, tc=1, debug=0):
    """all groups in ONE call; returns rc, classes and a check(path) closure against fp64"""
    L = _lib()
    flat = [q for g in groups for q in g]
    arr = (L.DwProblem * len(flat))(*[q.struct() for q in flat])
    sizes = (ctypes.c_int * len(groups))(*[len(g) for g in groups])
    nb = L.lib.gib_test_dw_scratch_bytes(arr, sizes, len(groups), plan_rows)
    assert nb > 0
    scratch = torch.full((nb // 4,), NAN, device="cuda")
    dsts = {}
    for q in flat:   # distinct destination tensors (a strided slice counts as its whole weight), values before the call
        for t in (q.dW, q.dbias):
            if t is not None:
                dsts.setdefault(_root(t).data_ptr(), (_root(t), _root(t).clone()))
    with _mode(tc=tc, debug=debug):
        rc, cls = _profiled(lambda: L.lib.gib_test_dw_groups(arr, sizes, len(groups), plan_rows, _p(scratch), _st()))

    def check(path, what):
        for base_ptr, (t, t0) in dsts.items():
            ref, mag = t0.double().flatten().clone(), t0.double().abs().flatten().clone()
            for q in flat:
                idx, w, wm, b, bm = q.contribution()
                if q.dW is not None and _root(q.dW).data_ptr() == base_ptr:
                    idx = (idx + (q.dW.data_ptr() - base_ptr) // 4).flatten()
                    ref.index_add_(0, idx, w.flatten())
                    mag.index_add_(0, idx, wm.flatten())
                if q.dbias is not None and _root(q.dbias).data_ptr() == base_ptr:
                    idx = torch.arange(q.R, device="cuda") + (q.dbias.data_ptr() - base_ptr) // 4
                    ref.index_add_(0, idx, b)
                    mag.index_add_(0, idx, bm)
            _within(path, t.flatten(), ref, mag, what)

    def untouched(what):
        for t, t0 in dsts.values():
            _same_bits(t, t0, what)

    return rc, cls, check, untouched


def _root(t):
    return t if t._base is None else t._base


def _slice_dst(big, off):
    """a destination that starts `off` floats into `big` (MNN: one weight holds the slices of every bond type)"""
    return big.view(-1)[off:]


MODES = [(1, 0), (0, 0), (1, 1)]


@pytest.mark.parametrize("M", [1, 31, 33, 2047, 2048, 4097, 40000])
@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_single(M, tc, debug):
    """R = 100 -> Nn = 112, C = 136 -> Kk = 144, accumulating into non-zero dW / dbias"""
    G, X = _operands(M, 112, 144, 100, 136, seed=M)
    dW = torch.randn(100, 136, device="cuda")
    db = torch.randn(100, device="cuda")
    groups = [[DW(G, X, M, dW, 100, 136, dbias=db)]]
    rc, cls, check, _ = _run_dw(groups, tc=tc, debug=debug)
    assert rc == 0, _lib().lib.gib_last_error().decode()
    assert cls == _dw_expect(groups, tc, debug), f"M={M}: kernel classes {cls}"
    check(_path(cls), f"dW M={M}")


@pytest.mark.parametrize("M", [33, 4097])
@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_gate_blocked(M, tc, debug):
    """GRU weights: R = 3H rows from the gate blocks of G at columns g * pad16(H)"""
    H, C = 100, 136
    Hp = pad16(H)
    G, X = _operands(M, 3 * Hp, 144, 3 * H, C, seed=M + 1)
    for g in range(3):
        G[:, g * Hp + H:(g + 1) * Hp] = 0
    dW = torch.randn(3 * H, C, device="cuda")
    db = torch.randn(3 * H, device="cuda")
    groups = [[DW(G, X, M, dW, 3 * H, C, dbias=db, Rb=H, Rbp=Hp)]]
    rc, cls, check, _ = _run_dw(groups, tc=tc, debug=debug)
    assert rc == 0 and cls == _dw_expect(groups, tc, debug), cls
    check(_path(cls), f"gate-blocked M={M}")


@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_mnn_strided_slices(tc, debug):
    """MNN: the bond types' [R, H] slices of one weight [R, H, Ef] (src_off = t, rs = H * Ef, cs = Ef), one member each"""
    R, H, Ef = 100, 64, 3
    big = torch.randn(R, H, Ef, device="cuda")
    db = torch.randn(R, device="cuda")
    grp = []
    for t, M in enumerate((2048, 1500, 700)):
        G, X = _operands(M, pad16(R), H, R, H, seed=40 + t)
        grp.append(DW(G, X, M, _slice_dst(big, t), R, H, dbias=db if t == 0 else None, rs=H * Ef, cs=Ef))
    rc, cls, check, _ = _run_dw([grp], tc=tc, debug=debug)
    assert rc == 0 and cls == _dw_expect([grp], tc, debug), cls
    check(_path(cls), "MNN slices")


@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_group_of_16(tc, debug):
    """16 members of different shapes (one empty, some without dbias), planned for more rows than they have"""
    grp = []
    shapes = [(4097, 100, 136), (1, 48, 32), (0, 64, 64), (2047, 256, 48), (33, 608, 144), (5000, 112, 688),
              (128, 64, 256), (3000, 48, 48), (129, 96, 96), (2048, 100, 100), (31, 256, 256), (700, 65, 129),
              (1500, 300, 64), (4096, 32, 32), (257, 128, 608), (999, 80, 112)]
    for k, (M, R, C) in enumerate(shapes):
        G, X = _operands(M, pad16(R), pad16(C), R, C, seed=100 + k)
        dW = torch.randn(R, C, device="cuda")
        db = torch.randn(R, device="cuda") if k % 3 else None
        grp.append(DW(G, X, M, dW, R, C, dbias=db))
    plan = 3 * sum(s[0] for s in shapes)
    rc, cls, check, _ = _run_dw([grp], plan_rows=plan, tc=tc, debug=debug)
    assert rc == 0 and cls == _dw_expect([grp], tc, debug), cls
    if tc and not debug:
        assert cls.count(TC_DW) == 1
    check(_path(cls), "group of 16")


def _shared_buffer_group(cap, Nn, Kk, R, C, ranges, seed):
    """members on disjoint row ranges of ONE buffer (capacity mode's bond-type groups), rows outside every live
    range NaN in G and Inf in X"""
    torch.manual_seed(seed)
    G = torch.full((cap, Nn), NAN, device="cuda")
    X = torch.full((cap, Kk), float("inf"), device="cuda")
    grp = []
    for k, (base, m) in enumerate(ranges):
        hi = min(base + m, cap)
        G[base:hi] = 0
        G[base:hi, :R] = torch.randn(hi - base, R, device="cuda")
        X[base:hi] = 0
        X[base:hi, :C] = torch.randn(hi - base, C, device="cuda")
        dW = torch.randn(R, C, device="cuda")
        db = torch.randn(R, device="cuda")
        grp.append(DW(G, X, cap, dW, R, C, dbias=db, rows=(_dev_int(m), _dev_int(base), base, hi)))
    return grp


@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_device_side_rows(tc, debug):
    """capacity mode: counts and bases in device memory, a count of 0 and one clamped to capacity - base"""
    cap = 8192
    grp = _shared_buffer_group(cap, 112, 144, 100, 136, [(0, 1900), (2048, 0), (4096, 3000), (8064, 500)], seed=9)
    rc, cls, check, untouched = _run_dw([grp], plan_rows=cap, tc=tc, debug=debug)
    if not tc or debug:
        assert rc < 0 and cls == []        # refused before any launch: device-side counts need the tensor cores
        untouched("refused")
        return
    assert rc == 0 and cls == [TC_DW], cls
    check("tc", "device-side rows")


@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_consecutive_groups_share_destinations(tc, debug):
    """the message-pass pattern: four groups in one call add into the SAME dW / dbias (member k of every group into
    destination k; the members of one group write disjoint ones); each group's partials reuse the scratch half of the
    group two before it while the side stream may still be reducing that group"""
    R, C = 100, 136
    dsts = [(torch.randn(R, C, device="cuda"), torch.randn(R, device="cuda")) for _ in range(3)]
    dW2 = torch.randn(48, 64, device="cuda")
    groups, seed = [], 300
    for sizes in ((4097, 2500), (3000, 33, 2048), (40000,), (2047, 5000)):
        grp = []
        for k, M in enumerate(sizes):
            seed += 1
            G, X = _operands(M, 112, 144, R, C, seed=seed)
            grp.append(DW(G, X, M, dsts[k][0], R, C, dbias=dsts[k][1]))
        G, X = _operands(sizes[0], 48, 64, 48, 64, seed=seed + 1000)
        grp.append(DW(G, X, sizes[0], dW2, 48, 64))
        groups.append(grp)
    rc, cls, check, _ = _run_dw(groups, tc=tc, debug=debug)
    assert rc == 0 and cls == _dw_expect(groups, tc, debug), cls
    if tc and not debug:
        assert cls == [TC_DW] * 4
    check(_path(cls), "consecutive groups")


@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_consecutive_device_side_groups(tc, debug):
    """three capacity-mode groups on one scratch, all adding into the first group's destinations"""
    if not tc or debug:
        pytest.skip("device-side counts need the default tensor-core call pattern (refusal: test_dw_device_side_rows)")
    cap = 4096
    groups = [_shared_buffer_group(cap, 112, 144, 100, 136, [(0, 1000), (1024, 2900)], seed=s) for s in (1, 2, 3)]
    for grp in groups[1:]:
        for q, q0 in zip(grp, groups[0]):
            q.dW, q.dbias = q0.dW, q0.dbias
    rc, cls, check, _ = _run_dw(groups, plan_rows=cap, tc=tc, debug=debug)
    assert rc == 0 and cls == [TC_DW] * 3, cls
    check("tc", "consecutive device-side groups")


def test_dw_large_row_count():
    """the largest weight-gradient row count of the C4 shape (155648 rows)"""
    G, X = _operands(155648, 256, 256, 256, 256, seed=5)
    dW = torch.zeros(256, 256, device="cuda")
    db = torch.zeros(256, device="cuda")
    groups = [[DW(G, X, 155648, dW, 256, 256, dbias=db)]]
    rc, cls, check, _ = _run_dw(groups)
    assert rc == 0 and cls == [TC_DW]
    check("tc", "M=155648")
