"""GPU: weight gradients with a pass extent (GemmDW::passes: the message-MLP and GRU weights that every message pass
shares, reduced once over all passes) through gib_test_dw_groups_passes, against float64.

Member p adds  dW += sum_t G_t[live]^T X_t[live]  and  dbias += sum_t colsum(G_t[live])  over its passes t, with prow /
Rb / Rbp / rs / cs as in tests/test_gpu_gemm_patterns.DW; the bound is that file's per-path eps times the same sums over
|G| and |X| (TF32 / bf16 / fp16: the rounded-operand oracles and bounds of tests/test_gpu_tf32.py and
tests/test_gpu_autocast.py).  The slices of one member lie in one allocation, pass_g / pass_x floats apart: tight
(rows * ld, so a k-block that ran past the last row would read the next pass's live rows) or with a gap; gaps and every
row outside the live range are NaN in G and Inf in X, the scratch is NaN, and dW / dbias start non-zero.  Every launch
runs twice from the same destinations and must give the same bits; its kernel classes are checked against the dispatch
rule (tensor cores when M * passes >= 2048 and eligible, else one SIMT launch per pass).
"""
import ctypes

import pytest
import torch

import tests.test_gpu_autocast as A
import tests.test_gpu_gemm_patterns as P
import tests.test_gpu_tf32 as T
from tests.guarded import Guarded
from tests.test_dw_pass_schedule_host import BKF, GRU, MSG, _hook

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
GAP = 4 * 37                   # floats between two slices in the gapped layout (TMA strides are multiples of 16 bytes)
PATH = {1: "tf32", 2: "bf16", 3: "fp16"}    # the tensor-core path of each precision code (0: "tc")
DTYPE16 = {2: torch.bfloat16, 3: torch.float16}
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\npass extent: worst error / magnitude per path:",
          {k: f"{v[0]:.3g} ({v[1]})" for k, v in sorted(WORST.items())})


def _within(path, got, ref, mag, what):
    """records the worst ratio of this file, then the bound of the file that owns the path"""
    ratio = ((got.double() - ref).abs() / (mag + 1e-300)).max().item()
    if not ratio <= WORST.get(path, (0.0, ""))[0]:
        WORST[path] = (ratio, what)
    if path in P.EPS:
        P._within(path, got, ref, mag, what)
    elif path == "tf32":
        T._within(got, ref, mag, what)
    else:
        A._within(got, ref, mag, f"{path} {what}")


class PassDW(P.DW):
    """a P.DW over the slices Gs[t], Xs[t] of its passes, pass_g / pass_x floats apart in one allocation each"""

    def __init__(self, Gs, Xs, M, dW, R, C, pass_g, pass_x, **kw):
        super().__init__(Gs[0], Xs[0], M, dW, R, C, **kw)
        self.passes, self.pass_g, self.pass_x = len(Gs), pass_g, pass_x
        self.parts = [P.DW(g, x, M, dW, R, C, **kw) for g, x in zip(Gs, Xs)]

    def extent(self):
        return P._lib().DwExtent(self.passes, self.pass_g, self.pass_x)

    def contribution(self, oracle=P.DW.contribution):
        """every pass's (index, sum, magnitude, bias sum, bias magnitude) through `oracle`, added up"""
        parts = [oracle(q) for q in self.parts]
        return (parts[0][0],) + tuple(sum(p[i] for p in parts) for i in range(1, 5))


def _oracle(prec, on_tc):
    if not on_tc or prec == 0:
        return P.DW.contribution
    if prec == 1:
        return lambda q: T._RoundedDW(q).contribution()
    return lambda q: A._RoundedDW(q, DTYPE16[prec]).contribution()


def _slices(passes, rows, Nn, Kk, gap):
    """G / X slices of `rows` rows, NaN / Inf throughout; slice t at t * (rows * ld + gap) floats"""
    pg, px = rows * Nn + gap, rows * Kk + gap
    gbuf = torch.full((passes * pg,), NAN, device="cuda")
    xbuf = torch.full((passes * px,), INF, device="cuda")
    Gs = [gbuf[t * pg:t * pg + rows * Nn].view(rows, Nn) for t in range(passes)]
    Xs = [xbuf[t * px:t * px + rows * Kk].view(rows, Kk) for t in range(passes)]
    return Gs, Xs, pg, px


def _fill(Gs, Xs, lo, hi, R, C, Rb=None, Rbp=None):
    """live rows [lo, hi) of every slice: random values in the R / C real columns, +0 in the pad columns (gate-blocked
    G: the real rows of each gate block)"""
    for G, X in zip(Gs, Xs):
        G[lo:hi] = 0
        if Rb is None:
            G[lo:hi, :R] = torch.randn(hi - lo, R, device="cuda")
        else:
            for g in range(R // Rb):
                G[lo:hi, g * Rbp:g * Rbp + Rb] = torch.randn(hi - lo, Rb, device="cuda")
        X[lo:hi] = 0
        X[lo:hi, :C] = torch.randn(hi - lo, C, device="cuda")


def member(M, R, C, passes, Nn=None, Kk=None, gap=0, Rb=None, Rbp=None, dW=None, dbias=True, rs=None, cs=1,
           dev=None, seed=0):
    """one member with its own slices.  dev = (cap, base[, count]): the slices hold cap rows and device-side counts give
    the live range [base, base + count) (count defaults to M; a count past cap - base is clamped)"""
    torch.manual_seed(seed)
    Nn, Kk = Nn or P.pad16(R), Kk or P.pad16(C)
    rows, lo, hi, kw = M, 0, M, {}
    if dev is not None:
        cap, base = dev[:2]
        count = dev[2] if len(dev) > 2 else M
        rows, lo, hi = cap, base, min(base + count, cap)
        kw["rows"] = (P._dev_int(count), P._dev_int(base), lo, hi)
    Gs, Xs, pg, px = _slices(passes, max(rows, 1), Nn, Kk, gap)
    _fill(Gs, Xs, lo, hi, R, C, Rb, Rbp)
    dW = torch.randn(R, C, device="cuda") if dW is None else dW
    db = torch.randn(R, device="cuda") if dbias is True else (dbias if torch.is_tensor(dbias) else None)
    return PassDW(Gs, Xs, rows, dW, R, C, pg, px, dbias=db, Rb=Rb, Rbp=Rbp, rs=rs, cs=cs, **kw)


def shared_buffer_group(cap, passes, Nn, Kk, R, C, ranges, gap=GAP, seed=0):
    """P._shared_buffer_group with a pass dimension: members on disjoint row ranges (base, count) of ONE set of
    capacity slices, through device-side counts (a count past cap - base is clamped)"""
    torch.manual_seed(seed)
    Gs, Xs, pg, px = _slices(passes, cap, Nn, Kk, gap)
    grp = []
    for base, m in ranges:
        hi = min(base + m, cap)
        _fill(Gs, Xs, base, hi, R, C)
        grp.append(PassDW(Gs, Xs, cap, torch.randn(R, C, device="cuda"), R, C, pg, px,
                          dbias=torch.randn(R, device="cuda"), rows=(P._dev_int(m), P._dev_int(base), base, hi)))
    return grp


# ---- dispatch rule -----------------------------------------------------------------------------------------------------
def _dispatch(groups, tc, debug, prec):
    """(sorted kernel classes, per member: ran on the tensor cores) of csrc/gemm_simt.cu: gemm_dw (a group of one) and
    gemm_dw_group with pass extents; None when the call is refused before any launch"""
    tc3 = bool(tc) and not debug & 1
    if prec >= 2 and not tc3:
        return None                           # 16-bit operands need the tensor-core path

    def elig(q):
        return q.dW is not None and q.Nn >= 32 and q.Kk >= 32

    def single(q):
        if q.M <= 0:
            return [], False
        if q.rows:
            return ([P.TC_DW], True) if tc3 and elig(q) else None
        if tc and elig(q) and q.M * q.passes >= 2048:
            return [P.TC_DW], True
        return [P.SIMT_DW] * q.passes, False  # no pass extent on the SIMT kernel: one launch per pass

    cls, on_tc = [], []
    for grp in groups:
        if len(grp) == 1:
            got = single(grp[0])
            if got is None:
                return None
            cls += got[0]
            on_tc.append(got[1])
            continue
        live = [q.M > 0 and tc3 and elig(q) for q in grp]
        if any(q.rows and q.M > 0 and not ok for q, ok in zip(grp, live)):
            return None
        dyn = any(q.rows and q.M > 0 for q in grp)
        if not dyn and sum(q.M * q.passes for q, ok in zip(grp, live) if ok) < 2048:
            live = [False] * len(grp)
        for q, ok in zip(grp, live):
            if not ok:
                got = single(q)
                cls += got[0]
        cls += [P.TC_DW] if any(live) else []
        on_tc += live
    return sorted(cls), on_tc


# ---- one call of the hook ----------------------------------------------------------------------------------------------
def _owner(roots, t):
    for r in roots:
        if r.data_ptr() <= t.data_ptr() < r.data_ptr() + r.numel() * r.element_size():
            return r
    return None


def _call(groups, prec, tc, debug, ext=True):
    """one gib_test_dw_groups_passes call on a NaN scratch: (rc, kernel classes)"""
    L = P._lib()
    flat = [q for g in groups for q in g]
    structs = [q.struct() for q in flat]
    for s in structs:
        s.tf32 = prec
    arr = (L.DwProblem * len(flat))(*structs)
    exts = (L.DwExtent * len(flat))(*[q.extent() for q in flat]) if ext else None
    sizes = (ctypes.c_int * len(groups))(*[len(g) for g in groups])
    nb = L.lib.gib_test_dw_scratch_bytes_passes(arr, exts, sizes, len(groups))
    assert nb > 0, L.lib.gib_last_error().decode()
    scratch = torch.full((nb // 4,), NAN, device="cuda")
    with P._mode(tc=tc, debug=debug):
        return P._profiled(lambda: L.lib.gib_test_dw_groups_passes(arr, exts, sizes, len(groups), P._p(scratch),
                                                                   P._st()))


def run(groups, what, prec=0, tc=1, debug=0, guarded=()):
    """the groups in one call, twice from the same destinations: the kernel classes the dispatch rule gives, the same
    bits both times, the guard bands of `guarded` untouched, and every destination against fp64"""
    flat = [q for g in groups for q in g]
    roots = [g.view(torch.float32) for g in guarded]
    for q in flat:
        for t in (q.dW, q.dbias):
            if t is not None and _owner(roots, t) is None:
                roots.append(P._root(t))
    before = [r.clone() for r in roots]
    expect = _dispatch(groups, tc, debug, prec)
    rc, cls = _call(groups, prec, tc, debug)
    if expect is None:
        assert rc < 0 and cls == [], f"{what}: expected a refusal before any launch, got rc {rc}, classes {cls}"
        for r, r0 in zip(roots, before):
            P._same_bits(r, r0, f"{what}: refused call")
        return
    assert rc == 0, f"{what}: " + P._lib().lib.gib_last_error().decode()
    assert cls == expect[0], f"{what}: kernel classes {cls}, expected {expect[0]}"
    first = [r.clone() for r in roots]
    for r, r0 in zip(roots, before):
        r.copy_(r0)
    assert _call(groups, prec, tc, debug) == (0, cls), f"{what}: second run"
    for r, r1 in zip(roots, first):
        assert torch.equal(r.view(torch.int32), r1.view(torch.int32)), f"{what}: two runs differ"
    for g in guarded:
        assert g.intact(), f"{what}: guard band written at {g.damage()}"
    refs = [[r0.double().flatten().clone(), r0.double().abs().flatten().clone(), set()] for r0 in before]
    for q, on_tc in zip(flat, expect[1]):
        idx, w, wm, b, bm = q.contribution(_oracle(prec, on_tc))
        path = ("tc" if prec == 0 else PATH[prec]) if on_tc else "simt"
        for t, at, v, vm in ((q.dW, idx, w, wm), (q.dbias, torch.arange(q.R, device="cuda"), b, bm)):
            if t is None:
                continue
            k = next(i for i, r in enumerate(roots) if r is _owner(roots, t))
            at = (at + (t.data_ptr() - roots[k].data_ptr()) // 4).flatten()
            refs[k][0].index_add_(0, at, v.flatten())
            refs[k][1].index_add_(0, at, vm.flatten())
            refs[k][2].add(path)
    for r, (ref, mag, paths) in zip(roots, refs):
        path = max(paths, key=lambda p: (p != "simt", p)) if paths else "simt"
        _within(path, r.flatten(), ref, mag, what)


def run_modes(make, what, precs=(1, 2, 3), guarded=()):
    """3xTF32 with tensor cores on, off and under gib_tc_debug bit 0 (as P.MODES), then the other precisions where the
    dispatch rule puts a member on the tensor cores; make() builds fresh groups (and guarded allocations) each time"""
    for tc, debug in P.MODES:
        groups, g = make()
        run(groups, f"{what} [tc={tc} debug={debug}]", 0, tc, debug, g)
    for prec in precs:
        groups, g = make()
        expect = _dispatch(groups, 1, 0, prec)
        if expect is not None and any(expect[1]):
            run(groups, f"{what} [{PATH[prec]}]", prec, 1, 0, g)


# ---- single members ----------------------------------------------------------------------------------------------------
SHAPES = {"message 256x128": dict(R=256, C=128), "GRU H=128": dict(R=384, C=128, Rb=128, Rbp=128)}


@pytest.mark.parametrize("M", [1, 31, 32, 33, 100, 600, 683, 700, 2047, 4097])
@pytest.mark.parametrize("passes", [2, 3, 4, 16])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_single_member_pass_grid(shape, passes, M):
    """C2's message layer and gate-blocked GRU projection over 2-16 passes: M = 683 / 700 at 3 passes reach the tensor
    cores with every pass below their 2048-row threshold, 600 x 3 stays on the SIMT kernel; rows that are fewer than
    one k-block, one exact k-block, one row past it; tight and gapped pass strides"""
    for gap in (0, GAP):
        run_modes(lambda: ([[member(M, passes=passes, gap=gap, seed=M * passes + gap, **SHAPES[shape])]], ()),
                  f"{shape} M={M} passes={passes} gap={gap}")


# ---- segments across pass boundaries -----------------------------------------------------------------------------------
CROSSING = {
    # one 128 x 128 tile, 4 k-blocks per pass, 16 passes: 64 units, 8 CTAs of 8 k-blocks, each across two passes;
    # device-side rows over a buffer of 160 (rows 100..159 NaN / Inf, inside the last k-block's box)
    "one tile, 16 passes, device rows": dict(M=100, R=120, C=100, passes=16, dev=(160, 0)),
    # an odd k-block count per pass (5): the 16-bit fragments alternate f0 / f1 across every pass boundary
    "odd k-blocks, 16 passes": dict(M=130, R=128, C=128, passes=16),
    "odd k-blocks, 3 passes, 2 tiles": dict(M=769, R=256, C=128, passes=3),
    "partial k-block, 4 passes, device rows": dict(M=1900, R=100, C=136, passes=4, dev=(2048, 0)),
}


@pytest.mark.parametrize("case", list(CROSSING))
def test_segments_cross_pass_boundaries(case):
    kw = CROSSING[case]
    m, passes = kw["M"], kw["passes"]
    kb = -(-m // BKF)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    _, segs, _ = _hook([m], [passes], [(P.pad16(kw["R"]), P.pad16(kw["C"]))], sms)
    crossing = [s for s in segs if s[4] // BKF + s[5] > kb]
    assert crossing, f"{case}: no segment crosses a pass boundary on {sms} SMs"
    if kb % 2:
        assert any((kb - s[4] // BKF) % 2 for s in crossing), f"{case}: no crossing segment changes the parity"
    for gap in (0, GAP):
        run_modes(lambda: ([[member(gap=gap, seed=3 + gap, **kw)]], ()), f"{case} gap={gap}")


# ---- device-side counts ------------------------------------------------------------------------------------------------
def test_device_side_rows_with_passes():
    """capacity slices per pass, bond-type members on disjoint live ranges: a count of 0 and one clamped to
    capacity - base (refused before any launch without the tensor-core call pattern)"""
    ranges = [(0, 1900), (2048, 0), (4096, 3000), (8064, 500)]
    run_modes(lambda: ([shared_buffer_group(8192, 3, 112, 144, 100, 136, ranges, seed=9)], ()), "device-side rows")


@pytest.mark.parametrize("prec", [0, 1, 2, 3])
def test_device_counts_compute_what_host_counts_compute(prec):
    """a launch on device-side row counts computes what the same launch on host counts computes, bit for bit: a
    member with count m and base 0 over a buffer of more rows against the host-count member of M = m rows on the same
    slices (same bases, same pass strides)"""
    m, passes, cap = 700, 3, 1024
    dev = member(m, 256, 128, passes, gap=GAP, dev=(cap, 0), seed=11)
    host = PassDW([g[:m] for g in (q.G for q in dev.parts)], [x[:m] for x in (q.X for q in dev.parts)], m,
                  dev.dW.clone(), 256, 128, dev.pass_g, dev.pass_x, dbias=dev.dbias.clone())
    for q in (dev, host):
        assert _dispatch([[q]], 1, 0, prec) == ([P.TC_DW], [True])
        rc, cls = _call([[q]], prec, 1, 0)
        assert rc == 0 and cls == [P.TC_DW], (rc, cls)
    assert torch.equal(dev.dW.view(torch.int32), host.dW.view(torch.int32))
    assert torch.equal(dev.dbias.view(torch.int32), host.dbias.view(torch.int32))


# ---- groups of 17 and 32 -----------------------------------------------------------------------------------------------
LIVE = (13452, 2242, 320)       # the bond types' message rows of a C2 batch
GRU_ROWS = 5000


def _group_17(device):
    """C2's deferred launch: 5 message-MLP layers x 3 bond types, then the GRU pair, all over 4 passes"""
    passes, grp = 4, []
    for li, (nn, kk) in enumerate(MSG):
        if device:   # one capacity buffer per layer, the bond types at 128-row aligned bases
            grp += shared_buffer_group(16384, passes, nn, kk, nn, kk, [(0, LIVE[0]), (13568, LIVE[1]),
                                                                       (15872, LIVE[2])], seed=50 + li)
        else:
            grp += [member(m, nn, kk, passes, gap=GAP, seed=50 + 3 * li + t) for t, m in enumerate(LIVE)]
    for k, (nn, kk) in enumerate(GRU):
        grp.append(member(GRU_ROWS, nn, kk, passes, Rb=128, Rbp=128, gap=GAP, seed=90 + k))
    assert len(grp) == 17
    return [grp], ()


def _group_32(device):
    """passes 1 and 2-16 mixed, empty members between them, some without dbias, ragged 144-wide shapes, and four MNN
    bond-type slices of one weight [R, H, Ef] (rs = H * Ef, cs = Ef) in a guarded allocation; with device-side counts
    every member sits at base 8 of a buffer 40 rows longer than its count, one count is clamped, and the empty members
    have a count of 0"""
    R, H, Ef = 100, 64, 4
    g = Guarded(R * H * Ef * 4, fill=None)
    big = g.view(torch.float32, (R, H, Ef))
    big.copy_(torch.randn(R, H, Ef, device="cuda"))
    mnn_bias = torch.randn(R, device="cuda")
    shapes = [(100, 136), (144, 128), (128, 144), (256, 144)]
    grp = []
    for k in range(32):
        passes = (1, 3, 16, 2, 4)[k % 5]
        m = 0 if k % 8 == 5 else (31, 100, 700, 2047, 33, 4097, 129)[k % 7]
        dev = None
        if device:
            dev = (m + 40, 8, m + 100) if k == 6 else (m + 40, 8)
        if 8 <= k < 12:
            t = k - 8
            grp.append(member(m, R, H, passes, Kk=H, gap=GAP, dW=P._slice_dst(big, t),
                              dbias=mnn_bias if t == 0 else None, rs=H * Ef, cs=Ef, dev=dev, seed=200 + k))
        else:
            r, c = shapes[k % 4]
            grp.append(member(m, r, c, passes, gap=GAP if k % 2 else 0, dbias=k % 3 != 2, dev=dev, seed=200 + k))
    return [grp], (g,)


@pytest.mark.parametrize("device", [False, True], ids=["host counts", "device counts"])
@pytest.mark.parametrize("size", [17, 32])
def test_groups_of_17_and_32(size, device):
    make = _group_17 if size == 17 else _group_32
    run_modes(lambda: make(device), f"group of {size} ({'device' if device else 'host'} counts)")


# ---- consecutive groups ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc,debug", P.MODES)
def test_consecutive_pass_groups_share_destinations(tc, debug):
    """four pass-extent groups in one call add into the SAME dW / dbias (member k of every group into destination k):
    each group's partials reuse the scratch half of the group two before it while the side stream may still be
    reducing that group; one group is a single member (gemm_dw), one stays below the tensor-core threshold"""
    R, C = 100, 136
    dsts = [(torch.randn(R, C, device="cuda"), torch.randn(R, device="cuda")) for _ in range(3)]
    dW2 = torch.randn(48, 64, device="cuda")
    groups, seed = [], 400
    for spec in (((4097, 2), (700, 3)), ((683, 3), (33, 16), (2048, 1)), ((100, 16),), ((31, 4), (129, 3)),
                 ((2047, 4), (600, 3))):
        grp = []
        for k, (m, passes) in enumerate(spec):
            seed += 1
            grp.append(member(m, R, C, passes, gap=GAP if seed % 2 else 0, dW=dsts[k][0], dbias=dsts[k][1],
                              seed=seed))
        if len(spec) > 1:
            grp.append(member(spec[0][0], 48, 64, spec[0][1], dW=dW2, dbias=False, seed=seed + 1000))
        groups.append(grp)
    run(groups, f"consecutive groups [tc={tc} debug={debug}]", 0, tc, debug)
    if tc and not debug:
        for prec in (1, 2, 3):      # from the destinations the run before left
            run(groups, f"consecutive groups [{PATH[prec]}]", prec, 1, 0)


# ---- anchors -----------------------------------------------------------------------------------------------------------
def _group_16():
    shapes = [(4097, 100, 136), (1, 48, 32), (0, 64, 64), (2047, 256, 48), (33, 608, 144), (5000, 112, 688),
              (128, 64, 256), (3000, 48, 48), (129, 96, 96), (2048, 100, 100), (31, 256, 256), (700, 65, 129),
              (1500, 300, 64), (4096, 32, 32), (257, 128, 608), (999, 80, 112)]
    grp = []
    for k, (m, R, C) in enumerate(shapes):
        G, X = P._operands(m, P.pad16(R), P.pad16(C), R, C, seed=100 + k)
        grp.append(P.DW(G, X, m, torch.randn(R, C, device="cuda"), R, C,
                        dbias=torch.randn(R, device="cuda") if k % 3 else None))
    return [grp]


@pytest.mark.parametrize("tc,debug", P.MODES)
@pytest.mark.parametrize("prec", [0, 1, 2])
def test_one_pass_is_bit_identical_to_the_one_pass_hook(tc, debug, prec):
    """passes = 1 (ext = NULL, and an explicit extent of one pass with strides that mean nothing) computes what
    gib_test_dw_groups computes on the same problems, bit for bit: P's group of 16, a single member and
    device-side rows"""
    if prec >= 2 and (not tc or debug):
        pytest.skip("16-bit operands need the tensor-core call pattern")
    cases = [_group_16(), [[P.DW(*P._operands(4097, 112, 144, 100, 136, seed=1), 4097, torch.randn(100, 136,
                                                                                                   device="cuda"),
                                 100, 136, dbias=torch.randn(100, device="cuda"))]]]
    if tc and not debug:
        cases.append([P._shared_buffer_group(8192, 112, 144, 100, 136, [(0, 1900), (2048, 0), (4096, 3000),
                                                                        (8064, 500)], seed=9)])
    L = P._lib()
    for groups in cases:
        flat = [q for g in groups for q in g]
        structs = [q.struct() for q in flat]
        for s in structs:
            s.tf32 = prec
        arr = (L.DwProblem * len(flat))(*structs)
        sizes = (ctypes.c_int * len(groups))(*[len(g) for g in groups])
        dsts = [t for q in flat for t in (q.dW, q.dbias) if t is not None]
        init = [t.clone() for t in dsts]
        outs = []
        for hook in ("one pass", "ext = NULL", "explicit extent"):
            for t, t0 in zip(dsts, init):
                t.copy_(t0)
            if hook == "one pass":
                nb = L.lib.gib_test_dw_scratch_bytes(arr, sizes, len(groups), 0)
            else:
                ext = None if hook == "ext = NULL" else (L.DwExtent * len(flat))(
                    *[L.DwExtent(1, -1, 7) for _ in flat])
                nb = L.lib.gib_test_dw_scratch_bytes_passes(arr, ext, sizes, len(groups))
            scratch = torch.full((nb // 4,), NAN, device="cuda")
            with P._mode(tc=tc, debug=debug):
                if hook == "one pass":
                    rc = L.lib.gib_test_dw_groups(arr, sizes, len(groups), 0, P._p(scratch), P._st())
                else:
                    rc = L.lib.gib_test_dw_groups_passes(arr, ext, sizes, len(groups), P._p(scratch), P._st())
            torch.cuda.synchronize()
            outs.append((rc, [t.clone() for t in dsts]))
        for rc, got in outs[1:]:
            assert rc == outs[0][0], (rc, outs[0][0])
            for a, b in zip(got, outs[0][1]):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "passes = 1 differs from the one-pass hook"
