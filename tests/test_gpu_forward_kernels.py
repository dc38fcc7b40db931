"""GPU: the forward graph kernels, the layout glue, the weight packing and the loss / sampler heads one at a time,
through the C-ABI, against float64 (csrc/graph_ops.cu, csrc/api.cu).

Inputs follow tests/test_gpu_graph_kernels.py: CSRs with segment degrees 0 to 300 (and the 4-entry trip boundary of
K2), energies up to |100| (expf overflows fp32 past 88: a softmax without its max shift fails), bond values w in
{0.5, 1, 2}, and the CSRs K0 builds from a real batch.  Bound, per element: |got - ref| <= EPS * (|ref| + m), m the
magnitude of the terms that enter the element, plus a fixed slack where the kernel evaluates a SELU derivative from its
output (2^-21 absolute), adds a long row in fp32 (depth * 2^-24 * the sum of |terms|) or takes an exp whose result
lies below the smallest normal fp32 (2^-126 absolute: a denormal or a flush to 0).  Outputs and rows a kernel
must not write start as NaN / 7.0 and come back bit-identical; pad columns must be +0; kernels that only move data
must match bit for bit.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# 4 x (rounded down) the worst error / magnitude over the whole file, measured on an H100 80GB HBM3 (SXM, 700 W power
# limit): 1.92e-7 (tanh_fwd)
EPS = 7.6e-7
SELU_S, SELU_A = 1.0507009873554805, 1.6732632423543772
DACT = 2.0 ** -21
U32 = 2.0 ** -24
TINY = 2.0 ** -126     # below the smallest normal fp32 an exp result loses its relative precision or flushes to 0
WORST = [0.0, ""]
NAN = float("nan")


def _lib():
    from graphinvent_b200 import _lib
    return _lib


def _p(t):
    return t.data_ptr() if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    assert rc == 0, f"{what}: {rc} {_lib().lib.gib_last_error().decode()}"


def _dev_int(v):
    return torch.tensor([v], dtype=torch.int32, device="cuda")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print(f"\nworst error / magnitude: {WORST[0]:.3g} ({WORST[1]})")


def _within(got, ref, mag, what, slack=0.0):
    """|got - ref| <= EPS * (|ref| + mag) + slack elementwise (NaN fails); records the worst (err - slack) / scale"""
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (ref.abs() + mag + 1e-300)).max().item() if err.numel() else 0.0
    if ratio >= WORST[0]:
        WORST[:] = [ratio, what]
    assert ratio <= EPS, f"{what}: error / magnitude {ratio:.3g} > {EPS:.1e}"


def _same_bits(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), f"{what}: changed"


def _plus_zero(t, what):
    assert (t.contiguous().view(torch.int32) == 0).all(), f"{what}: not +0"


def _dselu64(y):
    return torch.where(y > 0, torch.full_like(y, SELU_S), y + SELU_S * SELU_A)


def _selu_out(shape, scale):
    """SELU outputs (what the kernels receive as EM / EN): selu of normal * scale"""
    return torch.selu((torch.randn(*shape, device="cuda") * scale).clamp(-90.0, 90.0))


def _degree_csr(degs, seed):
    """CSR over len(degs) segments with the given degrees; entry rows are a random permutation"""
    g = torch.Generator().manual_seed(seed)
    degs = torch.tensor(degs)
    ptr = torch.zeros(len(degs) + 1, dtype=torch.int32)
    ptr[1:] = degs.cumsum(0)
    E = int(degs.sum())
    ent = torch.randperm(E, generator=g).int()
    seg_of_pos = torch.repeat_interleave(torch.arange(len(degs)), degs)
    seg = torch.empty(E, dtype=torch.long)
    seg[ent.long()] = seg_of_pos                      # segment of every entry row
    return ptr.cuda(), ent.cuda(), seg.cuda(), E


DEGS = [0, 1, 40, 300, 0, 1, 1, 40, 2, 300, 7, 0]
# K2 reads 4 entries per trip: degrees around the trip boundary; 13 segments, so the 2-slot variants have a last thread
# whose second slot lies past S
K2_DEGS = [0, 1, 3, 4, 5, 8, 9, 40, 300, 0, 4, 9, 1]


_K0 = []


def _k0_graph():
    """the EMN entries K0 builds from a real batch with a degree-5 atom and a self loop: (ent_dst, ent_src, dst_ptr,
    src_ptr, src_ent) on the device, S, E (built once per module)"""
    if not _K0:
        _K0.append(_build_k0_graph())
    return _K0[0]


def _build_k0_graph():
    from graphinvent_b200 import functional as Fn, synthetic as Sy
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = O.make_constants("EMN", max_n_nodes=40, n_node_features=12, len_f_add_per_node=81)
    _, e = Sy.random_graphs(32, 40, 9, 3, seed=5)
    edges = torch.from_numpy(e).float()
    edges[3, 0, 0, 1] = 1.0                          # self loop
    for k in range(1, 6):                            # atom 0 of molecule 4: degree 5
        edges[4, 0, k] = 0; edges[4, k, 0] = 0
        edges[4, 0, k, 0] = 1.0; edges[4, k, 0, 0] = 1.0
    net = mpnn.create(C)
    d = Fn.make_dims(net, edges.shape[0])
    g = Fn.GraphBatch(d, edges.cuda())
    torch.cuda.synchronize()
    E, S = int(g.hdr_np[0]), edges.shape[0] * edges.shape[1]
    arrays = [g.array(d, k, n).clone() for k, n in ((1, E), (0, E), (3, S + 1), (5, S + 1), (6, E))]
    return arrays, S, E


# ----------------------------------------------------------------------------------------------------------------------
# K2 scatter-aggregate
# ----------------------------------------------------------------------------------------------------------------------
def _scatter(out, msg, ld, ptr, ent, w, acc, S):
    _ok(_lib().lib.gib_test_scatter_sum(_p(out), _p(msg), ld, _p(ptr), _p(ent), _p(w), acc, S, _st()), "scatter_sum")


def _scatter_ref(out0, msg, ptr, ent, w, acc):
    """fp64: out0 (accumulate) + sum over every segment of w * msg, and the magnitude of the terms"""
    S = ptr.numel() - 1
    ent = ent.long()
    seg = torch.repeat_interleave(torch.arange(S, device="cuda"), (ptr[1:] - ptr[:-1]).long())
    ww = w.double()[ent, None] if w is not None else 1.0
    terms = msg.double()[ent] * ww
    ref = torch.zeros(S, msg.shape[1], dtype=torch.float64, device="cuda").index_add(0, seg, terms)
    mag = torch.zeros_like(ref).index_add(0, seg, terms.abs())
    if acc:
        ref, mag = ref + out0[:S].double(), mag + out0[:S].double().abs()
    return ref, mag


def _scatter_case(ptr, ent, E, ld, w, acc, what, tail=5):
    """one launch over S = len(ptr) - 1 segments: entry rows past E are NaN (never read), output rows past S stay"""
    S = ptr.numel() - 1
    msg = torch.randn(E + tail, ld, device="cuda")
    msg[E:] = NAN
    out = torch.randn(S + tail, ld, device="cuda") if acc else torch.full((S + tail, ld), NAN, device="cuda")
    out[S:] = 7.0
    out0 = out.clone()
    _scatter(out, msg, ld, ptr, ent, w, acc, S)
    ref, mag = _scatter_ref(out0, msg[:E], ptr, ent, w, acc)
    _within(out[:S], ref, mag, what)
    empty = (ptr[1:] == ptr[:-1])
    if not acc:
        _plus_zero(out[:S][empty], what + " empty segments")
    _same_bits(out[S:], out0[S:], what + " rows past S")
    return out


def _bond_w(n):
    return torch.tensor([0.5, 1.0, 2.0], device="cuda")[torch.randint(0, 3, (n,), device="cuda")]


@pytest.mark.parametrize("wmode", ["none", "0.5/1/2"])
@pytest.mark.parametrize("acc", [0, 1])
@pytest.mark.parametrize("variant", [0, 1, 2, 3])
def test_scatter_sum(variant, acc, wmode):
    """every K2 variant (1 / 2 slots per thread, default / streaming hints), with and without accumulation (the
    backward gather-reduce adds into dh), over degrees 0-300 and the CSRs K0 builds from a real batch"""
    L = _lib().lib
    torch.manual_seed(variant * 4 + acc * 2 + (wmode != "none"))
    L.gib_scatter_variant(variant)
    try:
        ptr, ent, _, E = _degree_csr(K2_DEGS, seed=variant)
        for ld in (16, 112):
            w = _bond_w(E + 5) if wmode != "none" else None
            _scatter_case(ptr, ent, E, ld, w, acc, f"scatter v{variant} acc={acc} w={wmode} ld={ld}")
        (ent_dst, ent_src, dst_ptr, src_ptr, src_ent), S, E = _k0_graph()
        ident = torch.arange(E, dtype=torch.int32, device="cuda")
        for name, p, e in (("K0 dst", dst_ptr, ident), ("K0 src", src_ptr, src_ent)):
            w = _bond_w(E + 5) if wmode != "none" else None
            _scatter_case(p, e, E, 48, w, acc, f"scatter v{variant} acc={acc} w={wmode} {name}")
    finally:
        L.gib_scatter_variant(2)


def test_scatter_sum_variants_are_bit_identical():
    """accumulation is ascending in q in every variant: the four variants agree bit for bit with each other and with a
    repeat run, at the degree CSR and at the C4 shape (155648 slots, 352256 entries, 112 columns)"""
    L = _lib().lib
    torch.manual_seed(3)
    g = torch.Generator().manual_seed(4)
    S4, E4, ld4 = 155648, 352256, 112
    dst = torch.randint(0, S4, (E4,), generator=g)
    ptr4 = torch.zeros(S4 + 1, dtype=torch.int32)
    ptr4[1:] = torch.bincount(dst, minlength=S4).cumsum(0).int()
    ent4 = torch.randperm(E4, generator=g).int()
    ptrd, entd, _, Ed = _degree_csr(K2_DEGS, seed=9)
    cases = [("degrees", ptrd, entd, Ed, 16), ("C4", ptr4.cuda(), ent4.cuda(), E4, ld4)]
    try:
        for name, ptr, ent, E, ld in cases:
            S = ptr.numel() - 1
            msg = torch.randn(E, ld, device="cuda")
            w = torch.rand(E, device="cuda") + 0.5
            base = torch.randn(S, ld, device="cuda")
            for acc in (0, 1):
                first = None
                for variant in (0, 1, 2, 3, 2):
                    L.gib_scatter_variant(variant)
                    out = base.clone() if acc else torch.full((S, ld), NAN, device="cuda")
                    _scatter(out, msg, ld, ptr, ent, w, acc, S)
                    if first is None:
                        first = out
                        ref, mag = _scatter_ref(base, msg, ptr, ent, w, acc)
                        _within(out, ref, mag, f"scatter {name} acc={acc}")
                    else:
                        _same_bits(out, first, f"scatter {name} acc={acc} variant {variant} vs variant 0")
    finally:
        L.gib_scatter_variant(2)


# ----------------------------------------------------------------------------------------------------------------------
# K2' segmented softmax
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wmode", ["none", "0.5/1/2"])
@pytest.mark.parametrize("scale", [1.0, 45.0])
def test_seg_softmax_fwd(wmode, scale):
    """out[s] = sum_p softmax_p(w EN) w EM over the degree CSR; |w EN| up to 100 at scale 45; empty segments give +0"""
    torch.manual_seed(int(scale) + (wmode != "none"))
    ptr, ent, seg, E = _degree_csr(DEGS, seed=3)
    S, ld, tail = len(DEGS), 48, 64
    EM = _selu_out((E + tail, ld), 1.0)
    EN = _selu_out((E + tail, ld), scale)
    EM[E:] = NAN; EN[E:] = NAN                          # rows of no segment: never read
    w = _bond_w(E + tail) if wmode != "none" else None
    out = torch.full((S + 3, ld), NAN, device="cuda")
    out[S:] = 7.0
    out0 = out.clone()
    _ok(_lib().lib.gib_seg_softmax(_p(out), _p(EM), _p(EN), ld, _p(ptr), _p(ent), _p(w), S, _st()), "seg_softmax")
    # the fp64 expression of tests/test_gpu_graph_kernels.py (_seg_softmax_ref)
    ww = w[:E].double()[:, None] if w is not None else torch.ones(E, 1, dtype=torch.float64, device="cuda")
    e = ww * EN[:E].double()
    assert e.abs().max() > (80 if scale > 1 else 0)
    mx = torch.full((S, ld), -float("inf"), dtype=torch.float64, device="cuda")
    mx = mx.scatter_reduce(0, seg[:, None].expand_as(e), e, "amax")
    x = torch.exp(e - mx[seg])
    den = torch.zeros(S, ld, dtype=torch.float64, device="cuda").index_add(0, seg, x)
    num = torch.zeros_like(den).index_add(0, seg, x * ww * EM[:E].double())
    nonempty = (ptr[1:] > ptr[:-1])
    ref = torch.where(nonempty[:, None], num / den, torch.zeros_like(den))
    R = torch.zeros_like(den).scatter_reduce(0, seg[:, None].expand_as(e), e.abs(), "amax")
    V = torch.zeros_like(den).scatter_reduce(0, seg[:, None].expand_as(e), (ww * EM[:E].double()).abs(), "amax")
    _within(out[:S], ref, (1 + R) * V, f"seg_softmax scale={scale} w={wmode}")
    _plus_zero(out[:S][~nonempty], "seg_softmax empty segments")
    _same_bits(out[S:], out0[S:], "seg_softmax rows past S")


# ----------------------------------------------------------------------------------------------------------------------
# GRU gates
# ----------------------------------------------------------------------------------------------------------------------
def _gru_fwd_ref(gi, gh, h, H):
    """fp64 torch.nn.GRUCell gate expression (r, z, n) over gate-blocked gi / gh, and the magnitude of every output:
    1 - z cancels, so the bound carries |n| and |h| whole, and the rounding of every gate argument through its slope"""
    Hp = gi.shape[1] // 3
    gi64, gh64 = gi.double(), gh.double().expand(gi.shape[0], -1)
    h64 = h.double() if h is not None else torch.zeros(gi.shape[0], Hp, dtype=torch.float64, device="cuda")
    ir, iz, in_ = gi64[:, :Hp], gi64[:, Hp:2 * Hp], gi64[:, 2 * Hp:]
    hr, hz, hn_ = gh64[:, :Hp], gh64[:, Hp:2 * Hp], gh64[:, 2 * Hp:]
    r = torch.sigmoid(ir + hr)
    z = torch.sigmoid(iz + hz)
    n = torch.tanh(in_ + r * hn_)
    ref = (1 - z) * n + z * h64
    mag = (n.abs() + h64.abs()
           + (1 - z) * (1 - n * n) * (in_.abs() + r * hn_.abs() + r * (1 - r) * (1 + ir.abs() + hr.abs()) * hn_.abs())
           + z * (1 - z) * (1 + iz.abs() + hz.abs()) * (h64 - n).abs())
    return ref, mag


def _gru_inputs(S, H, Hp, rows_gh, saturate):
    """gate-blocked gi / gh with zero pad columns (as the packed GEMMs store them); the second half of the rows at
    pre-activations up to +-90 when saturate"""
    def blocked(rows, scale):
        t = torch.zeros(rows, 3 * Hp, device="cuda")
        for k in range(3):
            t[:, k * Hp:k * Hp + H] = torch.randn(rows, H, device="cuda") * scale
        return t
    gi, gh = blocked(S, 2.0), blocked(rows_gh, 2.0)
    if saturate:
        big = blocked(S, 40.0).clamp(-60.0, 60.0)
        gi[S // 2:] = big[S // 2:]
        gh_big = blocked(rows_gh, 20.0).clamp(-30.0, 30.0)
        gh[rows_gh // 2:] = gh_big[rows_gh // 2:]
    return gi, gh


@pytest.mark.parametrize("saturate", [False, True])
@pytest.mark.parametrize("form", ["node", "emn"])
def test_gru_fwd(form, saturate):
    """node form: rows with an empty CSR segment keep h bit for bit.  EMN form: h = NULL, ONE gh bias row, a live count
    below S, rows at or past it untouched.  Saturated gates (pre-activations up to +-90) give no NaN; pad columns +0"""
    torch.manual_seed(17 + saturate)
    S, H = 700, 100
    Hp = (H + 15) // 16 * 16
    emn = form == "emn"
    gi, gh = _gru_inputs(S, H, Hp, 1 if emn else S, saturate)
    if saturate:
        assert (gi + gh).abs().max() > 80
    hn = torch.full((S, Hp), NAN, device="cuda")
    if emn:
        h, ptr, live_n = None, None, 555
        live = _dev_int(live_n)
        gi[live_n:] = NAN                              # rows past the live count: never read
        active = torch.ones(S, dtype=torch.bool, device="cuda")
    else:
        h = torch.zeros(S, Hp, device="cuda")
        h[:, :H] = torch.randn(S, H, device="cuda")
        active = torch.rand(S, device="cuda") < 0.7
        ptr = torch.zeros(S + 1, dtype=torch.int32, device="cuda")
        ptr[1:] = active.int().cumsum(0)
        live_n, live = S, None
    hn0 = hn.clone()
    _ok(_lib().lib.gib_test_gru_fwd(_p(hn), _p(gi), _p(gh), _p(h), Hp, _p(ptr), S, _p(live), _st()), "gru_fwd")
    n = live_n
    ref, mag = _gru_fwd_ref(gi[:n], gh, h[:n] if h is not None else None, H)
    a = active[:n]
    what = f"gru_fwd {form}" + (" saturated" if saturate else "")
    _within(hn[:n][a][:, :H], ref[a][:, :H], mag[a][:, :H], what)
    assert not hn[:n].isnan().any()
    _plus_zero(hn[:n, H:], what + " pad columns")
    if emn:
        _same_bits(hn[n:], hn0[n:], what + " rows past the live count")
    else:
        _same_bits(hn[~active], h[~active], what + " rows with an empty segment")


# ----------------------------------------------------------------------------------------------------------------------
# readouts
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 13, 40])
def test_graph_gather_fwd(N):
    """masked softmax over the atoms of every molecule (modules.py:39-52): energies en - 1e6 * (mask == 0) formed in
    fp32 as the reference does, softmax in fp64; g and the stored attention the backward consumes.  Molecules with no
    active atom, with every atom active, energies up to |100|"""
    torch.manual_seed(N)
    B, W, ld = 40, 100, 112
    en = torch.zeros(B * N, ld, device="cuda"); em = torch.zeros(B * N, ld, device="cuda")
    en[:, :W] = (torch.randn(B * N, W, device="cuda") * 45).clamp(-100, 100)
    em[:, :W] = _selu_out((B * N, W), 1.0)
    en[: 10 * N, :W] = torch.randn(10 * N, W, device="cuda") * 2          # a few molecules at ordinary energies
    mask = torch.rand(B, N) < 0.6
    mask[0] = False; mask[1] = True; mask[5] = False; mask[6] = True
    ptr = torch.zeros(B * N + 1, dtype=torch.int32)
    ptr[1:] = mask.view(-1).int().cumsum(0).int()
    ptr = ptr.cuda()
    g = torch.full((B + 2, ld), NAN, device="cuda"); g[B:] = 7.0
    att = torch.full((B * N + 2, ld), NAN, device="cuda"); att[B * N:] = 7.0
    g0, att0 = g.clone(), att.clone()
    _ok(_lib().lib.gib_graph_gather(_p(g), _p(att), _p(en), _p(em), ld, _p(ptr), N, B, 1e6, _st()), "gather")
    e32 = en.view(B, N, ld) - ((~mask).float() * 1e6).cuda()[:, :, None]      # fp32, the reference's quantisation
    e = e32.double()
    mx = e.max(1, keepdim=True).values
    x = torch.exp(e - mx)
    a = x / x.sum(1, keepdim=True)
    m = em.double().view(B, N, ld)
    ref_g = (a * m).sum(1)
    D = (a * (1 + (e - mx).abs())).sum(1, keepdim=True)
    mag_a = a * (1 + (e - mx).abs()) + a * D
    _within(att[:B * N].view(B, N, ld), a, mag_a, f"graph_gather att N={N}", TINY)
    _within(g[:B], ref_g, (mag_a * m.abs()).sum(1) + (a * m.abs()).sum(1), f"graph_gather g N={N}",
            TINY * m.abs().sum(1))
    _plus_zero(g[:B, W:], "graph_gather pad columns")
    _same_bits(g[B:], g0[B:], "graph_gather rows past B")
    _same_bits(att[B * N:], att0[B * N:], "graph_gather attention rows past B*N")


@pytest.mark.parametrize("N", [1, 13, 40])
def test_sum_nodes_fwd_and_bcast_nodes_add(N):
    """MNN readout g[b] = sum_i h[b*N + i] and its backward dh[s] += dg[s / N] (into a non-zero dh)"""
    L = _lib().lib
    torch.manual_seed(N)
    B, ld = 37, 112
    S = B * N
    h = torch.randn(S, ld, device="cuda") * 3
    g = torch.full((B + 2, ld), NAN, device="cuda"); g[B:] = 7.0
    g0 = g.clone()
    _ok(L.gib_test_sum_nodes_fwd(_p(g), _p(h), ld, N, B, _st()), "sum_nodes_fwd")
    h64 = h.double().view(B, N, ld)
    _within(g[:B], h64.sum(1), h64.abs().sum(1), f"sum_nodes N={N}")
    _same_bits(g[B:], g0[B:], "sum_nodes rows past B")
    dg = torch.randn(B, ld, device="cuda")
    dh = torch.randn(S + 3, ld, device="cuda")
    dh[S:] = 7.0
    dh0 = dh.clone()
    _ok(L.gib_test_bcast_nodes_add(_p(dh), _p(dg), ld, N, S, _st()), "bcast_nodes_add")
    b_of = torch.arange(S, device="cuda") // N
    ref = dh0[:S].double() + dg.double()[b_of]
    _within(dh[:S], ref, dh0[:S].double().abs() + dg.double()[b_of].abs(), f"bcast_nodes_add N={N}")
    _same_bits(dh[S:], dh0[S:], "bcast_nodes_add rows past S")


# ----------------------------------------------------------------------------------------------------------------------
# layout glue
# ----------------------------------------------------------------------------------------------------------------------
def _i8(rows, cols):
    t = torch.randint(-128, 128, (rows, cols), dtype=torch.int8, device="cuda")
    t[0, 0], t[0, 1] = -128, 127
    return t


def test_concat2_in():
    """dst = [a[:, :wa] | b[:, :wb] | +0] bit for bit: int8 inputs (-128 and 127 included), float inputs, b = NULL with
    wb = 0 (the first hidden state), and a == b (the EMN's [h | h])"""
    L = _lib().lib
    torch.manual_seed(0)
    rows, ldd = 301, 112
    hT = torch.randn(rows, 112, device="cuda")
    nodes8, nodesf = _i8(rows, 12), torch.randn(rows, 12, device="cuda")
    cases = [("float | int8", hT, 112, 100, 0, nodes8, 12, 12, 1),
             ("float | float", hT, 112, 100, 0, nodesf, 12, 12, 0),
             ("int8 | NULL", nodes8, 12, 12, 1, None, 0, 0, 0),
             ("float | NULL", nodesf, 12, 12, 0, None, 0, 0, 0),
             ("int8 | int8", nodes8, 12, 9, 1, nodes8, 12, 12, 1),
             ("a == b", hT, 112, 50, 0, hT, 112, 50, 0)]
    for what, a, lda, wa, a8, b, ldb, wb, b8 in cases:
        dst = torch.full((rows + 2, ldd), NAN, device="cuda"); dst[rows:] = 7.0
        dst0 = dst.clone()
        _ok(L.gib_test_concat2_in(_p(dst), ldd, _p(a), lda, wa, a8, _p(b), ldb, wb, b8, rows, _st()), what)
        ref = torch.zeros(rows, ldd, device="cuda")
        ref[:, :wa] = a[:, :wa].float()
        if b is not None:
            ref[:, wa:wa + wb] = b[:, :wb].float()
        _same_bits(dst[:rows], ref, f"concat2_in {what}")
        _same_bits(dst[rows:], dst0[rows:], f"concat2_in {what} rows past the count")


def test_concat_flat_and_unflatten_dact():
    """the fAdd / fConn head glue with N * fa wider than a row of f1 (modules.py:257-268): concat_flat bit for bit,
    unflatten_dact against fp64 with zero pad columns"""
    L = _lib().lib
    torch.manual_seed(1)
    B, N, fa, ldf, W, ldg = 29, 13, 81, 96, 100, 112
    S = B * N
    ldd = (N * fa + W + 15) // 16 * 16
    assert N * fa > ldf
    f1 = torch.full((S, ldf), NAN, device="cuda")
    f1[:, :fa] = _selu_out((S, fa), 1.5)                                 # columns past fa: never read
    g = torch.full((B, ldg), NAN, device="cuda")
    g[:, :W] = torch.randn(B, W, device="cuda")
    dst = torch.full((B + 1, ldd), NAN, device="cuda"); dst[B:] = 7.0
    dst0 = dst.clone()
    _ok(L.gib_test_concat_flat(_p(dst), ldd, _p(f1), ldf, N, fa, _p(g), ldg, W, B, _st()), "concat_flat")
    ref = torch.zeros(B, ldd, device="cuda")
    ref[:, :N * fa] = f1[:, :fa].reshape(B, N * fa)
    ref[:, N * fa:N * fa + W] = g[:, :W]
    _same_bits(dst[:B], ref, "concat_flat")
    _same_bits(dst[B:], dst0[B:], "concat_flat rows past B")

    dcat = torch.randn(B, ldd, device="cuda")
    G = torch.full((S + 1, ldf), NAN, device="cuda"); G[S:] = 7.0
    G0 = G.clone()
    _ok(L.gib_test_unflatten_dact(_p(G), ldf, _p(dcat), ldd, _p(f1), N, fa, S, _st()), "unflatten_dact")
    d = dcat[:, :N * fa].double().reshape(S, fa)
    ds = _dselu64(f1[:, :fa].double())
    _within(G[:S, :fa], d * ds, d.abs() * ds.abs(), "unflatten_dact", d.abs() * DACT)
    _plus_zero(G[:S, fa:], "unflatten_dact pad columns")
    _same_bits(G[S:], G0[S:], "unflatten_dact rows past S")


@pytest.mark.parametrize("act", [1, 2])
def test_dact_slice(act):
    """G[m, n] = dout[m, off + n] * act'(out[m, off + n]) for a head slice at off > 0 of the APD row; pads +0"""
    torch.manual_seed(act)
    B, apd, off, width, ldg = 77, 625, 13 * 9, 13 * 36, 480
    pre = torch.randn(B, apd, device="cuda") * 2
    out = torch.selu(pre) if act == 1 else torch.tanh(pre)
    dout = torch.randn(B, apd, device="cuda")
    G = torch.full((B + 1, ldg), NAN, device="cuda"); G[B:] = 7.0
    G0 = G.clone()
    _ok(_lib().lib.gib_test_dact_slice(_p(G), ldg, _p(dout), _p(out), apd, off, width, act, B, _st()), "dact_slice")
    y = out[:, off:off + width].double()
    d = dout[:, off:off + width].double()
    da = _dselu64(y) if act == 1 else 1 - y * y
    # tanh: 1 - y^2 in fp32 cancels near |y| = 1 (absolute error ~2^-24 of the 1)
    _within(G[:B, :width], d * da, d.abs() * (da.abs() + (act == 2)), f"dact_slice act={act}", d.abs() * DACT)
    _plus_zero(G[:B, width:], "dact_slice pad columns")
    _same_bits(G[B:], G0[B:], "dact_slice rows past B")


def test_sum3_cols():
    """dst = a[:, offa:] + b2[:, offb:] + c3 over W columns, +0 up to ldd: with NULL operands, and with dst == c3 (the
    hidden-state gradient of modules.py:46 added into dh in place)"""
    L = _lib().lib
    torch.manual_seed(2)
    rows, W, ldd, lda = 503, 100, 112, 240
    a = torch.randn(rows, lda, device="cuda"); b2 = torch.randn(rows, lda, device="cuda")
    c3 = torch.full((rows, ldd), NAN, device="cuda"); c3[:, :W] = torch.randn(rows, W, device="cuda")
    for what, ua, ub, uc in (("a + b + c", 1, 1, 1), ("a", 1, 0, 0), ("b + c", 0, 1, 1), ("none", 0, 0, 0),
                             ("dst == c3", 1, 1, 2)):
        dst = torch.full((rows + 1, ldd), NAN, device="cuda"); dst[rows:] = 7.0
        if uc == 2:
            dst[:rows] = c3
        dst0 = dst.clone()
        cptr = dst if uc == 2 else (c3 if uc else None)
        _ok(L.gib_test_sum3_cols(_p(dst), ldd, W, _p(a) if ua else None, lda, 17, _p(b2) if ub else None, lda, 100,
                                 _p(cptr), ldd, rows, _st()), what)
        terms = []
        if ua:
            terms.append(a[:, 17:17 + W].double())
        if ub:
            terms.append(b2[:, 100:100 + W].double())
        if uc:
            terms.append(c3[:, :W].double())
        ref = sum(terms) if terms else torch.zeros(rows, W, dtype=torch.float64, device="cuda")
        mag = sum(t.abs() for t in terms) if terms else torch.zeros_like(ref)
        _within(dst[:rows, :W], ref, mag, f"sum3_cols {what}")
        _plus_zero(dst[:rows, W:], f"sum3_cols {what} pad columns")
        _same_bits(dst[rows:], dst0[rows:], f"sum3_cols {what} rows past the count")


@pytest.mark.parametrize("live_n", [None, 0, 333, 5000])
def test_emn_elementwise_live_counts(live_n):
    """tanh_fwd, tanh_selu_bwd and mul_dselu over the first min(*live, rows) rows; rows past it untouched"""
    L = _lib().lib
    torch.manual_seed(7)
    rows, ld = 700, 112
    n = rows if live_n is None else min(live_n, rows)
    live = None if live_n is None else _dev_int(live_n)
    pre = _selu_out((rows, ld), 2.0)                  # the SELU output that feeds tanh
    x = pre.clone()
    x[n:] = NAN
    y = torch.full((rows, ld), 7.0, device="cuda")
    y0 = y.clone()
    _ok(L.gib_test_tanh_fwd(_p(y), _p(x), rows, ld, _p(live), _st()), "tanh_fwd")
    _within(y[:n], torch.tanh(pre[:n].double()), torch.zeros(n, ld, dtype=torch.float64, device="cuda"), "tanh_fwd")
    _same_bits(y[n:], y0[n:], "tanh_fwd rows past the live count")

    yt = torch.tanh(pre)
    dy = torch.randn(rows, ld, device="cuda")
    dy[n:] = NAN
    G = torch.full((rows, ld), NAN, device="cuda")
    G0 = G.clone()
    _ok(L.gib_test_tanh_selu_bwd(_p(G), _p(dy), _p(yt), _p(pre), rows, ld, _p(live), _st()), "tanh_selu_bwd")
    d, t, ds = dy[:n].double(), yt[:n].double(), _dselu64(pre[:n].double())
    ref = d * (1 - t * t) * ds
    _within(G[:n], ref, d.abs() * ds.abs(), "tanh_selu_bwd", (d * (1 - t * t)).abs() * DACT)
    _same_bits(G[n:], G0[n:], "tanh_selu_bwd rows past the live count")

    G = torch.full((rows, ld), 7.0, device="cuda")
    G0 = G.clone()
    _ok(L.gib_test_mul_dselu(_p(G), _p(dy), _p(pre), rows, ld, _p(live), _st()), "mul_dselu")
    _within(G[:n], d * ds, torch.zeros_like(ref), "mul_dselu", d.abs() * DACT)
    _same_bits(G[n:], G0[n:], "mul_dselu rows past the live count")


@pytest.mark.parametrize("live_n", [None, 0, 1999, 5000])
@pytest.mark.parametrize("scale", [0, 1])
def test_gather_rows(scale, live_n):
    """dst[p] = (scale ? w_p : 1) * h[src_p] bit for bit; pad rows (src = -1) give +0; rows past the live count stay"""
    L = _lib().lib
    torch.manual_seed(scale)
    S, P, ld = 500, 3000, 112
    n = P if live_n is None else min(live_n, P)
    h = torch.randn(S, ld, device="cuda")
    src = torch.randint(0, S, (P,), dtype=torch.int32, device="cuda")
    src[::7] = -1
    src[n:] = -7                                       # past the live count: never read
    w = _bond_w(P)
    dst = torch.full((P, ld), NAN, device="cuda")
    dst0 = dst.clone()
    live = None if live_n is None else _dev_int(live_n)
    _ok(L.gib_test_gather_rows(_p(dst), _p(h), ld, _p(src), _p(w), scale, P, _p(live), _st()), "gather_rows")
    s = src[:n].long()
    ref = h[s.clamp(min=0)] * (w[:n, None] if scale else 1.0)
    ref[s < 0] = 0.0
    _same_bits(dst[:n], ref, f"gather_rows scale={scale}")
    _same_bits(dst[n:], dst0[n:], "gather_rows rows past the live count")


@pytest.mark.parametrize("i8", [0, 1])
def test_emn_input(i8):
    """X[r] = [nodes[i] | nodes[j] | edges[i, j % N] | +0] bit for bit, from int8 and float inputs, with self loops,
    molecules past the first, and pad entries (i = -1) that give +0"""
    L = _lib().lib
    torch.manual_seed(i8)
    B, N, F, Ef, ld = 6, 13, 12, 3, 32
    S = B * N
    if i8:
        nodes = _i8(S, F)
        edges = torch.randint(-128, 128, (B, N, N, Ef), dtype=torch.int8, device="cuda")
        edges.view(-1)[:2] = torch.tensor([-128, 127], dtype=torch.int8, device="cuda")
    else:
        nodes = torch.randn(S, F, device="cuda")
        edges = torch.randn(B, N, N, Ef, device="cuda")
    P, pad = 400, 37
    b = torch.randint(0, B, (P,), device="cuda")
    i = torch.randint(0, N, (P,), device="cuda"); j = torch.randint(0, N, (P,), device="cuda")
    j[::11] = i[::11]                                  # self loops
    ent_dst = torch.cat([b * N + i, torch.full((pad,), -1, device="cuda")]).int()
    ent_src = torch.cat([b * N + j, torch.full((pad,), -1, device="cuda")]).int()
    X = torch.full((P + pad + 1, ld), NAN, device="cuda"); X[P + pad:] = 7.0
    X0 = X.clone()
    _ok(L.gib_test_emn_input(_p(X), ld, _p(nodes), _p(edges), i8, _p(ent_dst), _p(ent_src), N, F, Ef, P + pad,
                             _st()), "emn_input")
    ref = torch.zeros(P + pad, ld, device="cuda")
    si, sj = (b * N + i), (b * N + j)
    ref[:P, :F] = nodes[si].float()
    ref[:P, F:2 * F] = nodes[sj].float()
    ref[:P, 2 * F:2 * F + Ef] = edges[b, i, j].float()
    assert int((b > 0).sum()) > 0 and int((si == sj).sum()) > 0
    _same_bits(X[:P + pad], ref, f"emn_input i8={i8}")
    _same_bits(X[P + pad:], X0[P + pad:], "emn_input rows past P")


# ----------------------------------------------------------------------------------------------------------------------
# weight packing (gib_model_pack)
# ----------------------------------------------------------------------------------------------------------------------
def _rna_tf32(v):
    """float32 -> TF32 (10-bit mantissa), round to nearest with ties away from zero, as float32 with the low 13 bits 0"""
    bits = np.ascontiguousarray(v, dtype=np.float32).view(np.uint32)
    return ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("model", ["GGNN", "MNN", "AttGGNN", "EMN"])
def test_model_pack_layout(model, big):
    """every Linear's Wp / WTp / bp equals the state_dict tensor placed by the plan (MNN strided slices of
    message_weights, the GRU's three gate blocks, Ct < C transposes) bit for bit, with +0 pads; the TF32 planes are
    hi = rna(v) and lo = rna(v - hi) with 13 zero low mantissa bits and |v - hi - lo| <= 2^-21 |v|.
    Deliberate constraint on the packing kernel, not a correctness property of the packed weights: the arena's
    alignment gaps between Linears stay unwritten (a NaN-filled arena keeps its NaNs there), so that a write outside a
    Linear's ranges is caught.  A packer that zero-fills the arena first would have to drop this check."""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import PLAN_LINEAR_FIELDS
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    L = _lib().lib
    kw = dict(hidden_node_features=128, message_size=128, message_passes=4, edge_emb_size=128,
              max_n_nodes=38, n_node_features=12, len_f_add_per_node=81) if big else {}
    torch.manual_seed(5)
    net = mpnn.create(O.make_constants(model, **kw))
    sd = net.state_dict()
    names = list(sd.keys())
    params = [(sd[k].float() + 0.01 * torch.randn_like(sd[k].float())).contiguous().cuda() for k in names]
    d = Fn.make_dims(net, 64)
    nbytes = L.gib_model_packed_bytes(ctypes.byref(d))
    packed = torch.full((nbytes // 4,), NAN, device="cuda")
    _ok(L.gib_model_pack(ctypes.byref(d), Fn._ptr_table(params), _p(packed), _st()), "gib_model_pack")
    arena = packed.cpu().numpy()
    written = np.zeros(arena.size, dtype=bool)
    host = [p.cpu().numpy() for p in params]
    out = (ctypes.c_longlong * len(PLAN_LINEAR_FIELDS))()
    n = L.gib_test_plan_linear(ctypes.byref(d), 0, out)
    assert n > 0
    seen_gru = seen_mnn = 0
    for li in range(n):
        assert L.gib_test_plan_linear(ctypes.byref(d), li, out) == n
        f = dict(zip(PLAN_LINEAR_FIELDS, out))
        nblk, Rb, Rbp, C, Cp, Ct, Ctp = (f[k] for k in ("nblk", "Rb", "Rbp", "C", "Cp", "Ct", "Ctp"))
        Rp = nblk * Rbp
        wname, W = names[f["pw"]], host[f["pw"]]
        # the source matrix [nblk * Rb, C] of this Linear, independent of the plan's strides
        if W.ndim == 3:                                            # MNN message_weights [msg, H, Ef]: slice t
            src = W[:, :, f["src_off"]]
            assert f["rs"] == W.shape[1] * W.shape[2] and f["cs"] == W.shape[2]
            seen_mnn += 1
        else:
            src = W
            assert f["src_off"] == 0 and f["rs"] == C and f["cs"] == 1
        assert src.shape == (nblk * Rb, C), (wname, src.shape, nblk, Rb, C)
        if "weight_ih" in wname or "weight_hh" in wname:
            assert nblk == 3
            seen_gru += 1
        Wp = np.zeros((Rp, Cp), np.float32)
        bp = np.zeros(Rp, np.float32)
        bias = host[f["pb"]] if f["pb"] >= 0 else None
        for gb in range(nblk):
            Wp[gb * Rbp:gb * Rbp + Rb, :C] = src[gb * Rb:(gb + 1) * Rb]
            if bias is not None:
                bp[gb * Rbp:gb * Rbp + Rb] = bias[gb * Rb:(gb + 1) * Rb]
        WTp = np.zeros((Ctp, Rp), np.float32)
        WTp[:Ct] = Wp[:, :Ct].T
        what = f"{model}{' big' if big else ''} Linear {li} ({wname})"
        for key, want in (("ow", Wp), ("owt", WTp), ("ob", bp)):
            got = arena[f[key]:f[key] + want.size]
            assert np.array_equal(_bits(got), _bits(want.ravel())), f"{what}: {key}"
            written[f[key]:f[key] + want.size] = True
        for base, v in (("ow", Wp.ravel()), ("owt", WTp.ravel())):
            hi = arena[f[base + "_hi"]:f[base + "_hi"] + v.size]
            lo = arena[f[base + "_lo"]:f[base + "_lo"] + v.size]
            written[f[base + "_hi"]:f[base + "_hi"] + v.size] = True
            written[f[base + "_lo"]:f[base + "_lo"] + v.size] = True
            assert not (_bits(hi) & 0x1FFF).any() and not (_bits(lo) & 0x1FFF).any(), f"{what}: {base} plane low bits"
            assert np.array_equal(_bits(hi), _bits(_rna_tf32(v))), f"{what}: {base}_hi is not rna(v)"
            assert np.array_equal(_bits(lo), _bits(_rna_tf32(v - hi))), f"{what}: {base}_lo is not rna(v - hi)"
            resid = np.abs(v.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
            assert (resid <= 2.0 ** -21 * np.abs(v.astype(np.float64))).all(), f"{what}: {base} planes"
    assert seen_gru == 2 and seen_mnn == (d.Ef if model == "MNN" else 0)
    assert np.isnan(arena[~written]).all(), "gib_model_pack wrote outside its Linears' ranges"


# ----------------------------------------------------------------------------------------------------------------------
# loss and sampler heads
# ----------------------------------------------------------------------------------------------------------------------
APDS = [1, 200, 256, 257, 625, 2000]
KINDS = ("dense", "sparse", "one-hot", "wide", "one-hot wide", "zero")


def _heads_batch(apd, B=60, seed=0):
    """B rows of logits and targets, row r of kind KINDS[r % 6]: dense / sparse (every third action 0) / one-hot
    targets at logits ~ N(0, 3^2); dense and one-hot (at the row's largest logit) targets at logits up to +-80; and an
    all-zero target row"""
    torch.manual_seed(seed * 1000 + apd)
    out = torch.randn(B, apd, device="cuda") * 3
    tgt = torch.rand(B, apd, device="cuda")
    kind = torch.arange(B, device="cuda") % len(KINDS)
    wide = (kind == 3) | (kind == 4)
    out[wide] = (torch.rand(int(wide.sum()), apd, device="cuda") * 160 - 80)
    tgt[kind == 1, 1::3] = 0
    for k, pos in ((2, None), (4, "argmax")):
        rows = (kind == k).nonzero()[:, 0]
        tgt[rows] = 0
        at = out[rows].argmax(1) if pos else torch.randint(0, apd, (rows.numel(),), device="cuda")
        tgt[rows, at] = 1.0
    tgt[kind == 5] = 0
    return out, tgt, kind


def _depth(apd):
    """the longest chain of fp32 additions in block_reduce<256>: a thread's strided terms, 5 shuffles, 8 warp sums"""
    return (apd + 255) // 256 + 5 + 8


@pytest.mark.parametrize("apd", APDS)
def test_kl_loss_fwd_bwd(apd):
    """loss[b] = sum_k th log th - th (o - lse), th = t / sum(t) and dout = (softmax(o) - th) * scale against fp64; an
    all-zero target row gives NaN, as in the reference"""
    out, tgt, kind = _heads_batch(apd)
    B, scale = out.shape[0], 1.0 / 60
    loss = torch.full((B + 1,), 7.0, device="cuda")
    dout = torch.full((B + 1, apd), 7.0, device="cuda")
    _ok(_lib().lib.gib_kl_loss_fwd_bwd(_p(out), _p(tgt), B, apd, scale, _p(loss), _p(dout), _st()), "kl_loss")
    assert loss[B] == 7.0 and (dout[B] == 7.0).all()
    ok = kind != 5
    o, t = out[ok].double(), tgt[ok].double()
    ts = t.sum(1, keepdim=True)
    th = t / ts
    mx = o.max(1, keepdim=True).values
    lse = mx + torch.log(torch.exp(o - mx).sum(1, keepdim=True))
    logp = o - lse
    xlogx = torch.where(th > 0, th * torch.log(th.clamp(min=1e-300)), torch.zeros_like(th))
    terms = xlogx - th * logp
    ref = terms.sum(1)
    # per term: th log th and th logp, with logp = o - (mx + log(sum exp(o - mx))) formed in fp32; the fp32 sums of t
    # and of the terms add depth * 2^-24 relative
    m_terms = xlogx.abs() + th * (1 + logp.abs() + o.abs() + lse.abs() + mx.abs())
    _within(loss[:B][ok], ref, m_terms.sum(1), f"kl_loss rows apd={apd}", _depth(apd) * U32 * 2 * m_terms.sum(1))
    p = torch.exp(logp)
    ref_d = (p - th) * scale
    mag_d = (p * (1 + (o - mx).abs() + lse.abs() + mx.abs()) + th) * scale
    _within(dout[:B][ok], ref_d, mag_d, f"kl_loss dout apd={apd}", (_depth(apd) * U32 * 2 * (p + th) + TINY) * scale)
    assert loss[:B][~ok].isnan().all() and dout[:B][~ok].isnan().all()


@pytest.mark.parametrize("apd", APDS)
def test_validation_nll(apd):
    """nll[b] = -log(sum_k softmax(o)_k t_k / sum(t)) against fp64; an all-zero target row gives NaN.
    Deliberately not covered: a one-hot target on an action whose probability underflows fp32 (wide logits, o_k - max
    below about -103).  There the sum is 0 and the kernel gives +inf, as an fp32 evaluation of the reference does,
    while fp64 gives a finite value; the wide-logit one-hot rows here put the target on the row's largest logit."""
    out, tgt, kind = _heads_batch(apd, seed=1)
    B = out.shape[0]
    nll = torch.full((B + 1,), 7.0, device="cuda")
    _ok(_lib().lib.gib_validation_nll(_p(out), _p(tgt), B, apd, _p(nll), _st()), "validation_nll")
    assert nll[B] == 7.0
    ok = kind != 5
    o, t = out[ok].double(), tgt[ok].double()
    mx = o.max(1, keepdim=True).values
    e = torch.exp(o - mx)
    ref = -torch.log((e * t).sum(1) / e.sum(1) / t.sum(1))
    # -log turns relative errors of the three sums into absolute ones: exp arguments up to |o - mx|, fp32 sum depth
    mag = 1 + ((o - mx).abs() * (t > 0)).max(1).values
    _within(nll[:B][ok], ref, mag, f"validation_nll apd={apd}", 3 * _depth(apd) * U32 * 4)
    assert nll[:B][~ok].isnan().all()


@pytest.mark.parametrize("apd", APDS)
def test_sample_actions(apd):
    """inverse-CDF sampling: the chosen index lies in its fp64 CDF bracket, its fp32 probability is > 0, its likelihood
    matches fp64; u = 0, u just below 1, logits up to +-80, rows whose trailing actions have probability 0, and a NaN
    row that gives (apd - 1, NaN)"""
    torch.manual_seed(apd)
    B = 4096
    out = torch.randn(B, apd, device="cuda") * 3
    out[1::4] = torch.rand(B // 4, apd, device="cuda") * 160 - 80
    # rows 2 mod 4: every action from a random cut on has probability 0 in fp32
    cut = torch.randint(1, apd + 1, (B,), device="cuda")
    dead = (torch.arange(apd, device="cuda")[None, :] >= cut[:, None]) & (torch.arange(B, device="cuda") % 4 == 2)[:, None]
    out[dead] = -1e4
    u = torch.rand(B, device="cuda")
    u[0::8] = 0.0
    u[1::8] = 1.0 - 2.0 ** -24                     # the largest float below 1
    u[2::8] = 1.0 - 2.0 ** -24
    u[3::8] = 1.0 - 2.0 ** -22
    nan_row = B - 1
    out[nan_row, apd // 2] = NAN
    action = torch.full((B + 1,), -5, dtype=torch.int32, device="cuda")
    lik = torch.full((B + 1,), 7.0, device="cuda")
    _ok(_lib().lib.gib_sample_actions(_p(out), B, apd, _p(u), _p(action), _p(lik), _st()), "sample_actions")
    assert action[B] == -5 and lik[B] == 7.0
    assert action[nan_row] == apd - 1 and lik[nan_row].isnan()
    a, lk, o, uu = action[:nan_row].long(), lik[:nan_row], out[:nan_row], u[:nan_row].double()
    assert ((a >= 0) & (a < apd)).all()
    mx32 = o.max(1, keepdim=True).values
    p32 = torch.exp(o - mx32).gather(1, a[:, None])[:, 0]
    bad = (p32 == 0).nonzero()[:, 0]
    assert bad.numel() == 0, f"apd={apd}: {bad.numel()} rows picked an action of probability 0 (rows {bad[:8].tolist()})"
    p = torch.softmax(o.double(), 1)
    cdf = p.cumsum(1)
    lo = torch.where(a > 0, cdf.gather(1, (a - 1).clamp(min=0)[:, None])[:, 0], torch.zeros_like(uu))
    hi = cdf.gather(1, a[:, None])[:, 0]
    assert ((lo - 1e-5 <= uu) & (uu <= hi + 1e-5)).all(), f"apd={apd}: index outside its CDF bracket"
    pa = p.gather(1, a[:, None])[:, 0]
    mx = o.double().max(1).values
    arg = (o.double().gather(1, a[:, None])[:, 0] - mx).abs()
    # the total is a fixed-order prefix over 256 chunk sums: 256 + ceil(apd / 256) sequential fp32 additions
    _within(lk, pa, pa * (1 + arg), f"sample_actions lik apd={apd}", pa * (256 + (apd + 255) // 256) * U32 * 2 + TINY)


@pytest.mark.parametrize("n", [1, 255, 4096])
def test_sum_scaled(n):
    """out = scale * sum(rows), one fixed-order CTA"""
    torch.manual_seed(n)
    rows = torch.randn(n, device="cuda") * 5 + 1
    o = torch.full((2,), 7.0, device="cuda")
    scale = 1.0 / 3
    _ok(_lib().lib.gib_sum_scaled(_p(rows), n, scale, _p(o), _st()), "sum_scaled")
    r = rows.double()
    s32 = torch.tensor(scale, dtype=torch.float32).double()
    ref = r.sum() * s32
    mag = r.abs().sum() * s32
    _within(o[:1], ref.reshape(1), mag.reshape(1), f"sum_scaled n={n}", (_depth(n) * U32 * 2 * mag).reshape(1))
    assert o[1] == 7.0
