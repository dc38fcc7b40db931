"""GPU: the backward and EMN line-graph kernels of csrc/graph_ops.cu one at a time, through the C-ABI test hooks,
against float64 autograd of the forward expression they differentiate (graph_gather_bwd: its backward formula evaluated
in float64 at the forward kernel's stored attention).

CSRs: random ones with segment degrees 0, 1, 40 and 300, energies up to |100| (expf overflows fp32 past 88: a softmax
without its max shift fails), bond values w in {0.5, 1, 2}, and the CSRs K0 builds from real batches.  Bound, per
element: |got - ref| <= EPS * (|ref| + m), m the magnitude of the terms that enter the element (for a softmax:
(1 + max |energy|) * |upstream| * max |value| over its set, since fp32 rounds the energies before the exp).  Rows a
kernel must not touch start as NaN / 7.0 and come back bit-identical.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

# 4 x (rounded down) the worst error / magnitude over the whole sweep, measured on an H100 80GB HBM3 (SXM):
# 9.33e-7 (the EMN aggregation's forward)
EPS = 3.7e-6
SELU_S, SELU_A = 1.0507009873554805, 1.6732632423543772
DACT = 2.0 ** -21
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


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print(f"\nworst error / magnitude: {WORST[0]:.3g} ({WORST[1]})")


def _within(got, ref, mag, what, slack=0.0):
    """|got - ref| <= EPS * (|ref| + mag) + slack, slack: the fp32 evaluation of a SELU / tanh derivative from its
    output (2^-21 absolute) times what it multiplies"""
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (ref.abs() + mag + 1e-300)).max().item() if err.numel() else 0.0
    if ratio >= WORST[0]:
        WORST[:] = [ratio, what]
    assert ratio <= EPS, f"{what}: error / magnitude {ratio:.3g} > {EPS:.1e}"


def _same_bits(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), f"{what}: changed"


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


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("wmode", ["none", "0.5/1/2"])
def test_scatter_bwd(act, wmode):
    """G[p] = w_p dM[dst_p] act'(Y_p): autograd of out[s] = sum_p w_p act(pre_p); pad rows (dst = -1) give zeros"""
    torch.manual_seed(act)
    S, P, ld = 50, 3000, 112
    dst = torch.randint(0, S, (P,), device="cuda", dtype=torch.int32)
    dst[::7] = -1
    pre = (torch.randn(P, ld, device="cuda", dtype=torch.float64) * 2).requires_grad_(True)
    Y = {0: pre, 1: torch.selu(pre), 2: torch.tanh(pre)}[act].detach().float()
    w = torch.tensor([0.5, 1.0, 2.0], device="cuda")[torch.randint(0, 3, (P,), device="cuda")] if wmode != "none" else None
    dM = torch.randn(S, ld, device="cuda")
    # forward in fp64 at the fp32 outputs: act'(pre) evaluated through Y, as the kernel does
    y64 = Y.double().requires_grad_(True)
    live = dst >= 0
    contrib = y64 * (w.double()[:, None] if w is not None else 1.0) * live[:, None]
    out = torch.zeros(S, ld, dtype=torch.float64, device="cuda").index_add(0, dst.clamp(min=0).long(), contrib)
    (gy,) = torch.autograd.grad(out, y64, dM.double())
    dact = {0: torch.ones_like(y64), 1: _dselu64(y64), 2: 1 - y64 * y64}[act].detach()
    ref = gy * dact
    G = torch.full((P, ld), NAN, device="cuda")
    _ok(_lib().lib.gib_test_scatter_bwd(_p(G), _p(dM), _p(Y), ld, _p(dst), _p(w), act, P, _st()), "scatter_bwd")
    _within(G, ref, gy.abs() * dact.abs(), "scatter_bwd", gy.abs() * DACT)
    assert (G[~live] == 0).all()


def _seg_softmax_ref(EM, EN, w, seg, S, dM):
    """fp64 autograd of out[s, c] = sum_{p in s} softmax_p(w EN)[c] * w EM[p, c] with respect to the SELU inputs of
    EM / EN (through their outputs), and the magnitude of every gradient element"""
    em = EM.double().requires_grad_(True)
    en = EN.double().requires_grad_(True)
    ww = w.double()[:, None] if w is not None else torch.ones(EM.shape[0], 1, dtype=torch.float64, device="cuda")
    e = ww * en
    mx = torch.full((S, EM.shape[1]), -float("inf"), dtype=torch.float64, device="cuda")
    mx = mx.scatter_reduce(0, seg[:, None].expand_as(e), e.detach(), "amax")
    x = torch.exp(e - mx[seg])
    den = torch.zeros_like(mx).index_add(0, seg, x)
    num = torch.zeros_like(mx).index_add(0, seg, x * ww * em)
    out = num / den
    gm, gn = torch.autograd.grad(out, (em, en), torch.nan_to_num(dM.double(), nan=0.0))
    R = torch.zeros_like(mx).scatter_reduce(0, seg[:, None].expand_as(e), e.detach().abs(), "amax")
    V = torch.zeros_like(mx).scatter_reduce(0, seg[:, None].expand_as(e), (ww * em).detach().abs(), "amax")
    mag = ((1 + R) * V * dM.double().abs())[seg] * ww.abs()
    dsm, dsn = _dselu64(EM.double()), _dselu64(EN.double())
    return gm * dsm, gn * dsn, mag * dsm.abs(), mag * dsn.abs(), mag


@pytest.mark.parametrize("wmode", ["none", "0.5/1/2"])
@pytest.mark.parametrize("scale", [1.0, 45.0])
def test_seg_softmax_bwd(wmode, scale):
    """|w EN| up to 100 at scale 45; entries of no segment (the tail rows) stay untouched"""
    torch.manual_seed(int(scale))
    ptr, ent, seg, E = _degree_csr(DEGS, seed=3)
    S, ld, tail = len(DEGS), 48, 64
    EM = _selu_out((E + tail, ld), 1.0)
    EN = _selu_out((E + tail, ld), scale)
    assert EN.abs().max() < 100
    w = torch.tensor([0.5, 1.0, 2.0], device="cuda")[torch.randint(0, 3, (E + tail,), device="cuda")] \
        if wmode != "none" else None
    dM = torch.randn(S, ld, device="cuda")
    GM = torch.full((E + tail, ld), NAN, device="cuda")
    GN = torch.full((E + tail, ld), 7.0, device="cuda")
    _ok(_lib().lib.gib_test_seg_softmax_bwd(_p(GM), _p(GN), _p(dM), _p(EM), _p(EN), ld, _p(ptr), _p(ent), _p(w), S,
                                            _st()), "seg_softmax_bwd")
    rm, rn, mm, mn, m0 = _seg_softmax_ref(EM[:E], EN[:E], w[:E] if w is not None else None, seg, S, dM)
    _within(GM[:E], rm, mm, "GM", m0 * DACT)
    _within(GN[:E], rn, mn, "GN", m0 * DACT)
    assert GM[E:].isnan().all() and (GN[E:] == 7.0).all()


def _gru_ref(gi, gh, h, d, active, emn):
    """fp64 autograd of torch.nn.GRUCell's gate expression (r, z, n order) over gate-blocked gi / gh"""
    Hp = d.shape[1]
    gi64 = gi.double().requires_grad_(True)
    gh64 = gh.double().requires_grad_(True)
    h64 = (h.double() if h is not None else torch.zeros_like(d, dtype=torch.float64)).requires_grad_(True)
    ghr = gh64.expand(gi.shape[0], -1) if emn else gh64
    r = torch.sigmoid(gi64[:, :Hp] + ghr[:, :Hp])
    z = torch.sigmoid(gi64[:, Hp:2 * Hp] + ghr[:, Hp:2 * Hp])
    n = torch.tanh(gi64[:, 2 * Hp:] + r * ghr[:, 2 * Hp:])
    hn = torch.where(active[:, None], (1 - z) * n + z * h64, h64)
    dgi, dgh_full, dh = torch.autograd.grad(hn, (gi64, ghr, h64), d.double(), allow_unused=True)
    mag = d.double().abs() * (1 + h64.detach().abs() + n.detach().abs() + ghr[:, 2 * Hp:].detach().abs())
    return dgi, dgh_full, dh, mag


@pytest.mark.parametrize("form", ["node", "emn"])
def test_gru_bwd(form):
    """node form: rows with an empty CSR segment give dgi = dgh = 0 and dh = d.  EMN form: h = NULL, ONE gh bias row,
    a live count < S, rows at or past it untouched"""
    torch.manual_seed(11)
    S, H = 700, 100
    Hp = (H + 15) // 16 * 16
    emn = form == "emn"
    gi = torch.randn(S, 3 * Hp, device="cuda") * 2
    gh = torch.randn(1 if emn else S, 3 * Hp, device="cuda") * 2
    h = None if emn else torch.randn(S, Hp, device="cuda")
    d = torch.randn(S, Hp, device="cuda")
    if emn:
        active = torch.ones(S, dtype=torch.bool, device="cuda")
        ptr, live_n = None, 555
        live = torch.tensor([live_n], dtype=torch.int32, device="cuda")
    else:
        active = torch.rand(S, device="cuda") < 0.7
        ptr = torch.zeros(S + 1, dtype=torch.int32, device="cuda")
        ptr[1:] = active.int().cumsum(0)
        live_n, live = S, None
    dgi = torch.full((S, 3 * Hp), NAN, device="cuda")
    dgh = torch.full((S, 3 * Hp), 7.0, device="cuda")
    dh = torch.full((S, Hp), NAN, device="cuda") if not emn else None
    _ok(_lib().lib.gib_test_gru_bwd(_p(dgi), _p(dgh), _p(dh), _p(d), _p(gi), _p(gh), _p(h), Hp, _p(ptr), S, _p(live),
                                    _st()), "gru_bwd")
    rgi, rgh, rdh, mag = _gru_ref(gi, gh, h, d, active, emn)
    n = live_n
    m3 = mag.repeat(1, 3)
    _within(dgi[:n], rgi[:n], m3[:n], "dgi")
    _within(dgh[:n], rgh[:n], m3[:n], "dgh")
    if not emn:
        _within(dh, rdh, mag, "dh")
        assert (dgi[~active] == 0).all() and (dgh[~active] == 0).all()
        assert torch.equal(dh[~active], d[~active])
    else:
        assert dgi[n:].isnan().all() and (dgh[n:] == 7.0).all()


@pytest.mark.parametrize("live_n", [None, 0, 777, 5000])
def test_colsum_add(live_n):
    """out[r] += sum_m G[m, prow(r)], gate-blocked rows (Rb = 100, Rbp = 112), over the first *live rows"""
    torch.manual_seed(5)
    M, H = 3000, 100
    Hp = 112
    G = torch.randn(M, 3 * Hp, device="cuda")
    n = M if live_n is None else min(live_n, M)
    G[n:] = NAN
    out = torch.randn(3 * H, device="cuda")
    out0 = out.clone()
    live = None if live_n is None else torch.tensor([live_n], dtype=torch.int32, device="cuda")
    _ok(_lib().lib.gib_test_colsum_add(_p(out), _p(G), 3 * Hp, M, 3 * H, H, Hp, _p(live), _st()), "colsum")
    r = torch.arange(3 * H, device="cuda")
    prow = (r // H) * Hp + r % H
    Gs = G[:n].double()[:, prow]
    _within(out, out0.double() + Gs.sum(0), out0.double().abs() + Gs.abs().sum(0), "colsum")


def test_graph_gather_bwd():
    """the backward formula in fp64 at the forward kernel's stored attention, incl. molecules without bonds"""
    L = _lib()
    torch.manual_seed(1)
    B, N, W = 40, 13, 100
    ld = 112
    en = torch.zeros(B * N, ld, device="cuda"); em = torch.zeros(B * N, ld, device="cuda")
    en[:, :W] = _selu_out((B * N, W), 2.0); em[:, :W] = _selu_out((B * N, W), 1.0)
    mask = torch.rand(B, N) < 0.6
    mask[0] = False; mask[1] = False; mask[2] = True
    ptr = torch.zeros(B * N + 1, dtype=torch.int32)
    ptr[1:] = mask.view(-1).int().cumsum(0).int()
    ptr = ptr.cuda()
    g = torch.empty(B, ld, device="cuda"); att = torch.empty(B * N, ld, device="cuda")
    _ok(L.lib.gib_graph_gather(_p(g), _p(att), _p(en), _p(em), ld, _p(ptr), N, B, 1e6, _st()), "gather")
    dg = torch.randn(B, ld, device="cuda")
    Gen = torch.full((B * N, ld), NAN, device="cuda"); Gem = torch.full((B * N, ld), NAN, device="cuda")
    _ok(L.lib.gib_test_graph_gather_bwd(_p(Gen), _p(Gem), _p(dg), _p(att), _p(en), _p(em), ld, N, B, _st()), "bwd")
    a = att.double().view(B, N, ld)
    e, m, d = en.double().view(B, N, ld), em.double().view(B, N, ld), dg.double()[:, None, :]
    dot = (a * d * m).sum(1, keepdim=True)
    ref_en = a * (d * m - dot) * _dselu64(e)
    ref_em = a * d * _dselu64(m)
    mag = a * d.abs() * (m.abs() + (a * m.abs()).sum(1, keepdim=True))
    _within(Gen.view(B, N, ld), ref_en, mag * _dselu64(e).abs(), "Gen", mag * DACT)
    _within(Gem.view(B, N, ld), ref_em, (a * d.abs() * _dselu64(m).abs()), "Gem", a * d.abs() * DACT)


# ----------------------------------------------------------------------------------------------------------------------
# EMN line-graph aggregation
# ----------------------------------------------------------------------------------------------------------------------
def _csr_from_entries(ent_dst, ent_src, S):
    """the K0 arrays of a bond-entry list ordered by (dst, src): dst_ptr, src_ptr, src_ent (ordered (src, dst))"""
    E = ent_dst.numel()
    dst_ptr = torch.zeros(S + 1, dtype=torch.int32)
    dst_ptr[1:] = torch.bincount(ent_dst, minlength=S).cumsum(0)
    src_ptr = torch.zeros(S + 1, dtype=torch.int32)
    src_ptr[1:] = torch.bincount(ent_src, minlength=S).cumsum(0)
    src_ent = torch.argsort(ent_src * (S + 1) + ent_dst, stable=True).int()
    assert E == 0 or bool((ent_dst[1:] >= ent_dst[:-1]).all())
    return dst_ptr, src_ptr, src_ent


def _line_graph(ent_dst, ent_src):
    """the oracle's rule (oracle/mpnn_oracle.py, emn_forward): receiver r = (i, j) hears every s = (j, k), k != i"""
    E = ent_dst.numel()
    same = ent_dst[None, :] == ent_src[:, None]                 # [r, s]: s leaves j = src of r
    keep = same & (ent_src[None, :] != ent_dst[:, None])        # ... and k != i
    r, s = keep.nonzero(as_tuple=True)
    return r, s


def _hub_graph():
    """atoms: 0 bonded to 1..300 (degree 300), 301 to 302..341 (degree 40), the pair 342-343 (degree 1), a self loop
    on 344, 345..349 isolated (degree 0), a few bonds among 1..300; entries in both directions, ordered (dst, src)"""
    und = [(0, k) for k in range(1, 301)] + [(301, k) for k in range(302, 342)] + [(342, 343)]
    und += [(k, k + 1) for k in range(1, 300, 37)]
    pairs = set()
    for a, b in und:
        pairs.add((a, b)); pairs.add((b, a))
    pairs.add((344, 344))
    ent = torch.tensor(sorted(pairs), dtype=torch.long)
    return ent[:, 0].contiguous(), ent[:, 1].contiguous(), 350


def _k0_graph():
    """the EMN entries K0 builds from a real batch with a degree-5 atom and a self loop"""
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
    arrays = [g.array(d, k, n) for k, n in ((1, E), (0, E), (3, S + 1), (5, S + 1), (6, E))]
    ent_dst, ent_src = arrays[0].long().cpu(), arrays[1].long().cpu()
    assert bool(((ent_dst == ent_src)).any())
    assert int(torch.bincount(ent_src).max()) >= 5
    return ent_dst, ent_src, S, arrays, g


def _emn_ref(EMx, ENx, EMm, ENm, r, s, E, dmsg):
    """fp64 autograd of msg[r] = softmax-weighted mean of {(ENx[r], EMx[r])} U {(ENm[s], EMm[s])}; magnitudes"""
    xs = [t.double().requires_grad_(True) for t in (EMx, ENx, EMm, ENm)]
    emx, enx, emm, enm = xs
    ld = EMx.shape[1]
    idx = r[:, None].expand(-1, ld)
    mx = enx.detach().clone().scatter_reduce(0, idx, enm.detach()[s], "amax")
    es = torch.exp(enx - mx)
    ep = torch.exp(enm[s] - mx[r])
    den = es + torch.zeros_like(es).index_add(0, r, ep)
    num = es * emx + torch.zeros_like(es).index_add(0, r, ep * emm[s])
    msg = num / den
    grads = torch.autograd.grad(msg, xs, dmsg.double())
    R = enx.detach().abs().scatter_reduce(0, idx, enm.detach().abs()[s], "amax")
    V = emx.detach().abs().scatter_reduce(0, idx, emm.detach().abs()[s], "amax")
    mag_r = (1 + R) * V * dmsg.double().abs() + dmsg.double().abs()
    mag_s = torch.zeros_like(mag_r).index_add(0, s, mag_r[r])
    return msg.detach(), grads, mag_r, mag_s


def _emn_run(ent_dst, ent_src, S, live_n=None, cap_pad=0, arrays=None, seed=0, scale=45.0):
    L = _lib()
    torch.manual_seed(seed)
    E = ent_dst.numel()
    rows = E + cap_pad
    ld = 48
    if arrays is None:
        dst_ptr, src_ptr, src_ent = _csr_from_entries(ent_dst, ent_src, S)
        pad = torch.full((cap_pad,), -1, dtype=torch.long)
        arrays = [torch.cat([ent_dst, pad]).int().cuda(), torch.cat([ent_src, pad]).int().cuda(), dst_ptr.cuda(),
                  src_ptr.cuda(), src_ent.cuda()]
    dd, ds, dp, sp, se = arrays
    n = E if live_n is None else live_n

    def buf(scale_):
        t = _selu_out((rows, ld), scale_)
        t[n:] = NAN                                   # pad rows / rows past the live count: never read
        return t
    EMx, ENx, EMm, ENm = buf(1.0), buf(scale), buf(1.0), buf(scale)
    dmsg = torch.randn(rows, ld, device="cuda")
    dmsg[n:] = NAN
    live = torch.tensor([n], dtype=torch.int32, device="cuda") if (live_n is not None or cap_pad) else None
    msg = torch.full((rows, ld), 7.0, device="cuda")
    _ok(L.lib.gib_test_emn_aggregate_fwd(_p(msg), _p(EMx), _p(ENx), _p(EMm), _p(ENm), ld, _p(dd), _p(ds), _p(dp),
                                         rows if live is not None else E, _p(live), _st()), "emn fwd")
    dEMx, dENx = torch.randn(rows, ld, device="cuda"), torch.randn(rows, ld, device="cuda")   # accumulated into
    x0 = (dEMx.clone(), dENx.clone())
    dEMm, dENm = torch.full((rows, ld), NAN, device="cuda"), torch.full((rows, ld), 7.0, device="cuda")
    m0 = (dEMm.clone(), dENm.clone())
    st3 = torch.full((3 * rows * ld,), NAN, device="cuda")
    _ok(L.lib.gib_test_emn_aggregate_bwd(_p(dEMx), _p(dENx), _p(dEMm), _p(dENm), _p(st3), _p(dmsg), _p(EMx), _p(ENx),
                                         _p(EMm), _p(ENm), ld, _p(dd), _p(ds), _p(dp), _p(sp), _p(se),
                                         rows if live is not None else E, _p(live), _st()), "emn bwd")
    r, s = _line_graph(ent_dst.cuda()[:n], ent_src.cuda()[:n])
    ref, (gemx, genx, gemm, genm), mag_r, mag_s = _emn_ref(EMx[:n], ENx[:n], EMm[:n], ENm[:n], r, s, n, dmsg[:n])
    _within(msg[:n], ref, mag_r, "msg")
    _within(dEMx[:n], x0[0][:n].double() + gemx, x0[0][:n].double().abs() + mag_r, "dEMx")
    _within(dENx[:n], x0[1][:n].double() + genx, x0[1][:n].double().abs() + mag_r, "dENx")
    _within(dEMm[:n], gemm, mag_s, "dEMm")
    _within(dENm[:n], genm, mag_s, "dENm")
    for t, t0, name in ((msg, torch.full_like(msg, 7.0), "msg"), (dEMx, x0[0], "dEMx"), (dENx, x0[1], "dENx"),
                        (dEMm, m0[0], "dEMm"), (dENm, m0[1], "dENm")):
        _same_bits(t[n:], t0[n:], name + " rows past the live count")
    return r, s


@pytest.mark.parametrize("scale", [1.0, 45.0])
def test_emn_aggregate_hub_graph(scale):
    """degrees 0, 1, 40, 300 and a self loop; energies up to |100| at scale 45"""
    ent_dst, ent_src, S = _hub_graph()
    r, s = _emn_run(ent_dst, ent_src, S, scale=scale)
    assert r.numel() > 80000                          # the 300-bond hub: 300 receivers x 299 senders


def test_emn_aggregate_live_count_and_nan_pad_rows():
    """capacity mode: a live count that cuts the batch between two molecules (the hub and the 40-star) inside buffers
    with NaN pad rows past it; rows >= live stay untouched"""
    ent_dst, ent_src, S = _hub_graph()
    n = int((ent_dst < 301).sum())
    r, s = _line_graph(ent_dst[:n], ent_src[:n])
    r2, s2 = _line_graph(ent_dst, ent_src)
    assert r.numel() == int((r2 < n).sum()) and bool((s2[r2 < n] < n).all())   # no sender past the cut
    _emn_run(ent_dst, ent_src, S, live_n=n, cap_pad=100)
    _emn_run(ent_dst, ent_src, S, live_n=0, cap_pad=100, seed=1)


def test_emn_aggregate_k0_graph():
    """the CSRs K0 builds for the EMN from a real batch (degree-5 atom, self loop)"""
    ent_dst, ent_src, S, arrays, g = _k0_graph()
    _emn_run(ent_dst, ent_src, S, arrays=arrays)
