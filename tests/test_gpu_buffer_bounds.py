"""GPU: memory discipline of the C-ABI.  Every caller-supplied buffer sits inside a guarded allocation
(tests/guarded.py): the buffers the contract lets hold garbage are filled with 0xFF bytes (NaN as float32, -1 as int32),
and after each call sequence both guard bands must be untouched.

  a. K0 against its numpy restatement (tests/k0_reference.py), every byte of the count workspace and the graph buffer,
     across batch sizes, bond-type counts, the supported-dims edge N^2 * groups = 32768, bond values, int8 input and
     capacity mode with its truncation rule;
  b. the whole training step (K0, packing, forward, loss, backward whole and in two parts, Adam) on poisoned buffers
     is bit-identical to the same step on zero-filled buffers, in exact mode and in a capacity that fits; a batch that
     overflows its capacity writes nothing out of bounds and its surviving molecules keep their logits;
  c. generation rounds whose output capacity is smaller than the molecules a round finishes;
  d. gib_adam_step against fp64 Adam with a grid-stride loop that iterates, every start modulo 16 bytes, grad_scale != 1.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.guarded import MIB, Guarded
from tests.k0_reference import FLAG_OVERFLOW, k0_reference

pytestmark = pytest.mark.gpu


def _lib():
    from graphinvent_b200._lib import check, lib
    return lib, check


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _vp(g):
    return ctypes.c_void_p(g.ptr())


def _assert_intact(bufs, what=""):
    bad = {name: g.damage() for name, g in bufs.items() if not g.intact()}
    assert not bad, f"{what}: writes into guard bands (first / last byte offset from the interior): {bad}"


# ---------------------------------------------------------------------------------------------------------------------
# a. K0 against the numpy reference
# ---------------------------------------------------------------------------------------------------------------------
def _k0_dims(B, N, Ef, by_type, in_dtype):
    from graphinvent_b200._lib import Dims
    d = Dims()
    d.model = 0 if by_type else 3            # GIB_GGNN (typed groups) / GIB_EMN (one group)
    d.B, d.N, d.Ef, d.in_dtype = B, N, Ef, in_dtype
    return d


def run_k0(edges, by_type, capacity=None, graph_bytes_delta=0):
    """K0 through the C-ABI on guarded buffers (count workspace and graph buffer poisoned).  Returns the host header,
    the guarded buffers and the graph-array addresses relative to the graph buffer."""
    lib, check = _lib()
    B, N, _, Ef = edges.shape
    d = _k0_dims(B, N, Ef, by_type, 1 if edges.dtype == np.int8 else 0)
    bd = ctypes.byref(d)
    e = Guarded.like(torch.from_numpy(np.ascontiguousarray(edges)))
    cws = Guarded(lib.gib_graph_count_ws_bytes(bd))
    check(lib.gib_graph_count(bd, _vp(e), _vp(cws), _st()), "gib_graph_count")
    hdr = np.zeros(16, np.int32)
    if capacity is None:
        hdr[:] = cws.view(torch.int32)[:16].cpu().numpy()
    else:
        check(lib.gib_graph_header_capacity(bd, int(capacity), _vp(cws), hdr.ctypes.data_as(ctypes.c_void_p)),
              "gib_graph_header_capacity")
    hp = hdr.ctypes.data_as(ctypes.c_void_p)
    nbytes = lib.gib_graph_bytes(bd, hp)
    gbuf = Guarded(nbytes + graph_bytes_delta)
    check(lib.gib_graph_fill(bd, _vp(e), _vp(cws), hp, _vp(gbuf), _st()), "gib_graph_fill")
    torch.cuda.synchronize()
    arrays = [lib.gib_graph_array(bd, hp, _vp(gbuf), w) - gbuf.ptr() for w in range(7)]
    return dict(hdr=hdr, edges=e, cws=cws, gbuf=gbuf, nbytes=nbytes, arrays=arrays)


def check_k0(edges, by_type, capacity=None):
    """every byte of both buffers equals the reference (bytes no kernel writes keep the poison), both bands intact"""
    ref = k0_reference(edges, by_type, capacity)
    got = run_k0(edges, by_type, capacity)
    _assert_intact({k: got[k] for k in ("edges", "cws", "gbuf")}, "K0")
    what = f"B={ref.B} N={ref.N} Ef={ref.Ef} {'typed' if by_type else 'EMN'} {edges.dtype} capacity={capacity}"
    if capacity is None:
        assert np.array_equal(got["hdr"], ref.hdr), (what, got["hdr"], ref.hdr)
    cws = got["cws"].view(torch.int32).cpu().numpy()
    assert np.array_equal(cws[:16], ref.hdr), (what, cws[:16], ref.hdr)
    assert np.array_equal(cws, ref.expected_cws), what
    assert got["nbytes"] == ref.expected_buf.size * 4, what
    lay = ref.layout
    assert got["arrays"] == [4 * lay[k] for k in ("ent_src", "ent_dst", "ent_w", "dst_ptr", "dst_ent", "src_ptr",
                                                  "src_ent")], what
    buf = got["gbuf"].view(torch.int32).cpu().numpy()
    if not np.array_equal(buf, ref.expected_buf):
        first = int(np.flatnonzero(buf != ref.expected_buf)[0])
        name = max((k for k in lay if lay[k] <= first), key=lambda k: lay[k])
        raise AssertionError(f"{what}: graph buffer differs first at int {first} ({name}[{first - lay[name]}]): "
                             f"{buf[first]} vs {ref.expected_buf[first]}")
    return ref


def _random_bonds(rng, B, N, Ef, p=0.12, multi=0.02):
    e = np.zeros((B, N, N, Ef), np.float32)
    b, i, j = np.nonzero(rng.random((B, N, N)) < p)
    e[b, i, j, rng.integers(0, Ef, b.size)] = 1.0
    b, i, j = np.nonzero(rng.random((B, N, N)) < multi)          # a second type on some cells
    e[b, i, j, rng.integers(0, Ef, b.size)] = 1.0
    return e


def _content(kind, B, N, Ef, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return _random_bonds(rng, B, N, Ef)
    if kind == "empty":
        return np.zeros((B, N, N, Ef), np.float32)
    if kind == "complete":                  # every cell and every type, self-loops included
        return np.ones((B, N, N, Ef), np.float32)
    if kind == "last_cell":
        e = np.zeros((B, N, N, Ef), np.float32)
        e[B - 1, N - 1, N - 1, Ef - 1] = 1.0
        return e
    e = _random_bonds(rng, B, N, Ef, p=0.3)
    vals = {"float_values": [0.5, 2.0, -0.0, np.nan, 1.0], "int8_values": [-128.0, -1.0, 2.0, 127.0, 1.0]}[kind]
    nz = np.nonzero(e)
    e[nz] = rng.choice(np.array(vals, np.float32), nz[0].size)
    return e


def _int8_copy(e):
    """the int8 copy of a float batch when it has one (integer values in range; -0.0 and 0 are both "no bond")"""
    if np.isnan(e).any() or (np.abs(e) > 128).any() or (e != np.round(e)).any() or (e >= 128).any():
        return None
    return e.astype(np.int8)


K0_CASES = (
    [("random", B, 13, 3) for B in (1, 1024, 1025, 4097)]
    + [("random", 300, 13, Ef) for Ef in (1, 2, 4)]
    + [("random", 1025, N, 3) for N in (1, 2)]
    + [("random", 65, 90, 4), ("random", 65, 128, 2), ("last_cell", 4097, 13, 3)]
    + [(c, 5, 13, 3) for c in ("empty", "complete", "last_cell", "float_values", "int8_values")]
    + [("complete", 2, 90, 4), ("complete", 2, 128, 2), ("complete", 3, 2, 4), ("complete", 3, 1, 1)]
)


@pytest.mark.parametrize("by_type", [True, False], ids=["typed", "EMN"])
@pytest.mark.parametrize("kind,B,N,Ef", K0_CASES, ids=[f"{c}-B{B}-N{N}-Ef{Ef}" for c, B, N, Ef in K0_CASES])
def test_k0_matches_reference(kind, B, N, Ef, by_type):
    e = _content(kind, B, N, Ef, seed=B * 131 + N * 7 + Ef)
    ref = check_k0(e, by_type)
    i8 = _int8_copy(e)
    if i8 is not None:                       # the int8 copy of the batch gives the same bytes
        ref8 = check_k0(i8, by_type)
        assert np.array_equal(ref8.expected_buf, ref.expected_buf)
    if kind == "complete":
        assert ref.E == B * N * N * (Ef if by_type else 1)


@pytest.mark.parametrize("B,kind", [(2, "complete"), (65, "random")])
def test_k0_emn_grouping_at_181_nodes(B, kind):
    """N = 181: 32761 cells, the largest N the one-group (EMN) layout supports with any Ef"""
    e = _content(kind, B, 181, 4, seed=181 + B)
    check_k0(e, by_type=False)
    check_k0(e[..., :1].copy(), by_type=True)          # typed with Ef = 1: the same cell count


def _capacities(ref):
    """E + 1, E, E - 1, a cut inside the second type group, a cut inside the first, and 1"""
    G, E = ref.G, ref.E
    caps = {"E+1": E + 1, "E": E, "E-1": E - 1, "1": 1}
    tc0, tc1 = int(ref.type_count[0]), int(ref.type_count[1]) if G > 1 else 0
    if G > 1 and tc1 > 300:
        x = int(ref.type_base[1]) + tc1 // 2 - 128 * G
        caps["inside_group1"] = x // 128 * 128
    caps["inside_group0"] = max(1, tc0 // 2 - 128 * G)
    return caps


@pytest.mark.parametrize("by_type", [True, False], ids=["typed", "EMN"])
@pytest.mark.parametrize("kind,B,N,Ef", [("random", 1025, 13, 3), ("random", 300, 13, 4), ("complete", 2, 128, 2),
                                         ("int8_values", 40, 13, 3)])
def test_k0_capacity_mode_truncates_inside_the_buffers(kind, B, N, Ef, by_type):
    e = _content(kind, B, N, Ef, seed=B + N + Ef)
    full = k0_reference(e, by_type)
    for name, cap in _capacities(full).items():
        ref = check_k0(e, by_type, capacity=cap)
        assert ref.overflow == (full.E > cap), name
        hdr = ref.hdr
        assert bool(hdr[11] & FLAG_OVERFLOW) == (full.E > cap), name
        if name == "inside_group1":
            assert full.type_base[1] < ref.cap_P < full.type_base[1] + full.type_count[1], name
        if name == "inside_group0":
            assert ref.cap_P < full.type_count[0], name
        i8 = _int8_copy(e)
        if i8 is not None and name in ("E-1", "inside_group0"):
            check_k0(i8, by_type, capacity=cap)


def test_the_band_check_sees_a_short_graph_buffer():
    """a graph buffer one 128-row tile (512 bytes) shorter than gib_graph_bytes asks for: K0 writes into the band"""
    e = _content("random", 300, 13, 3, seed=1)
    got = run_k0(e, True, graph_bytes_delta=-512)
    assert got["cws"].intact() and got["edges"].intact()
    assert not got["gbuf"].intact()
    lo, hi = got["gbuf"].damage()
    assert got["gbuf"].n <= lo and hi < got["nbytes"], (lo, hi, got["nbytes"])


# ---------------------------------------------------------------------------------------------------------------------
# b. the whole training step through the C-ABI
# ---------------------------------------------------------------------------------------------------------------------
STEP_MODELS = ["small_GGNN", "small_MNN", "small_AttGGNN", "small_EMN", "row_A", "row_G", "row_I"]


def _model_case(name):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    if name.startswith("small_"):
        from tests.conftest import load_small
        fx = load_small(name[len("small_"):])
        C, sd, nodes, edges, target = fx["C"], fx["sd"], fx["nodes"], fx["edges"], fx["target"]
    else:
        from tests.test_gpu_model_dims import _batch
        C, nodes, edges, target = _batch(name[len("row_"):])
        sd = O.init_state_dict(C, seed=0)
    net = mpnn.create(C)
    net.load_state_dict(sd)
    net = net.cuda()
    return C, net, nodes.cuda(), edges.cuda(), target.float().cuda()


def run_step(net, nodes, edges, target, capacity, fill, parts=False, grad_fill="zero", ws_delta=0):
    """K0 -> header -> fill -> pack -> forward -> KL loss -> backward (whole, or part 1 then 2) -> Adam, every buffer
    guarded.  fill: "poison" or "zero" for the buffers the contract lets hold garbage; the gradient bucket (accumulated
    into) and the Adam moments are zeroed unless grad_fill says otherwise.  int8 nodes / edges run as an int8 batch."""
    from graphinvent_b200 import functional as Fn
    lib, check = _lib()
    B = nodes.shape[0]
    d = Fn.make_dims(net, B, Fn.input_dtype_code(nodes, edges))
    bd, st = ctypes.byref(d), _st()
    params = [p.detach() for p in net.parameters()]
    total = sum(p.numel() for p in params)
    apd = target.shape[1]
    guard = max(4 * MIB, 128 * 4 * apd)      # more than one 128-row tile of the widest activation of these models
    g = {}
    g["nodes"], g["edges"], g["target"] = (Guarded.like(t, guard=guard) for t in (nodes, edges, target))
    g["params"] = Guarded.like(torch.cat([p.flatten() for p in params]), guard=guard)
    pflat = g["params"].view()
    views, o = [], 0
    for p in params:
        views.append(pflat[o:o + p.numel()].view(p.shape))
        o += p.numel()
    g["cws"] = Guarded(lib.gib_graph_count_ws_bytes(bd), fill=fill, guard=guard)
    check(lib.gib_graph_count(bd, _vp(g["edges"]), _vp(g["cws"]), st), "gib_graph_count")
    hdr = np.zeros(16, np.int32)
    if capacity is None:
        hdr[:] = g["cws"].view(torch.int32)[:16].cpu().numpy()
    else:
        check(lib.gib_graph_header_capacity(bd, int(capacity), _vp(g["cws"]), hdr.ctypes.data_as(ctypes.c_void_p)),
              "gib_graph_header_capacity")
    hp = hdr.ctypes.data_as(ctypes.c_void_p)
    g["graph"] = Guarded(lib.gib_graph_bytes(bd, hp), fill=fill, guard=guard)
    check(lib.gib_graph_fill(bd, _vp(g["edges"]), _vp(g["cws"]), hp, _vp(g["graph"]), st), "gib_graph_fill")
    g["packed"] = Guarded(lib.gib_model_packed_bytes(bd), fill=fill, guard=guard)
    check(lib.gib_model_pack(bd, Fn._ptr_table(views), _vp(g["packed"]), st), "gib_model_pack")
    ws_bytes = lib.gib_model_workspace_bytes(bd, hp)
    assert ws_bytes > 0
    g["ws"] = Guarded(ws_bytes + ws_delta, fill=fill, guard=max(guard, ws_bytes))
    g["out"] = Guarded(B * apd * 4, fill=fill, guard=guard)
    check(lib.gib_model_forward(bd, hp, _vp(g["nodes"]), _vp(g["edges"]), _vp(g["graph"]), _vp(g["packed"]),
                                _vp(g["ws"]), _vp(g["out"]), st), "gib_model_forward")
    g["rows"] = Guarded(B * 4, fill=fill, guard=guard)
    g["dout"] = Guarded(B * apd * 4, fill=fill, guard=guard)
    check(lib.gib_kl_loss_fwd_bwd(_vp(g["out"]), _vp(g["target"]), B, apd, 1.0 / B, _vp(g["rows"]), _vp(g["dout"]),
                                  st), "gib_kl_loss_fwd_bwd")
    g["loss"] = Guarded(4, fill=fill, guard=guard)
    check(lib.gib_sum_scaled(_vp(g["rows"]), B, 1.0 / B, _vp(g["loss"]), st), "gib_sum_scaled")
    g["grads"] = Guarded(total * 4, fill=grad_fill, guard=guard)
    gflat = g["grads"].view(torch.float32)
    gviews, o = [], 0
    for p in params:
        gviews.append(gflat[o:o + p.numel()])
        o += p.numel()
    g["scratch"] = Guarded(lib.gib_model_bwd_scratch_bytes(bd, hp), fill=fill, guard=guard)
    args = (bd, hp, _vp(g["nodes"]), _vp(g["edges"]), _vp(g["graph"]), _vp(g["packed"]), _vp(g["ws"]), _vp(g["out"]),
            _vp(g["dout"]), Fn._ptr_table(gviews), _vp(g["scratch"]))
    if parts:
        check(lib.gib_model_backward_part(*args, 1, st), "gib_model_backward_part(1)")
        check(lib.gib_model_backward_part(*args, 2, st), "gib_model_backward_part(2)")
    else:
        check(lib.gib_model_backward(*args, st), "gib_model_backward")
    g["exp_avg"] = Guarded(total * 4, fill="zero", guard=guard)
    g["exp_avg_sq"] = Guarded(total * 4, fill="zero", guard=guard)
    check(lib.gib_adam_step(_vp(g["params"]), _vp(g["grads"]), _vp(g["exp_avg"]), _vp(g["exp_avg_sq"]), total, 1,
                            1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0, st), "gib_adam_step")
    torch.cuda.synchronize()
    return dict(g=g, hdr=hdr, out=g["out"].view(torch.float32).view(B, apd).clone(),
                loss=g["loss"].view(torch.float32).clone(), grads=gflat.clone(),
                params=g["params"].view().clone(), flags=int(g["cws"].view(torch.int32)[11]))


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _overflow_capacity(edges, by_type, E):
    """an overflowing capacity that keeps some molecules whole and truncates others"""
    e = edges.cpu().numpy()
    for cap in (int(E * 0.8), int(E * 0.9), E - 1):
        r = k0_reference(e, by_type, cap)
        if 0 < cap < E and r.survivors.any() and not r.survivors.all():
            return cap, r.survivors
    raise AssertionError("no overflowing capacity with survivors")


@pytest.mark.parametrize("name", STEP_MODELS)
def test_training_step_reads_only_what_it_wrote(name):
    C, net, nodes, edges, target = _model_case(name)
    by_type = C.model != "EMN"
    exact = run_step(net, nodes, edges, target, None, "zero")
    E = int(exact["hdr"][0])
    modes = {"exact": None, "fit": int(E * 1.3) + 64}
    results = {}
    for mode, cap in modes.items():
        ref = exact if cap is None else run_step(net, nodes, edges, target, cap, "zero")
        _assert_intact(ref["g"], f"{name} {mode} zero-filled")
        assert ref["flags"] & FLAG_OVERFLOW == 0
        assert torch.isfinite(ref["out"]).all() and torch.isfinite(ref["grads"]).all()
        for parts in (False, True):
            got = run_step(net, nodes, edges, target, cap, "poison", parts=parts)
            what = f"{name} {mode} poisoned, backward {'in two parts' if parts else 'whole'}"
            _assert_intact(got["g"], what)
            assert _bits_equal(got["out"], ref["out"]), what
            assert _bits_equal(got["loss"], ref["loss"]), what
            assert _bits_equal(got["grads"], ref["grads"]), what
            assert _bits_equal(got["params"], ref["params"]), what
        results[mode] = ref
    # an overflowing batch: truncated inside its buffers, and the molecules whose bonds all fit keep their logits
    cap, survivors = _overflow_capacity(edges, by_type, E)
    keep = torch.from_numpy(survivors).cuda()
    for fill in ("zero", "poison"):
        got = run_step(net, nodes, edges, target, cap, fill)
        what = f"{name} overflow (capacity {cap} < {E} entries, {int(survivors.sum())} of {len(survivors)} survive)"
        _assert_intact(got["g"], f"{what}, {fill}")
        assert got["flags"] & FLAG_OVERFLOW
        # same kernels, same tiles as the capacity that fits: the surviving rows agree to the last bit
        assert _bits_equal(got["out"][keep], results["fit"]["out"][keep]), what


def test_the_band_check_sees_a_short_forward_workspace():
    """a forward workspace of half the bytes gib_model_workspace_bytes asks for: the forward writes into the band"""
    C, net, nodes, edges, target = _model_case("small_GGNN")
    exact = run_step(net, nodes, edges, target, None, "zero")
    ws_bytes = exact["g"]["ws"].n
    got = run_step(net, nodes, edges, target, None, "poison", ws_delta=-(ws_bytes // 2))
    assert not got["g"]["ws"].intact()
    lo, hi = got["g"]["ws"].damage()
    assert lo >= got["g"]["ws"].n and hi < ws_bytes, (lo, hi, ws_bytes)


def test_a_read_of_poisoned_bytes_shows_in_the_results():
    """the gradient bucket is accumulated into: poisoned, every gradient and every updated parameter is NaN"""
    C, net, nodes, edges, target = _model_case("small_GGNN")
    ref = run_step(net, nodes, edges, target, None, "zero")
    got = run_step(net, nodes, edges, target, None, "poison", grad_fill="poison")
    _assert_intact(got["g"], "poisoned gradient bucket")
    assert _bits_equal(got["out"], ref["out"])                  # the forward does not read it
    assert torch.isnan(got["grads"]).all() and torch.isnan(got["params"]).all()
    assert torch.isfinite(ref["grads"]).all() and torch.isfinite(ref["params"]).all()


# ---------------------------------------------------------------------------------------------------------------------
# c. generation rounds with an output capacity smaller than what a round finishes
# ---------------------------------------------------------------------------------------------------------------------
class _GenBuffers:
    """the generator's state and output buffers, guarded; state as GraphGenerator._allocate leaves it, outputs and
    scratch poisoned, properly_terminated and the counters zeroed (the kernels only ever set its flags to 1)"""

    def __init__(self, B, N, F, Ef, cap):
        lib, _ = _lib()
        z = dict(fill="zero")
        self.nodes, self.edges = Guarded(B * N * F * 4, **z), Guarded(B * N * N * Ef * 4, **z)
        self.n_nodes, self.likelihoods = Guarded(B * 4, **z), Guarded(B * 2 * N * 4, **z)
        self.gen_nodes, self.gen_edges = Guarded(cap * N * F * 4), Guarded(cap * N * N * Ef * 4)
        self.gen_n_nodes, self.gen_lik = Guarded(cap), Guarded(cap * 2 * N * 4)
        self.proper, self.counters = Guarded(cap, **z), Guarded(8, **z)
        self.scratch = Guarded(lib.gib_generation_scratch_bytes(B))
        self.action, self.lik = Guarded(B * 4), Guarded(B * 4)
        self.shape = (B, N, F, Ef, cap)
        self.nodes.view(torch.float32)[: N * F].fill_(1.0)          # the dummy graph in slot 0
        self.edges.view(torch.float32)[0].fill_(1.0)
        self.n_nodes.view(torch.int32)[0].fill_(1)

    def all(self):
        return {k: v for k, v in vars(self).items() if isinstance(v, Guarded)}

    def outputs(self, cap):
        B, N, F, Ef, _ = self.shape
        f = torch.float32
        return (self.gen_nodes.view(f).view(cap, N, F)[:cap].cpu().numpy(),
                self.gen_edges.view(f).view(cap, N, N, Ef)[:cap].cpu().numpy(),
                self.gen_n_nodes.view(torch.int8)[:cap].cpu().numpy(),
                self.gen_lik.view(f).view(cap, 2 * N)[:cap].cpu().numpy(),
                self.proper.view(torch.int8)[:cap].cpu().numpy())

    def assert_state(self, st, what):
        B, N, F, Ef, _ = self.shape
        f = torch.float32
        assert int(self.counters.view(torch.int32)[0]) == st.n_generated, what
        assert (self.nodes.view(f).view(B, N, F).cpu().numpy() == st.nodes).all(), what
        assert (self.edges.view(f).view(B, N, N, Ef).cpu().numpy() == st.edges).all(), what
        assert (self.n_nodes.view(torch.int32).cpu().numpy() == st.n_nodes).all(), what
        assert (self.likelihoods.view(f).view(B, 2 * N).cpu().numpy() == st.likelihoods).all(), what

    def ptrs(self):
        return (_vp(self.nodes), _vp(self.edges), _vp(self.n_nodes), _vp(self.likelihoods), _vp(self.gen_nodes),
                _vp(self.gen_edges), _vp(self.gen_n_nodes), _vp(self.gen_lik), _vp(self.proper))


def _oracle_state(B, N, A, CH, Ef, H, C, cap):
    from tests import generation_layout_oracle as L
    st = L.LayoutState(B, N, A, CH, Ef, H, C)
    for k in ("generated_nodes", "generated_edges", "generated_n_nodes", "generated_likelihoods",
              "properly_terminated"):
        setattr(st, k, getattr(st, k)[:cap].copy())               # the oracle's `p < cap` rule at this capacity
    return st


def _assert_outputs(gb, st, cap, rows=None):
    """the first `rows` output rows (default: all `cap`, every one of them written) equal the oracle's"""
    rows = cap if rows is None else rows
    got = gb.outputs(cap)
    want = (st.generated_nodes, st.generated_edges, st.generated_n_nodes, st.generated_likelihoods,
            st.properly_terminated)
    for name, a, b in zip(("nodes", "edges", "n_nodes", "likelihoods", "properly_terminated"), got, want):
        assert (a[:rows] == b[:rows]).all(), name


@pytest.mark.parametrize("seed,H,C", [(0, 0, 0), (1, 4, 3)], ids=["L0", "L3"])
def test_generation_rounds_stay_inside_a_small_output_capacity(seed, H, C):
    from tests import generation_layout_oracle as L
    from tests.test_gpu_generation_layouts import _layout_stream
    lib, check = _lib()
    B, N, A, CH, Ef, cap = 200, 13, 5, 3, 3, 16
    F = A + CH + H + C
    rng = np.random.default_rng(seed)
    gb = _GenBuffers(B, N, F, Ef, cap)
    st = _oracle_state(B, N, A, CH, Ef, H, C, cap)
    for rnd in range(2 * N - 1):
        a, _ = _layout_stream(rng, st)
        lk = rng.random(B).astype(np.float32)
        gb.action.view(torch.int32).copy_(torch.from_numpy(a))
        gb.lik.view(torch.float32).copy_(torch.from_numpy(lk))
        written = L.generation_round(st, rnd, a, lk)
        check(lib.gib_generation_round_layout(B, N, F, Ef, A, CH, H, C, rnd, _vp(gb.action), _vp(gb.lik), *gb.ptrs(),
                                              cap, _vp(gb.counters), _vp(gb.scratch), _st()),
              "gib_generation_round_layout")
        gb.assert_state(st, rnd)
        assert int(gb.counters.view(torch.int32)[1]) == written, rnd
    torch.cuda.synchronize()
    assert st.n_generated > 2 * cap          # rounds past the capacity took the -2 ("would overflow") path
    _assert_outputs(gb, st, cap)
    _assert_intact(gb.all(), "generation rounds")


def test_out_of_range_actions_terminate_once_as_invalid():
    """an action index outside the APD (a corrupted replay trace) terminates its slot as invalid and edits nothing: it
    is counted once, among the invalid slots, so the finished graphs fill the output rows without a gap.  The oracle
    gets a connect to atom N - 1 in its place, which is invalid in every state and also edits nothing."""
    from tests import generation_layout_oracle as L
    from tests.test_gpu_generation_layouts import _layout_stream
    lib, check = _lib()
    B, N, A, CH, Ef = 200, 13, 5, 3, 3
    F, cap = A + CH, 2 * B
    rng = np.random.default_rng(11)
    gb = _GenBuffers(B, N, F, Ef, cap)
    st = _oracle_state(B, N, A, CH, Ef, 0, 0, cap)
    bad_total = 0
    for rnd in range(2 * N - 1):
        if st.n_generated > B:           # a round writes at most B - 1 graphs: stay inside the 2B output rows
            break
        a, len_add = _layout_stream(rng, st)
        apd = len_add + N * Ef + 1
        bad = np.zeros(B, bool)
        bad[1:] = rng.random(B - 1) < 0.05
        bad_total += int(bad.sum())
        a_dev = np.where(bad, rng.choice(np.array([-1, apd, apd + 7, 2 ** 31 - 1], np.int64), B), a).astype(np.int32)
        a_oracle = np.where(bad, len_add + (N - 1) * Ef, a).astype(np.int32)
        lk = rng.random(B).astype(np.float32)
        gb.action.view(torch.int32).copy_(torch.from_numpy(a_dev))
        gb.lik.view(torch.float32).copy_(torch.from_numpy(lk))
        written = L.generation_round(st, rnd, a_oracle, lk)
        check(lib.gib_generation_round_layout(B, N, F, Ef, A, CH, 0, 0, rnd, _vp(gb.action), _vp(gb.lik), *gb.ptrs(),
                                              cap, _vp(gb.counters), _vp(gb.scratch), _st()),
              "gib_generation_round_layout")
        gb.assert_state(st, rnd)
        assert int(gb.counters.view(torch.int32)[1]) == written, rnd
    torch.cuda.synchronize()
    assert bad_total > 50 and st.n_generated > B // 2
    _assert_outputs(gb, st, cap, rows=st.n_generated)
    _assert_intact(gb.all(), "out-of-range actions")


def test_sampled_generation_rounds_stay_inside_a_small_output_capacity():
    from tests import generation_layout_oracle as L
    lib, check = _lib()
    B, N, A, CH, Ef, H, C, cap = 300, 9, 4, 3, 3, 2, 0, 24
    F = A + CH + H + C
    apd = N * A * CH * H * Ef + N * Ef + 1
    gen = torch.Generator(device="cuda").manual_seed(5)
    logits = Guarded.like(torch.randn(B, apd, device="cuda", generator=gen) * 3)
    uniforms = Guarded.like(torch.rand(2 * N, B, device="cuda", generator=gen))
    state = Guarded(8, fill="zero")
    gb = _GenBuffers(B, N, F, Ef, cap)
    st = _oracle_state(B, N, A, CH, Ef, H, C, cap)
    runs = 0
    for call in range(2 * N + 1):
        s0 = state.view(torch.int32).cpu().numpy().copy()
        inert = st.n_generated >= B or s0[1] != 0
        check(lib.gib_generation_sample_round(B, N, F, Ef, A, CH, H, C, _vp(logits), apd, _vp(uniforms), _vp(state),
                                              _vp(gb.action), _vp(gb.lik), *gb.ptrs(), cap, _vp(gb.counters),
                                              _vp(gb.scratch), _st()), "gib_generation_sample_round")
        s1 = state.view(torch.int32).cpu().numpy()
        if inert:
            assert (s1 == s0).all(), call
        else:
            runs += 1
            assert s1[0] == s0[0] + 1, call
            a = gb.action.view(torch.int32).cpu().numpy()
            lk = gb.lik.view(torch.float32).cpu().numpy()
            L.generation_round(st, int(s0[0]), a, lk)
        gb.assert_state(st, call)
    torch.cuda.synchronize()
    assert runs >= 1 and st.n_generated >= B > cap
    _assert_outputs(gb, st, cap)
    _assert_intact({**gb.all(), "logits": logits, "uniforms": uniforms, "state": state}, "sampled rounds")


# ---------------------------------------------------------------------------------------------------------------------
# d. gib_adam_step at the edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0, 4, 8, 12])
@pytest.mark.parametrize("grad_scale,wd", [(1.0, 0.0), (0.5, 0.01), (1.0 / 3.0, 0.0)])
def test_adam_step_matches_fp64(offset, grad_scale, wd):
    lib, check = _lib()
    # one wave is 6 CTAs x 256 threads per SM, 4 floats a thread: three passes of the grid-stride loop and a ragged tail
    n = lib.gib_device_sm_count() * 6 * 256 * 4 * 3 + 13
    gen = torch.Generator(device="cuda").manual_seed(offset + 7)
    init = {"p": torch.randn(n, device="cuda", generator=gen),
            "g": torch.randn(n, device="cuda", generator=gen) * 1e-2,
            "m": torch.randn(n, device="cuda", generator=gen) * 1e-3,
            "v": torch.rand(n, device="cuda", generator=gen) * 1e-4}
    bufs = {}
    for k, t in init.items():
        bufs[k] = Guarded(n * 4 + offset, fill="poison")
        bufs[k].view(torch.uint8)[offset:].view(torch.float32).copy_(t)
    view = {k: b.t[offset:].view(torch.float32) for k, b in bufs.items()}
    step, lr, b1, b2, eps = 5, 1e-3, 0.9, 0.999, 1e-8
    check(lib.gib_adam_step(*(ctypes.c_void_p(view[k].data_ptr()) for k in "pgmv"), n, step, lr, b1, b2, eps, wd,
                            grad_scale, _st()), "gib_adam_step")
    torch.cuda.synchronize()
    _assert_intact(bufs, f"adam offset {offset}")
    assert (bufs["p"].t[:offset] == 0xFF).all() and (bufs["g"].t[:offset] == 0xFF).all()
    # fp64 Adam (torch.optim.Adam, non-amsgrad, L2 weight decay), bias corrections as the host evaluates them
    p, g, m, v = (init[k].double() for k in "pgmv")
    g = g * grad_scale + wd * p
    m = m + (g - m) * (1 - b1)
    v = v * b2 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    upd = (lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + eps)
    p = p - upd
    # bounds: a few float32 roundings of each operand's magnitude (sums can cancel, so every quantity is bounded through
    # the magnitudes of its terms rather than through itself)
    u = 2.0 ** -24
    denom = v.sqrt() / bc2 ** 0.5 + eps
    gscale = init["g"].double().abs() * grad_scale + wd * init["p"].double().abs()     # g * scale + wd * p can cancel
    mscale = init["m"].double().abs() + gscale
    scales = {"m": mscale, "v": init["v"].double() + gscale * gscale, "p": p.abs() + (lr / bc1) * mscale / denom}
    for k, want in (("m", m), ("v", v), ("p", p)):
        err = (view[k].double() - want).abs()
        assert bool((err <= 16 * u * scales[k]).all()), (k, float((err / scales[k]).max() / u))
    assert float(upd.abs().mean()) > 1e-5              # the step moved the parameters
