"""GPU: the GGNN / MNN message-row path (one message-MLP row per molecule, source atom and bond type, and one per bond
entry whose value is not 1) against fp64, on the shapes one-hot molecules never produce.

  a. seg_reduce_dact -- K2's segmented sum with the fused row_w * act'(Y) epilogue, the backward of the message rows --
     on its own through gib_test_seg_reduce_dact, against fp64 autograd of out[dst] += w_row * act(pre_row): row
     degrees on both sides of every 4-entry trip boundary up to 300, act 0 / 1 / 2, row_w absent or in {0.5, 1, 2, -3},
     ld 16 to 704, row counts that are no multiple of the block; pad rows (empty segments) come back as exact 0 without
     reading their NaN Y; the four K2 variants agree bit for bit;
  b. both models through _fp64_anchored (tests/test_gpu_parity.py) on seeded batches built here, each with the
     generator's corner graphs: hubs (stars at N = 13, 40, 90 and complete graphs at N = 40: shared rows of up to 89
     entries), value-1 and other values in one (source, type), no sharing at all, unit bonds only, multi-type cells with
     a bond type absent from the batch -- in exact mode with tensor cores on and off, in capacity mode and on the
     per-entry path (gib_tc_debug bit 3); the message-row and per-entry logits are bit-identical on them; an int8 batch
     with values 2, -1, 127, -128 equals its float copy bit for bit; a capacity cut inside a hub's shared row keeps the
     table equal to its restatement, writes no guard band and leaves the surviving molecules' logits unchanged;
  c. the rows the message MLPs ran on, from the profiling records of one forward: on the device-count branch the
     forward GEMM work of the per-entry path minus that of the message rows is exactly T * sum_t (P_t - U_t) * sum_l w_l
     (P_t entries and U_t message rows of type t, w_l the work per row model.cu charges for message-MLP layer l); on the
     host-range branch (tensor cores off) the two are equal and every launch is a SIMT class.
"""
import contextlib
import ctypes
import functools

import numpy as np
import pytest
import torch

from tests.test_gpu_buffer_bounds import _assert_intact, _bits_equal, run_step
from tests.test_gpu_graph_kernels import DACT, EPS, NAN, _dselu64, _lib, _ok, _p, _same_bits, _st, _within
from tests.test_gpu_message_rows import _mode, _table_of
from tests.test_gpu_parity import _fp64_anchored
from tests.test_model_dims_host import SMALL

pytestmark = pytest.mark.gpu

MODELS = ["GGNN", "MNN"]
WORST = {}          # what -> worst error / bound of the kernel checks


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for what, r in sorted(WORST.items()):
        print(f"\nworst error / bound: {r:.3g} ({what})")


# ----------------------------------------------------------------------------------------------------------------------
# a. seg_reduce_dact against fp64
# ----------------------------------------------------------------------------------------------------------------------
# K2 reads 4 entries per trip: a row of degree 4k ends a trip exactly, 4k + 1 needs one more
TRIP_DEGS = [0, 1, 3, 4, 5, 8, 9, 40, 300]
ROW_W = (0.5, 1.0, 2.0, -3.0)
N_DST = 500
TAIL = 3


def _row_degrees(kind):
    g = torch.Generator().manual_seed(7)
    if kind == "trip degrees":              # every degree three times, shuffled: 27 rows + 1 empty
        degs = torch.tensor(TRIP_DEGS * 3)[torch.randperm(27, generator=g)].tolist() + [0]
    else:                                   # 1237 rows (odd: the 2-slot variants' last thread has no second slot)
        degs = torch.tensor([0, 1, 2, 3, 4, 5, 8, 9])[torch.randint(0, 8, (1237,), generator=g)].tolist()
        degs[611] = 40
    return degs


def _row_csr(degs, seed):
    """message rows -> destination CSR: row u owns the entries [ptr[u], ptr[u+1]), entry q names destination ent[q]"""
    g = torch.Generator().manual_seed(seed)
    d = torch.tensor(degs)
    ptr = torch.zeros(len(degs) + 1, dtype=torch.int32)
    ptr[1:] = d.cumsum(0)
    E = int(d.sum())
    ent = torch.randint(0, N_DST, (E,), generator=g, dtype=torch.int32)
    row = torch.repeat_interleave(torch.arange(len(degs)), d)
    return ptr.cuda(), ent.cuda(), row.cuda()


def _check(got, ref, mag, slack, what):
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (ref.abs() + mag + 1e-300)).max().item() if err.numel() else 0.0
    WORST["seg_reduce_dact"] = max(WORST.get("seg_reduce_dact", 0.0), ratio / EPS)
    _within(got, ref, mag, what, slack)


@pytest.mark.parametrize("ld", [16, 112, 704])
@pytest.mark.parametrize("wmode", ["none", "0.5/1/2/-3"])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_seg_reduce_dact_matches_fp64(act, wmode, ld):
    """G[u] = row_w[u] act'(Y[u]) sum_q dM[ent[q]]: fp64 autograd of out[ent[q]] += row_w[u] act(pre[u]) w.r.t. pre,
    evaluated through the fp32 Y as the kernel does; bound as in test_scatter_bwd with the magnitude of the sum's terms"""
    L = _lib().lib
    torch.manual_seed(100 * act + ld + (wmode != "none"))
    try:
        for kind in ("trip degrees", "1237 rows"):
            degs = _row_degrees(kind)
            rows = len(degs)
            ptr, ent, row = _row_csr(degs, seed=ld)
            empty = (ptr[1:] == ptr[:-1])
            pre = torch.randn(rows, ld, device="cuda", dtype=torch.float64) * 2
            Y = {0: pre, 1: torch.selu(pre), 2: torch.tanh(pre)}[act].float()
            Y[empty] = NAN                                  # pad rows: the kernel must not read them
            w = (torch.tensor(ROW_W, device="cuda")[torch.randint(0, len(ROW_W), (rows,), device="cuda")]
                 if wmode != "none" else None)
            dM = torch.randn(N_DST, ld, device="cuda")
            ww = w.double() if w is not None else torch.ones(rows, device="cuda", dtype=torch.float64)
            y64 = torch.where(empty[:, None], 0.0, Y.double()).requires_grad_(True)
            out = torch.zeros(N_DST, ld, dtype=torch.float64, device="cuda").index_add(
                0, ent.long(), (y64 * ww[:, None])[row])
            (gy,) = torch.autograd.grad(out, y64, dM.double())
            terms = torch.zeros(rows, ld, dtype=torch.float64, device="cuda").index_add(
                0, row, dM.double().abs()[ent.long()]) * ww.abs()[:, None]
            dact = {0: torch.ones_like(y64), 1: _dselu64(y64), 2: 1 - y64 * y64}[act].detach()
            ref, live = gy * dact, ~empty
            first = None
            for variant in (0, 1, 2, 3):
                what = f"seg_reduce_dact {kind} act={act} w={wmode} ld={ld} variant {variant}"
                L.gib_scatter_variant(variant)
                G = torch.full((rows + TAIL, ld), NAN, device="cuda")
                G[rows:] = 7.0
                _ok(L.gib_test_seg_reduce_dact(_p(G), _p(dM), _p(Y), ld, _p(ptr), _p(ent), _p(w), act, rows, _st()),
                    what)
                if first is None:
                    _check(G[:rows][live], ref[live], (terms * dact.abs())[live], (gy.abs() * DACT)[live], what)
                    assert (G[:rows][empty].view(torch.int32) == 0).all(), what + ": pad rows are not +0"
                    assert (G[rows:] == 7.0).all(), what + ": rows past the row count written"
                    first = G
                else:
                    _same_bits(G, first, what + " vs variant 0")
    finally:
        L.gib_scatter_variant(2)         # the library's default, which every other caller expects


# ----------------------------------------------------------------------------------------------------------------------
# b. batches that stress the message-row table
# ----------------------------------------------------------------------------------------------------------------------
def _constants(model, N, Ef):
    from graphinvent_b200.config import layout_dims
    from oracle import mpnn_oracle as O
    return O.make_constants(model, max_n_nodes=N, **layout_dims(5, 3, Ef), **SMALL)


def _molecule(N, Ef, n_atoms, rng):
    """n_atoms atoms (random type, neutral charge) and no bonds yet"""
    nodes = np.zeros((1, N, 8), np.float32)
    nodes[0, np.arange(n_atoms), rng.integers(0, 5, n_atoms)] = 1
    nodes[0, :n_atoms, 6] = 1
    return nodes, np.zeros((1, N, N, Ef), np.float32)


def _star(N, Ef, centre, types, rng):
    """the centre bonded to every other atom; bond k has type types[k % len(types)]"""
    n, e = _molecule(N, Ef, N, rng)
    for k, j in enumerate(j for j in range(N) if j != centre):
        t = types[k % len(types)]
        e[0, centre, j, t] = e[0, j, centre, t] = 1
    return n, e


def _complete(N, Ef, rng, types=None):
    """every pair bonded, a random type per bond (or `types`)"""
    n, e = _molecule(N, Ef, N, rng)
    for i in range(N):
        for j in range(i + 1, N):
            t = int(rng.integers(0, Ef)) if types is None else types
            e[0, i, j, t] = e[0, j, i, t] = 1
    return n, e


def _revalue(e, values, rng, p=1.0):
    """each bond (both directions alike) takes a value drawn from `values` with probability p; then no atom's values
    cancel (_keep_atoms_bonded)"""
    for b, i, j, t in zip(*np.nonzero(e)):
        if i <= j and rng.random() < p:
            e[b, i, j, t] = e[b, j, i, t] = rng.choice(values)
    return _keep_atoms_bonded(e)


def _cancelling_atoms(e):
    """atoms with bonds whose values sum to 0.  The reference decides whether an atom is bonded -- whether the GRU
    updates it and the readout sees it -- from that sum (summation_mpnn.py:109, 146: adjacency.sum(-1) != 0), K0 from
    its non-zero entries: the two agree unless negative values cancel"""
    return np.argwhere((e != 0).any((2, 3)) & (e.sum((2, 3)) == 0))


def _keep_atoms_bonded(e):
    """re-value one bond of every cancelling atom, so that neither of its two atoms cancels afterwards"""
    while len(bad := _cancelling_atoms(e)):
        b, i = bad[0]
        j, t = np.argwhere(e[b, i] != 0)[0]
        rest_i, rest_j = e[b, i].sum() - e[b, i, j, t], e[b, j].sum() - e[b, j, i, t]
        v = next(v for v in (2.0, 4.0, 3.0) if rest_i + v != 0 and rest_j + v != 0)
        e[b, i, j, t] = e[b, j, i, t] = v
    return e


def _stack(N, Ef, n_random, extra, seed):
    """the generator's corner graphs, n_random seeded random molecules, then `extra` (list of (nodes, edges))"""
    from graphinvent_b200 import synthetic as S
    n2, e2 = S.corner_case_graphs(N, 8, Ef)
    n, e = S.random_graphs(n_random, N, 5, 3, n_edge_features=Ef, seed=seed, min_atoms=0)
    nodes = np.concatenate([n2, n] + [x[0] for x in extra]).astype(np.float32)
    edges = np.concatenate([e2, e] + [x[1] for x in extra]).astype(np.float32)
    return nodes, edges


def _batch_hubs13(rng):
    return 13, 3, _stack(13, 3, 40, [_star(13, 3, 0, [0], rng), _star(13, 3, 6, [1], rng), _star(13, 3, 12, [2], rng)],
                         seed=31)


def _batch_hubs40(rng):
    return 40, 3, _stack(40, 3, 4, [_star(40, 3, 0, [0], rng), _star(40, 3, 20, [2], rng), _complete(40, 3, rng)],
                         seed=32)


def _batch_hubs90(rng):
    return 90, 4, _stack(90, 4, 1, [_star(90, 4, 0, [0], rng), _star(90, 4, 45, [3], rng)], seed=33)


def _batch_mixed_values(rng):
    """hubs whose bonds of one type carry 1 and 0.5 / 2 / -3: one shared row, then the rows of their own"""
    extra = []
    for centre, t in ((0, 0), (5, 1), (12, 2)):
        n, e = _star(13, 3, centre, [t], rng)
        vals = [1.0, 0.5, 1.0, 2.0, 1.0, -3.0, 1.0, 1.0, 0.5, 2.0, -3.0, 1.0]
        for k, j in enumerate(j for j in range(13) if j != centre):
            e[0, centre, j, t] = e[0, j, centre, t] = vals[k]
        extra.append((n, e))
    nodes, edges = _stack(13, 3, 40, extra, seed=34)
    _revalue(edges[5:45], [0.5, 2.0, -3.0], rng, p=0.3)
    return 13, 3, (nodes, edges)


def _batch_no_sharing(rng):
    nodes, edges = _stack(13, 3, 40, [_star(13, 3, 3, [0, 1], rng)], seed=35)
    return 13, 3, (nodes, _revalue(edges, [0.5, 2.0, -3.0], rng))


def _batch_unit(rng):
    return 13, 3, _stack(13, 3, 40, [_star(13, 3, 0, [0], rng), _complete(13, 3, rng)], seed=36)


def _batch_multitype_absent(rng):
    """bond type 1 occurs nowhere (a zero device count in a grouped launch); some cells carry types 0 and 2 at once"""
    nodes, edges = _stack(13, 3, 40, [_star(13, 3, 4, [0, 2], rng)], seed=37)
    edges[..., 0] += edges[..., 1]
    edges[..., 1] = 0
    for b, i, j in zip(*np.nonzero(edges.sum(-1))):
        if i < j and rng.random() < 0.25:
            edges[b, i, j, :] = edges[b, j, i, :] = (1, 0, 1)
    edges[-1, 4, :, 0] = edges[-1, :, 4, 0] = 1            # the star's centre: every bond of both types
    edges[-1, 4, 4, 0] = 0
    return 13, 3, (nodes, edges)


def _batch_int8_values(rng):
    nodes, edges = _stack(13, 3, 40, [_star(13, 3, 0, [0], rng)], seed=38)
    return 13, 3, (nodes, _revalue(edges, [1.0, 2.0, -1.0, 127.0, -128.0], rng))


BATCHES = {"hubs13": _batch_hubs13, "hubs40": _batch_hubs40, "hubs90": _batch_hubs90,
           "mixed_values": _batch_mixed_values, "no_sharing": _batch_no_sharing, "unit": _batch_unit,
           "multitype_absent": _batch_multitype_absent, "int8_values": _batch_int8_values}


@functools.lru_cache(maxsize=None)
def _case(name, model):
    """constants, state dict and the batch (CPU float32 tensors) of one case"""
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    from oracle import mpnn_oracle as O
    rng = np.random.default_rng(sum(map(ord, name)))
    N, Ef, (nodes, edges) = BATCHES[name](rng)
    C = _constants(model, N, Ef)
    target = torch.from_numpy(S.random_targets(nodes.shape[0], apd_length(C), seed=4))
    return C, O.init_state_dict(C, seed=1), torch.from_numpy(nodes), torch.from_numpy(edges), target


def _net(C, sd, capacity=None):
    from graphinvent_b200.gnn import mpnn
    net = mpnn.create(C)
    net.load_state_dict(sd)
    net.entry_capacity = capacity
    return net.cuda()


def test_the_batches_have_the_shapes_they_are_meant_to():
    """the properties the cases exist for, checked on K0's header and the bond tensor"""
    for name in BATCHES:
        C, _, nodes, edges, _ = _case(name, "GGNN")
        v = edges[edges != 0]
        assert (edges.sum(-1) != 0).sum((1, 2))[:3].tolist() == [1, 0, 0], name     # dummy self loop, empty, isolated
        assert len(_cancelling_atoms(edges.numpy())) == 0, name
        if name.startswith("hubs"):
            assert int((edges != 0).sum((2, 3)).max()) == C.max_n_nodes - 1, name
        if name == "no_sharing":
            assert (v != 1).all()
        if name == "unit":
            assert (v == 1).all()
        if name == "mixed_values":
            assert {0.5, 1.0, 2.0, -3.0} <= set(v.tolist())
        if name == "multitype_absent":
            assert int(edges[..., 1].abs().sum()) == 0 and int(((edges != 0).sum(-1) > 1).sum()) > 0
        if name == "int8_values":
            assert {2.0, -1.0, 127.0, -128.0} <= set(v.tolist())


@contextlib.contextmanager
def _oracle_once():
    """the fp32 / fp64 / kink-probe oracle runs of _fp64_anchored, computed once for the configurations of one case"""
    from oracle import mpnn_oracle as O
    real, memo = O.train_step_grads, {}

    def cached(sd, C, nodes, edges, target, dtype=None):
        key = (dtype, O.KINK)
        if key not in memo:
            memo[key] = real(sd, C, nodes, edges, target, dtype=dtype)
        return memo[key]

    O.train_step_grads = cached
    try:
        yield
    finally:
        O.train_step_grads = real


@contextlib.contextmanager
def _created_with_capacity(capacity):
    """the models _fp64_anchored builds run in capacity mode"""
    from graphinvent_b200.gnn import mpnn
    create = mpnn.create

    def create_in_capacity_mode(c):
        net = create(c)
        net.entry_capacity = capacity
        return net

    mpnn.create = create_in_capacity_mode
    try:
        yield
    finally:
        mpnn.create = create


# name -> (tensor cores, gib_tc_debug, capacity mode)
CONFIGS = {"exact, tensor cores": (1, 0, False), "exact, fp32 SIMT": (0, 0, False),
           "capacity mode": (1, 0, True), "per-entry path": (1, 8, False)}


# With tensor cores off, three cases exceed _fp64_anchored's gradient bound (GEMM_EPS 1e-6 x |g| with the fp32 SIMT
# kernels), measured on an H100 80GB HBM3: GGNN hubs40 by 1.13x (msg_nns.1.seq.3.bias) and MNN hubs90 by 1.94x
# (gru.weight_ih) on the message rows and on the per-entry path alike (1.12x / 1.92x) -- the fp32 sums over a hub's 39 /
# 89 bonds carry more rounding than the reference's own fp32 evaluation -- and GGNN mixed_values by 1.002x
# (msg_nns.0.seq.0.weight: 1.589e-3 against a kink band of 1.586e-3).  They run in test_fp32_simt_exceeds_the_bound.
SIMT_OVER_BOUND = [("hubs40", "GGNN", 0), ("hubs40", "GGNN", 8), ("hubs90", "MNN", 0), ("hubs90", "MNN", 8),
                   ("mixed_values", "GGNN", 0)]
# The int8 case's values 127 and -128 scale the GGNN message MLP's input and output by up to 128 each: the 3xTF32
# arithmetic then moves a logit 1.3e-3 past the logit bound, which has no GEMM term (the per-entry path's logits are the
# same to the bit, test_message_row_logits_equal_the_per_entry_path).  It runs against fp64 with tensor cores off only.
TC_OVER_BOUND = [("int8_values", "GGNN")]


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("case", list(BATCHES))
def test_fp64_anchored_on_message_row_batches(case, model):
    from graphinvent_b200._lib import lib
    C, sd, nodes, edges, target = _case(case, model)
    entries = int((edges != 0).sum())
    with _oracle_once():
        for config, (tc, debug, cap) in CONFIGS.items():
            if (tc == 0 and (case, model, 0) in SIMT_OVER_BOUND) or (tc == 1 and (case, model) in TC_OVER_BOUND):
                continue
            lib.gib_tc_debug(debug)
            try:
                with _created_with_capacity(entries + 64 if cap else None):
                    _fp64_anchored(C, sd, nodes, edges, target, f"{model} {case}, {config}", tc)
            finally:
                lib.gib_tc_debug(0)


@pytest.mark.xfail(strict=True, raises=AssertionError, reason="fp32 SIMT sums exceed GEMM_EPS[0] (SIMT_OVER_BOUND)")
@pytest.mark.parametrize("case,model,debug", SIMT_OVER_BOUND)
def test_fp32_simt_exceeds_the_bound(case, model, debug):
    """strict: the day one of these passes, it belongs in test_fp64_anchored_on_message_row_batches"""
    from graphinvent_b200._lib import lib
    C, sd, nodes, edges, target = _case(case, model)
    lib.gib_tc_debug(debug)
    try:
        _fp64_anchored(C, sd, nodes, edges, target, f"{model} {case}, exact, fp32 SIMT, gib_tc_debug {debug}", 0)
    finally:
        lib.gib_tc_debug(0)


def _logits(net, nodes, edges):
    with torch.no_grad():
        out = net(nodes.cuda(), edges.cuda())
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("case", list(BATCHES))
def test_message_row_logits_equal_the_per_entry_path(case, model):
    """the forward of the message rows computes every message row from that row alone and sums the same values in
    the same order as the per-entry path: bit-identical logits, tensor cores on and off, exact and capacity mode"""
    C, sd, nodes, edges, _ = _case(case, model)
    cap = int((edges != 0).sum()) + 64
    for tc, capacity in ((True, None), (False, None), (True, cap)):
        outs = []
        for debug in (0, 8):
            with _mode(debug, tc):
                outs.append(_logits(_net(C, sd, capacity), nodes, edges))
        what = f"{model} {case} tensor cores {tc} capacity {capacity}"
        assert torch.isfinite(outs[0]).all(), what
        assert _bits_equal(outs[0], outs[1]), what


@pytest.mark.parametrize("model", MODELS)
def test_int8_batch_equals_its_float_copy(model):
    """bond values 2, -1, 127 and -128 read from int8 by K0 and the first-layer kernels: logits, loss and gradients
    are those of the same batch in float32, bit for bit"""
    from graphinvent_b200 import functional as Fn
    C, sd, nodes, edges, target = _case("int8_values", model)
    cap = int((edges != 0).sum()) + 64
    for capacity in (None, cap):
        res = []
        for dt in (torch.float32, torch.int8):
            net = _net(C, sd, capacity)
            out = net(nodes.to(dt).cuda(), edges.to(dt).cuda())
            loss = Fn.kl_loss(out, target.cuda())
            loss.backward()
            torch.cuda.synchronize()
            res.append((out.detach(), loss.detach(), torch.cat([p.grad.flatten() for p in net.parameters()])))
        what = f"{model} int8 capacity {capacity}"
        assert torch.isfinite(res[0][0]).all(), what
        for a, b in zip(*res):
            assert _bits_equal(a.float().contiguous(), b.float().contiguous()), what


@pytest.mark.parametrize("cut", ["star", "complete"])
@pytest.mark.parametrize("model", MODELS)
def test_capacity_cut_inside_a_shared_row(model, cut):
    """a capacity that ends inside the entries of a hub's shared row: the table still equals its restatement, no
    guard band is written, and the molecules that survive keep the logits of a capacity that fits, bit for bit"""
    from tests.k0_reference import FLAG_OVERFLOW, k0_reference
    rng = np.random.default_rng(41)
    N = 40
    nodes, edges = _stack(N, 3, 4, [_complete(N, 3, rng, types=0), _star(N, 3, 0, [0], rng)], seed=42)
    C = _constants(model, N, 3)
    from oracle import mpnn_oracle as O
    net = _net(C, O.init_state_dict(C, seed=1))
    B = nodes.shape[0]
    full = k0_reference(edges, True)
    m = B - 1 if cut == "star" else B - 2                 # the molecule the cut falls in
    off = int(np.concatenate([[0], np.cumsum((edges != 0).sum((1, 2, 3)))])[m])
    # star (last molecule): its dst-ordered entries are (0, j) j = 1..39, then (i, 0) -- the centre's shared row; the
    # cut keeps 19 of those 39.  Complete graph: half its entries, so every atom's shared row loses some of its own.
    cap = off + (N - 1) + (N - 1) // 2 if cut == "star" else off + N * (N - 1) // 2
    ref = k0_reference(edges, True, cap)
    assert ref.overflow and ref.survivors.any() and not ref.survivors[m:].any(), ref.survivors
    nodes_d, edges_d = torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda()
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    target = torch.from_numpy(S.random_targets(B, apd_length(C), seed=6)).cuda()
    fit = run_step(net, nodes_d, edges_d, target, full.E + 300, "zero")
    got = run_step(net, nodes_d, edges_d, target, cap, "poison")
    what = f"{model} cut inside the {cut} at capacity {cap} of {full.E}"
    _assert_intact(got["g"], what)
    assert got["flags"] & FLAG_OVERFLOW, what
    table, tref = _table_of(got, net, B)
    for k in table:
        assert np.array_equal(table[k], tref[k]), (what, k, np.flatnonzero(table[k] != tref[k])[:8])
    keep = torch.from_numpy(ref.survivors).cuda()
    assert _bits_equal(got["out"][keep], fit["out"][keep]), what


# ----------------------------------------------------------------------------------------------------------------------
# c. the rows the message MLPs ran on
# ----------------------------------------------------------------------------------------------------------------------
PROF_GEMM_NT, PROF_GEMM_NT_SIMT = 0, 3
MR_COUNT = 0


def _forward_records(net, nodes, edges, capacity):
    """one forward through the C-ABI with the per-launch profile on: (kernel classes, work) of its launches, the
    message-row meta ints (gib_model_msg_rows) and the live header"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import check, lib
    B = nodes.shape[0]
    d = Fn.make_dims(net, B, 0)
    bd, st = ctypes.byref(d), _st()
    g = Fn.GraphBatch(d, edges, capacity=capacity)
    packed = Fn.packed_weights(net, d, list(net.parameters()))
    ws = torch.empty(lib.gib_model_workspace_bytes(bd, g.hdr), dtype=torch.uint8, device="cuda")
    out = torch.empty(B, d.N * d.f_add + d.N * d.f_conn + 1, device="cuda")
    torch.cuda.synchronize()
    cap = 4096
    ms, work, cls = (ctypes.c_double * cap)(), (ctypes.c_double * cap)(), (ctypes.c_int * cap)()
    lib.gib_profile_enable(1)
    try:
        check(lib.gib_model_forward(bd, g.hdr, _p(nodes), _p(edges), _p(g.buf), _p(packed), _p(ws), _p(out), st),
              "gib_model_forward")
        torch.cuda.synchronize()
        n = lib.gib_profile_records(ms, work, cls, cap)
    finally:
        lib.gib_profile_enable(0)
    assert 0 < n <= cap
    addr = lib.gib_model_msg_rows(bd, g.hdr, ctypes.c_void_p(ws.data_ptr()), 8)
    o = addr - ws.data_ptr()
    meta = ws[o:o + 64].view(torch.int32).cpu().numpy()
    return list(cls[:n]), list(work[:n]), meta, g.device_header()


def _msg_work_per_row(net, C):
    """sum over the layers of one bond type's message MLP of the per-row work model.cu charges: 2 R C"""
    if C.model == "MNN":
        return 2.0 * net.message_weights.numel() // C.n_edge_features
    return 2.0 * sum(p.numel() for k, p in net.named_parameters() if k.startswith("msg_nns.0.") and k.endswith("weight"))


def _profile_case(name):
    if name.startswith("row_"):
        from oracle import mpnn_oracle as O
        from tests.test_gpu_model_dims import _batch
        C, nodes, edges, _ = _batch(name[len("row_"):])
        return C, O.init_state_dict(C, seed=0), nodes, edges
    model, case = name.split(":")
    C, sd, nodes, edges, _ = _case(case, model)
    return C, sd, nodes, edges


PROFILE_CASES = ["GGNN:hubs40", "MNN:hubs40", "GGNN:mixed_values", "MNN:mixed_values", "GGNN:multitype_absent",
                 "GGNN:unit", "row_A", "row_G"]


@pytest.mark.parametrize("mode", ["exact", "capacity", "exact fp32"])
@pytest.mark.parametrize("name", PROFILE_CASES)
def test_message_mlps_run_on_message_rows(name, mode):
    from graphinvent_b200._lib import HDR_TYPE_COUNT
    C, sd, nodes, edges = _profile_case(name)
    nodes, edges = nodes.float().cuda(), edges.float().cuda()
    capacity = int((edges != 0).sum()) + 64 if mode == "capacity" else None
    tc = mode != "exact fp32"
    net = _net(C, sd, capacity)
    runs = {}
    for debug in (0, 8):
        with _mode(debug, tc):
            runs[debug] = _forward_records(net, nodes, edges, capacity)
    cls0, work0, meta, hdr = runs[0]
    cls8, work8, _, _ = runs[8]
    fwd = (PROF_GEMM_NT, PROF_GEMM_NT_SIMT)
    saved = sum(w for c, w in zip(cls8, work8) if c in fwd) - sum(w for c, w in zip(cls0, work0) if c in fwd)
    G = C.n_edge_features
    P = [int(hdr[HDR_TYPE_COUNT + t]) for t in range(G)]
    U = [int(meta[MR_COUNT + t]) for t in range(G)]
    assert all(0 <= u <= p for u, p in zip(U, P)), (P, U)
    expect = C.message_passes * sum(p - u for p, u in zip(P, U)) * _msg_work_per_row(net, C)
    what = f"{name} {mode}: entries {P}, message rows {U}"
    print(f"\n{what}: per-entry minus message-row forward GEMM work {saved:.6g} (T sum (P_t - U_t) sum w_l = "
          f"{expect:.6g}), launches {len(cls0)} / {len(cls8)}")
    assert sum(P) > sum(U), what + ": no row is shared"
    if tc:           # device-count branch: the message MLPs run on the table's per-type row counts
        assert saved == expect, what
    else:            # host-range branch: the entry groups' ranges, on the SIMT kernels
        assert saved == 0, what
        assert set(cls0) <= {PROF_GEMM_NT_SIMT, 2} and set(cls8) <= {PROF_GEMM_NT_SIMT, 2}, what
