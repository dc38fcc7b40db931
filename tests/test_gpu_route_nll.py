"""GPU: graphed.RouteScorer -- the decoding-route likelihoods of molecules -- against the fp64 restatement
(tests/route_nll_reference.py) for the four models and the four action layouts, against the live reference's
pretrained-GGNN fixture, bit-for-bit invariance over chunk size, batch size and input placement, the probabilities
GraphedGeneratorRL records when it replays the same routes, refusals, guarded buffers, the TF32 / bf16 modes and
parameter changes."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R
from tests.conftest import GOLDEN, MODELS, pretrained_path
from tests.guarded import Guarded

pytestmark = pytest.mark.gpu

GDB13 = dict(n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0)
SEGS = P.segments(5, 3)


def _fixture(n=None):
    z = np.load(os.path.join(GOLDEN, "route_nll_gdb13.npz"))
    return z["nodes"][:n], z["edges"][:n], z


def _net(model, C=None, seed=0):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = C or O.make_constants(model)
    sd = O.init_state_dict(C, seed=seed)
    net = mpnn.create(C)
    net.load_state_dict(sd)
    return net.cuda().eval(), sd, C


def _layout_molecules(layout, M=24, N=13, seed=3):
    from graphinvent_b200 import synthetic as S
    A, Fc, H, X = layout
    nodes, edges = S.random_graphs(M, N, A, Fc, n_edge_features=3, seed=seed, min_atoms=1)
    rng = np.random.default_rng(seed + 1)
    extra = []
    for w in (H, X):
        if w:
            seg = np.zeros((M, N, w), np.int8)
            present = nodes.any(2)
            seg[present, rng.integers(0, w, int(present.sum()))] = 1
            extra.append(seg)
    return np.concatenate([nodes] + extra, axis=2), edges


@pytest.mark.parametrize("model", MODELS)
def test_models_against_fp64(model):
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(40)
    net, sd, C = _net(model)
    out = RouteScorer(net, 128, **GDB13).score(nodes, edges)
    oracle = R.score(sd, C, nodes, edges, SEGS)
    assert torch.equal(out.offsets.cpu(), torch.from_numpy(oracle[1]))
    assert out.likelihoods.dtype == torch.float32 and out.offsets.dtype == torch.int64
    R.assert_within(out.likelihoods, out.nll, out.final, oracle, model)


LAYOUTS = {"gdb13": (5, 3, 0, 0), "imp_H": (5, 3, 4, 0), "chirality": (5, 3, 0, 3), "imp_H+chirality": (4, 3, 4, 3)}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_action_layouts_against_fp64(layout):
    from graphinvent_b200.config import layout_dims
    from graphinvent_b200.graphed import RouteScorer
    from oracle import mpnn_oracle as O
    A, Fc, H, X = LAYOUTS[layout]
    L = layout_dims(A, Fc, 3, ignore_H=not H, use_chirality=bool(X))
    C = O.make_constants("GGNN", n_node_features=L["n_node_features"], len_f_add_per_node=L["len_f_add_per_node"])
    net, sd, C = _net("GGNN", C)
    nodes, edges = _layout_molecules(LAYOUTS[layout])
    out = RouteScorer(net, 64, n_atom_types=A, n_formal_charge=Fc, n_imp_H=L["n_imp_H"],
                      n_chirality=L["n_chirality"]).score(nodes, edges)
    R.assert_within(out.likelihoods, out.nll, out.final, R.score(sd, C, nodes, edges, P.segments(A, Fc, H, X)), layout)


def test_pretrained_ggnn_matches_the_live_reference():
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import RouteScorer
    from oracle import mpnn_oracle as O
    nodes, edges, z = _fixture()
    sd = torch.load(path, map_location="cpu", weights_only=False)
    C = O.make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(sd)
    out = RouteScorer(net.cuda(), 500, **GDB13).score(nodes, edges)
    oracle = R.score(sd, C, nodes, edges, SEGS)
    R.assert_within(out.likelihoods, out.nll, out.final, oracle, "pretrained")
    # the reference's fp32 probabilities and ours are each within the bound of fp64
    ref = torch.from_numpy(z["likelihoods"]).double()
    d = (torch.log(out.likelihoods.cpu().double()) - torch.log(ref)).abs()
    assert (d <= 2 * oracle[4]).all()
    assert np.array_equal(out.offsets.cpu().numpy(), z["offsets"])


def test_outputs_do_not_depend_on_chunk_batch_or_placement():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture()
    net, _, _ = _net("GGNN")
    base = RouteScorer(net, 256, **GDB13).score(nodes, edges)
    S = base.likelihoods.numel()
    assert S == 1517
    runs = [(1, 4096, "host"), (256, 1, "host"), (300, 4096, "device"), (100, 13, "device"), (S, 4096, "host"),
            (2000, 4096, "device"), (1, 5, "device"), (511, 1, "host")]   # 1517 % 256, % 300, % 511: short batches
    for B, chunk, where in runs:
        x = (torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda()) if where == "device" else (nodes, edges)
        got = RouteScorer(net, B, chunk_molecules=chunk, **GDB13).score(*x)
        for a, b, name in zip(got, base, got._fields):
            assert torch.equal(a, b), f"B={B} chunk={chunk} {where}: {name}"


def test_generation_replaying_the_routes_records_the_same_probabilities():
    """GraphedGeneratorRL replays each molecule's build-order actions (molecule j in slots 1 + j, 1 + j + M, ...;
    slot 0 copies slot 1); the molecules it rebuilds equal the input and their per-round agent probabilities equal
    `likelihoods` bit for bit"""
    from graphinvent_b200.graphed import GraphedGeneratorRL, RouteScorer
    nodes, edges, _ = _fixture()
    lengths = edges.reshape(edges.shape[0], -1).astype(np.int64).sum(1) // 2 + 2
    L = int(np.bincount(lengths).argmax())
    pick = np.flatnonzero(lengths == L)[:32]
    nodes, edges = nodes[pick], edges[pick]
    net, _, _ = _net("GGNN")
    out = RouteScorer(net, 64, **GDB13).score(nodes, edges)
    _, _, acts, offsets = R.build_order_states(nodes, edges, SEGS)
    M = len(pick)
    B = 257                     # >= ROUTE_MIN_BATCH: the rollout's forward runs the scorer's GEMM kernels
    actions = np.full((L + 1, B), -1, np.int64)
    for b in range(1, B):
        j = (b - 1) % M
        actions[:L, b] = acts[offsets[j]:offsets[j + 1]]
    actions[:L, 0] = actions[:L, 1]
    gen = GraphedGeneratorRL(net, B, **GDB13)
    with torch.no_grad():
        gen.sample(net, copy.deepcopy(net), actions=torch.from_numpy(actions).to(torch.int32).cuda())
    gn = gen.generated_nodes.cpu().to(torch.int8).numpy()
    ge = gen.generated_edges.cpu().to(torch.int8).numpy()
    lik = gen.generated_agent_likelihoods.detach().cpu()
    proper = gen.properly_terminated.cpu().numpy()
    found = 0
    for j in range(M):
        rows = [g for g in range(gn.shape[0]) if proper[g] and np.array_equal(gn[g], nodes[j])
                and np.array_equal(ge[g], edges[j])]
        assert rows, f"molecule {j} was not rebuilt"
        want = out.likelihoods[offsets[j]:offsets[j + 1]].cpu()
        assert any(torch.equal(lik[g, :L], want) for g in rows), f"molecule {j}: {lik[rows[0], :L]} vs {want}"
        found += 1
    assert found == M


def _bad_sets():
    nodes, edges, _ = _fixture(12)
    cases = {}
    n, e = nodes.copy(), edges.copy()
    n[5, 0, :] = 0
    n[5, 0, 0] = n[5, 0, 1] = 1
    cases["node row"] = (n, e, "not one-hot")
    n, e = nodes.copy(), edges.copy()
    e[5, 0, 1, :] = 0
    e[5, 0, 1, 0] = 1
    e[5, 1, 0, :] = 0
    cases["edges"] = (n, e, "symmetric")
    n, e = nodes.copy(), edges.copy()
    n[5], e[5] = 0, 0
    cases["empty"] = (n, e, "no atoms")
    n, e = nodes.copy(), edges.copy()
    last = P.n_atoms(n[5]) - 1
    e[5, last, :, :] = 0
    e[5, :, last, :] = 0
    cases["disconnected"] = (n, e, "disconnects")
    return cases


@pytest.mark.parametrize("case", ["node row", "edges", "empty", "disconnected"])
def test_invalid_molecules_are_refused_as_preprocess_refuses_them(case):
    from graphinvent_b200 import preprocess
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, why = _bad_sets()[case]
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 32, **GDB13)
    with pytest.raises(ValueError) as ours:
        scorer.score(nodes, edges)
    with pytest.raises(ValueError) as theirs:
        list(preprocess.groups(nodes, edges, 32, 5, 3))
    assert str(ours.value) == str(theirs.value)
    assert "molecule 5" in str(ours.value) and why in str(ours.value)
    assert scorer.replays == 0                    # refused before any state was scored


def test_kernels_stay_inside_their_buffers():
    """plan, fill, probs and reduce on guard-banded buffers whose interiors start poisoned (NaN / -1): the filled
    inputs and actions equal the restatement's states, every likelihood is written and finite, no band changes"""
    from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, check, lib
    nodes, edges, _ = _fixture(30)
    X, E, acts, offsets = R.build_order_states(nodes, edges, SEGS)
    S, M, B, N, Fd, Ef, apd = X.shape[0], nodes.shape[0], 37, 13, 8, 3, 625
    d = PPDims(N=N, F=Fd, Ef=Ef, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=B)
    bd = ctypes.byref(d)
    chunk = 40
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    ws = Guarded(lib.gib_route_plan_ws_bytes(bd, chunk))
    off = Guarded(4 * (M + 1))
    status = Guarded(4 * PP_STATUS_INTS)
    ctl, slots = Guarded(8), Guarded(8 * B)
    on, oe = Guarded(B * N * Fd), Guarded(B * N * N * Ef)
    lik, nll, fin = Guarded(4 * S), Guarded(4 * M), Guarded(4 * M)
    logits = Guarded.like(torch.randn(B, apd, device="cuda", generator=torch.Generator("cuda").manual_seed(1)) * 4)
    bufs = (gn, ge, ws, off, status, ctl, slots, on, oe, lik, nll, fin, logits)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda g: ctypes.c_void_p(g.ptr())
    check(lib.gib_route_plan(bd, p(gn), p(ge), M, chunk, p(ws), p(off), p(status), st), "gib_route_plan")
    sw = status.view(torch.int32, (PP_STATUS_INTS,)).cpu().numpy()
    assert sw[3] == 0 and sw[5] == S and sw[6] == 0
    assert np.array_equal(off.view(torch.int32, (M + 1,)).cpu().numpy(), offsets)
    lg = logits.view().double().cpu()
    for r in range(-(-S // B)):
        check(lib.gib_route_fill(bd, p(gn), p(ge), chunk, p(ws), p(off), p(status), p(ctl), p(slots), p(on), p(oe),
                                 st), "gib_route_fill")
        check(lib.gib_route_probs(B, apd, p(logits), p(slots), p(lik), st), "gib_route_probs")
        check(lib.gib_rl_next_round(ctypes.c_void_p(status.ptr() + 24), st), "gib_rl_next_round")
        sl = slots.view(torch.int32, (2, B)).cpu().numpy()
        live = min(B, S - r * B)
        assert int(ctl.view(torch.int32, (2,))[0]) == live
        dst = sl[1]
        assert (dst[:live] >= 0).all() and (dst[live:] == -1).all() and (sl[0][live:] == -1).all()
        assert np.array_equal(sl[0][:live], acts[dst[:live]])
        xn, xe = on.view(torch.int8, (B, N, Fd)).cpu().numpy(), oe.view(torch.int8, (B, N, N, Ef)).cpu().numpy()
        assert np.array_equal(xn[:live], X[dst[:live]]) and np.array_equal(xe[:live], E[dst[:live]])
        assert not xn[live:].any() and not xe[live:].any()
        got = lik.view(torch.float32, (S,)).cpu().double()[torch.from_numpy(dst[:live]).long()]
        want = torch.softmax(lg[:live], 1).gather(1, torch.from_numpy(sl[0][:live]).long().view(-1, 1)).view(-1)
        assert ((got - want).abs() <= 1e-6 * want + 1e-12).all()
    check(lib.gib_route_reduce(M, p(off), p(lik), p(nll), p(fin), st), "gib_route_reduce")
    pl = lik.view(torch.float32, (S,)).cpu()
    assert torch.isfinite(pl).all() and (pl > 0).all()
    n64, f64 = R.reduce(pl.double(), offsets)
    assert ((nll.view(torch.float32, (M,)).cpu().double() - n64).abs() <= 1e-6 * n64.abs()).all()
    assert ((fin.view(torch.float32, (M,)).cpu().double() - f64).abs() <= 1e-6 * (1 + f64.abs())).all()
    torch.cuda.synchronize()
    for g in bufs:
        assert g.intact(), g.damage()


MODES = {"tf32": (None, 2.0 ** -11), "bf16": (torch.bfloat16, 2.0 ** -8)}


@pytest.mark.parametrize("mode", list(MODES))
def test_reduced_precision_modes_against_fp64(mode):
    """the scorer built in the mode bakes it in; |d log p| stays within twice its logits' own bound in that mode:
    3x the package's eager forward error in the mode plus one operand rounding of the row's size"""
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(24)
    net, sd, C = _net("GGNN")
    dtype, u = MODES[mode]
    X, E, acts, offsets = R.build_order_states(nodes, edges, SEGS)
    p64, l64 = R.probabilities(sd, C, X, E, acts)
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        if dtype is None:
            torch.backends.cuda.matmul.allow_tf32 = True
            scorer = RouteScorer(net, 128, **GDB13)
            with torch.no_grad():
                lm = net(torch.from_numpy(X).float().cuda(), torch.from_numpy(E).float().cuda())
        else:
            with torch.autocast("cuda", dtype=dtype):
                scorer = RouteScorer(net, 128, **GDB13)
                with torch.no_grad():
                    lm = net(torch.from_numpy(X).float().cuda(), torch.from_numpy(E).float().cuda())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert scorer.tf32 == (dtype is None) and scorer.autocast_dtype == dtype
    out = scorer.score(nodes, edges)
    e_mode = (lm.float().cpu().double() - l64).abs().max(1).values
    b = 2 * (3 * e_mode + u * (1 + l64.abs().max(1).values))
    R.assert_within(out.likelihoods, out.nll, out.final, (p64, offsets, *R.reduce(p64, offsets), b), mode)


def test_parameter_changes_between_calls_are_picked_up():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(16)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 64, **GDB13)
    first = scorer.score(nodes, edges)
    assert all(torch.equal(a, b) for a, b in zip(scorer.score(nodes, edges), first))
    with torch.no_grad():
        next(net.parameters()).mul_(1.5)
    second = scorer.score(nodes, edges)
    assert not torch.equal(second.likelihoods, first.likelihoods)
    fresh = RouteScorer(net, 64, **GDB13).score(nodes, edges)
    assert all(torch.equal(a, b) for a, b in zip(second, fresh))


def test_dropout_model_is_scored_like_its_dropout_free_twin():
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import RouteScorer
    from oracle import mpnn_oracle as O
    nodes, edges, _ = _fixture(16)
    net, sd, C = _net("GGNN")
    Cd = O.make_constants("GGNN", dropout_p=0.2)
    twin = mpnn.create(Cd)
    twin.load_state_dict(sd)
    twin = twin.cuda().train()
    a = RouteScorer(net, 64, **GDB13).score(nodes, edges)
    b = RouteScorer(twin, 64, **GDB13).score(nodes, edges)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
