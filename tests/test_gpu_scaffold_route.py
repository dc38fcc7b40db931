"""GPU: conditional route likelihoods p(molecule | scaffold) (graphed.RouteScorer.score(..., scaffold_ids=)) -- against
the fp64 masked-softmax restatement (tests/scaffold_route_reference.py) for the four models and the four action
layouts with and without attachment points, bit for bit against the unconditional scorer and the scaffold generator
replaying the conditional routes, invariance, gradients, refusals, guarded buffers and fine-tuning."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R
from tests import scaffold_route_reference as SR
from tests.conftest import GOLDEN, MODELS
from tests.guarded import Guarded
from tests.test_gpu_route_grad import KINK_TAU, _assert_fp64_anchored, _weights
from tests.test_gpu_route_nll import GDB13, LAYOUTS, SEGS, _fixture, _layout_molecules, _net

pytestmark = pytest.mark.gpu


def _case(nodes, edges, seed=0, whole=()):
    """per molecule m a k in 1..n_atoms (a spread), its prefix as scaffold m, ids = arange(M) with the molecules in
    `whole` scored whole (-1), and the attachment points each decoration uses"""
    rng = np.random.default_rng(seed)
    M = nodes.shape[0]
    ks = np.array([rng.integers(1, P.n_atoms(nodes[m]) + 1) for m in range(M)])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    ids = np.arange(M)
    ids[list(whole)] = -1
    attach = [SR.decoration_points(nodes[m], edges[m], int(ks[m])) for m in range(M)]
    return sn, se, ids, attach


def _scorer(net, B, sn, se, attach, masked, **kw):
    from graphinvent_b200.graphed import RouteScorer
    layout = kw.pop("layout", GDB13)
    return RouteScorer(net, B, scaffolds=(sn, se), attachment=attach if masked else None, **layout, **kw)


@pytest.mark.parametrize("masked", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("model", MODELS)
def test_models_against_fp64(model, masked):
    nodes, edges, _ = _fixture(40)
    sn, se, ids, attach = _case(nodes, edges, whole=(3, 17))
    net, sd, C = _net(model)
    out = _scorer(net, 128, sn, se, attach, masked).score(nodes, edges, scaffold_ids=ids)
    protect = SR.protect_of(sn, attach) if masked else None
    oracle = SR.score(sd, C, nodes, edges, ids, sn, SEGS, protect)
    assert torch.equal(out.offsets.cpu(), torch.from_numpy(oracle[1]))
    R.assert_within(out.likelihoods, out.nll, out.final, oracle, f"{model} masked={masked}")


@pytest.mark.parametrize("masked", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_action_layouts_against_fp64(layout, masked):
    from graphinvent_b200.config import layout_dims
    from oracle import mpnn_oracle as O
    A, Fc, H, X = LAYOUTS[layout]
    L = layout_dims(A, Fc, 3, ignore_H=not H, use_chirality=bool(X))
    C = O.make_constants("GGNN", n_node_features=L["n_node_features"], len_f_add_per_node=L["len_f_add_per_node"])
    net, sd, C = _net("GGNN", C)
    nodes, edges = _layout_molecules(LAYOUTS[layout])
    sn, se, ids, attach = _case(nodes, edges, seed=1, whole=(2,))
    kw = dict(n_atom_types=A, n_formal_charge=Fc, n_imp_H=L["n_imp_H"], n_chirality=L["n_chirality"])
    out = _scorer(net, 64, sn, se, attach, masked, layout=kw).score(nodes, edges, scaffold_ids=ids)
    protect = SR.protect_of(sn, attach) if masked else None
    R.assert_within(out.likelihoods, out.nll, out.final,
                    SR.score(sd, C, nodes, edges, ids, sn, P.segments(A, Fc, H, X), protect), layout)


def test_consistency_with_the_unconditional_scorer():
    """free scaffolds: each conditional route is the tail of the whole route's likelihoods bit for bit, nll / final
    are gib_route_reduce over that tail, and molecules scored whole (-1) equal the unconditional scores bit for bit"""
    from graphinvent_b200._lib import check, lib
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture()
    sn, se, ids, _ = _case(nodes, edges, seed=2, whole=range(0, 96, 7))
    net, _, _ = _net("GGNN")
    full = RouteScorer(net, 256, **GDB13).score(nodes, edges)
    cond = RouteScorer(net, 256, scaffolds=(sn, se), **GDB13).score(nodes, edges, scaffold_ids=ids)
    fo, co = full.offsets.cpu().numpy(), cond.offsets.cpu().numpy()
    tail = []
    for m in range(nodes.shape[0]):
        n_c = co[m + 1] - co[m]
        if ids[m] < 0:
            assert n_c == fo[m + 1] - fo[m]
            assert torch.equal(full.nll[m], cond.nll[m]) and torch.equal(full.final[m], cond.final[m])
        else:
            assert n_c == SR.n_bonds(edges[m]) - SR.n_bonds(se[m]) + 1
        assert torch.equal(cond.likelihoods[co[m]:co[m + 1]], full.likelihoods[fo[m + 1] - n_c:fo[m + 1]]), m
        tail.append(full.likelihoods[fo[m + 1] - n_c:fo[m + 1]])
    tail = torch.cat(tail)
    off = cond.offsets.to(torch.int32)
    nll, fin = torch.empty_like(cond.nll), torch.empty_like(cond.final)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    check(lib.gib_route_reduce(nodes.shape[0], p(off), p(tail), p(nll), p(fin), st), "gib_route_reduce")
    assert torch.equal(nll, cond.nll) and torch.equal(fin, cond.final)


def test_generation_replaying_the_conditional_routes_records_the_same_probabilities():
    """GraphedGeneratorRL with the same table and attachment points replays each molecule's conditional actions
    (scaffold j in slots 1 + j, 1 + j + M, ...; slot 0 copies slot 1); the molecules it rebuilds equal the input and
    their per-round agent probabilities equal the conditional likelihoods bit for bit"""
    from graphinvent_b200.graphed import GraphedGeneratorRL, RouteScorer
    nodes, edges, _ = _fixture()
    # (molecule, k) pairs whose conditional routes have the most common length L of at least 4 states
    pairs = [(m, k, SR.n_bonds(edges[m]) - SR.n_bonds(SR.prefix(nodes[m], edges[m], k)[1]) + 1)
             for m in range(nodes.shape[0]) for k in range(1, P.n_atoms(nodes[m]) + 1)]
    L = int(np.bincount([c for _, _, c in pairs if c >= 4]).argmax())
    chosen = {}
    for m, k, c in pairs:
        if c == L and m not in chosen:
            chosen[m] = k
    pick = sorted(chosen)[:32]
    nodes, edges = nodes[pick], edges[pick]
    ks = np.array([chosen[m] for m in pick])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    attach = [SR.decoration_points(nodes[j], edges[j], int(ks[j])) for j in range(len(pick))]
    M = len(pick)
    ids = np.arange(M)
    net, _, _ = _net("GGNN")
    out = RouteScorer(net, 64, scaffolds=(sn, se), attachment=attach, **GDB13).score(nodes, edges, scaffold_ids=ids)
    _, _, acts, offsets, _, _ = SR.conditional_states(nodes, edges, ids, sn, SEGS)
    assert np.array_equal(offsets, out.offsets.cpu().numpy()) and (np.diff(offsets) == L).all()
    B = 257
    actions = np.full((L + 1, B), -1, np.int64)
    for b in range(1, B):
        j = (b - 1) % M
        actions[:L, b] = acts[offsets[j]:offsets[j + 1]]
    actions[:L, 0] = actions[:L, 1]
    gen = GraphedGeneratorRL(net, B, scaffolds=(sn, se), attachment=attach, **GDB13)
    with torch.no_grad():
        gen.sample(net, copy.deepcopy(net), actions=torch.from_numpy(actions).to(torch.int32).cuda())
    gn = gen.generated_nodes.cpu().to(torch.int8).numpy()
    ge = gen.generated_edges.cpu().to(torch.int8).numpy()
    gs = gen.generated_scaffolds.cpu().numpy()
    lik = gen.generated_agent_likelihoods.detach().cpu()
    proper = gen.properly_terminated.cpu().numpy()
    for j in range(M):
        rows = [g for g in range(gn.shape[0]) if proper[g] and gs[g] == j and np.array_equal(gn[g], nodes[j])
                and np.array_equal(ge[g], edges[j])]
        assert rows, f"molecule {j} was not rebuilt"
        want = out.likelihoods[offsets[j]:offsets[j + 1]].cpu()
        assert any(torch.equal(lik[g, :L], want) for g in rows), f"molecule {j}: {lik[rows[0], :L]} vs {want}"
        # the generated molecules score as they are: the same ids from generated_scaffolds
    n = 2 * M
    again = RouteScorer(net, 64, scaffolds=(sn, se), attachment=attach, **GDB13).score(
        gen.generated_nodes[:n].to(torch.int8), gen.generated_edges[:n].to(torch.int8),
        scaffold_ids=gen.generated_scaffolds[:n])
    assert torch.isfinite(again.nll).all()


def test_outputs_do_not_depend_on_chunk_batch_or_placement():
    nodes, edges, _ = _fixture()
    sn, se, ids, attach = _case(nodes, edges, seed=3, whole=(1, 50))
    net, _, _ = _net("GGNN")
    base = _scorer(net, 256, sn, se, attach, True).score(nodes, edges, scaffold_ids=ids)
    S = base.likelihoods.numel()
    runs = [(1, 4096, "host", "host"), (300, 13, "device", "device"), (100, 1, "device", "host"),
            (S, 4096, "host", "device"), (511, 7, "host", "host"), (2000, 4096, "device", "device")]
    for B, chunk, where, id_where in runs:
        x = (torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda()) if where == "device" else (nodes, edges)
        i = torch.from_numpy(ids).cuda() if id_where == "device" else ids
        got = _scorer(net, B, sn, se, attach, True, chunk_molecules=chunk).score(*x, scaffold_ids=i)
        for a, b, name in zip(got, base, got._fields):
            assert torch.equal(a, b), f"B={B} chunk={chunk} {where} ids {id_where}: {name}"


# ---- gradients -----------------------------------------------------------------------------------------------------
def _oracle_grads(sd, C, X, E, acts, masks, w_state, dtype, batch=512):
    """gradients of sum_s w_s * -log masked_softmax(forward(state s))[a_s] through mpnn_oracle.forward in `dtype`"""
    from collections import OrderedDict
    from oracle import mpnn_oracle as O
    leaves = OrderedDict((k, v.to(dtype).detach().clone().requires_grad_(True)) for k, v in sd.items())
    total = OrderedDict((k, torch.zeros_like(v)) for k, v in leaves.items())
    for s in range(0, X.shape[0], batch):
        o = O.forward(leaves, C, torch.from_numpy(X[s:s + batch]).to(dtype), torch.from_numpy(E[s:s + batch]).to(dtype))
        o = o.masked_fill(torch.from_numpy(masks[s:s + batch]), float("-inf"))
        a = torch.from_numpy(acts[s:s + batch]).view(-1, 1)
        loss = (w_state[s:s + batch].to(dtype) * -torch.log_softmax(o, 1).gather(1, a).view(-1)).sum()
        for (k, t), g in zip(total.items(), torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)):
            if g is not None:
                t += g.detach()
    return total


@pytest.mark.parametrize("masked", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("model", MODELS)
def test_gradients_against_fp64(model, masked):
    from oracle import mpnn_oracle as O
    nodes, edges, _ = _fixture(40)
    sn, se, ids, attach = _case(nodes, edges, seed=4, whole=(5,))
    net, sd, C = _net(model)
    M = nodes.shape[0]
    w = _weights(M, seed=M)
    scorer = _scorer(net, 128, sn, se, attach, masked)
    out = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
    grads = torch.autograd.grad((w.cuda() * out.nll).sum(), list(net.parameters()))
    protect = SR.protect_of(sn, attach) if masked else None
    X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, SEGS)
    masks = SR.state_masks(sid, n_at, sn, protect, 13, 3, C.len_f_add_per_node)
    assert masks.any() == masked
    w_state = torch.repeat_interleave(w, torch.from_numpy(np.diff(offsets)))
    g = lambda dt: _oracle_grads(sd, C, X, E, acts, masks, w_state, dt)
    g32, g64 = g(torch.float32), g(torch.float64)
    try:
        O.KINK = (KINK_TAU, "L")
        gL = g(torch.float64)
        O.KINK = (KINK_TAU, "R")
        gR = g(torch.float64)
    finally:
        O.KINK = None
    _assert_fp64_anchored(net, grads, (g32, g64, gL, gR), f"{model} masked={masked}")


def test_recomputed_probabilities_several_calls_and_stale_records():
    """the backward's recomputed probabilities equal the forward's bit for bit; two score() calls (conditional and
    whole) wait for one backward and give the sum of their single gradients; set_scaffolds or an in-place parameter
    change between score() and the backward raises"""
    nodes, edges, _ = _fixture(30)
    sn, se, ids, attach = _case(nodes, edges, seed=5, whole=(0,))
    net, _, _ = _net("GGNN")
    scorer = _scorer(net, 64, sn, se, attach, True, chunk_molecules=30)
    out = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
    g1 = torch.autograd.grad(out.nll.sum(), list(net.parameters()))
    assert torch.equal(scorer.lik[:out.likelihoods.numel()], out.likelihoods)
    whole = scorer.score(nodes, edges, requires_grad=True)
    g2 = torch.autograd.grad(whole.nll.sum(), list(net.parameters()))
    a = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
    b = scorer.score(nodes, edges, requires_grad=True)
    both = torch.autograd.grad(a.nll.sum() + b.nll.sum(), list(net.parameters()))
    for x, y, z in zip(g1, g2, both):
        assert torch.allclose(x + y, z, rtol=1e-5, atol=1e-6)
    again = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
    scorer.set_scaffolds((sn, se), attach)                 # in place: same table, a new version
    with pytest.raises(RuntimeError, match="set_scaffolds"):
        again.nll.sum().backward()
    net.zero_grad()
    stale = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
    with torch.no_grad():
        next(net.parameters()).mul_(1.0)
    with pytest.raises(RuntimeError, match="inplace"):
        stale.nll.sum().backward()


# ---- refusals ------------------------------------------------------------------------------------------------------
def _valid_scaffold(x, e):
    try:
        P.route(x, e, SEGS)
        return True
    except ValueError:
        return False


def _refusal(case):
    """molecules, scaffold table, ids and attachment points where molecule m is the first the rule cannot score"""
    nodes, edges, _ = _fixture(40)
    M = nodes.shape[0]
    ks = np.array([min(3, P.n_atoms(nodes[i])) for i in range(M)])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    ids = np.arange(M)
    attach = [SR.decoration_points(nodes[i], edges[i], int(ks[i])) for i in range(M)]
    nodes, edges = nodes.copy(), edges.copy()
    m = 5
    if case == "prefix":                       # another atom type in the scaffold's rows
        t = int(np.argmax(nodes[m, 1, :5]))
        nodes[m, 1, :5] = 0
        nodes[m, 1, (t + 1) % 5] = 1
    elif case == "extra bond":                 # the scaffold lacks one bond among its atoms (a ring bond of a prefix)
        found = None
        for i in range(M):
            k = min(6, P.n_atoms(nodes[i]))
            x, e = SR.prefix(nodes[i], edges[i], k)
            for u, v in np.argwhere(np.triu(e.any(-1))):
                e2 = e.copy()
                e2[u, v] = e2[v, u] = 0
                if _valid_scaffold(x, e2):
                    found = (i, x, e2)
                    break
            if found:
                break
        if found is None:
            pytest.skip("no ring among the fixture's 6-atom prefixes")
        m, sn[found[0]], se[found[0]] = found
    elif case == "fewer atoms":                # the scaffold is molecule m plus one atom bonded to its last one
        m = next(i for i in range(M) if P.n_atoms(nodes[i]) < 13)
        n = P.n_atoms(nodes[m])
        sn[m], se[m] = nodes[m], edges[m]
        sn[m, n, 0] = sn[m, n, 5] = 1
        se[m, n - 1, n, 0] = se[m, n, n - 1, 0] = 1
    elif case == "masked":                     # every scaffold atom protected: the first decoration add is forbidden
        attach[m] = []
    else:
        ids[m] = M
    return nodes, edges, sn, se, ids, attach, m


WHY = {"prefix": "does not begin with its scaffold", "extra bond": "does not begin with its scaffold",
       "fewer atoms": "does not begin with its scaffold", "masked": "attachment points forbid", "id": "outside [-1, 40)"}


@pytest.mark.parametrize("case", list(WHY))
def test_refusals_name_the_molecule_before_any_replay(case):
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, sn, se, ids, attach, m = _refusal(case)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 32, scaffolds=(sn, se), attachment=attach if case == "masked" else None, **GDB13)
    with pytest.raises(ValueError) as e:
        scorer.score(nodes, edges, scaffold_ids=ids)
    msg = str(e.value)
    assert WHY[case] in msg, msg
    assert (f"molecule {m} " in msg) or (f"scaffold_ids[{m}]" in msg), msg
    assert scorer.replays == 0
    if case == "extra bond":
        assert "extra bond between two scaffold atoms" in msg


def test_scaffold_ids_need_a_table_and_invalid_molecules_keep_their_message():
    from graphinvent_b200 import preprocess
    from graphinvent_b200.graphed import RouteScorer
    from tests.test_gpu_route_nll import _bad_sets
    nodes, edges, _ = _fixture(12)
    net, _, _ = _net("GGNN")
    with pytest.raises(ValueError, match="scaffold table"):
        RouteScorer(net, 32, **GDB13).score(nodes, edges, scaffold_ids=np.zeros(12, np.int64))
    for case, (n, e, why) in _bad_sets().items():
        ks = np.array([min(2, max(P.n_atoms(nodes[m]), 1)) for m in range(12)])
        sn, se = SR.prefix_scaffolds(nodes, edges, ks)
        scorer = RouteScorer(net, 32, scaffolds=(sn, se), **GDB13)
        ids = np.arange(12)
        with pytest.raises(ValueError) as ours:
            scorer.score(n, e, scaffold_ids=ids)
        with pytest.raises(ValueError) as theirs:
            list(preprocess.groups(n, e, 32, 5, 3))
        assert str(ours.value) == str(theirs.value), case
        assert scorer.replays == 0


# ---- guarded buffers -----------------------------------------------------------------------------------------------
def test_kernels_stay_inside_their_buffers():
    """plan, fill, mask, probs and dlogits of the conditional route on guard-banded buffers whose interiors start
    poisoned: the filled states, actions, scaffold ids and atom counts equal the restatement's, the masked rows equal
    the fp64 rule, and no band changes"""
    from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, check, lib
    from graphinvent_b200.generation import ScaffoldTable
    nodes, edges, _ = _fixture(30)
    sn, se, ids, attach = _case(nodes, edges, seed=6, whole=(4,))
    X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, SEGS)
    protect = SR.protect_of(sn, attach)
    masks = SR.state_masks(sid, n_at, sn, protect, 13, 3, 45)
    S, M, B, N, Fd, Ef, apd = X.shape[0], nodes.shape[0], 37, 13, 8, 3, 625
    table = ScaffoldTable(sn, se, attach, N, Fd, Ef, (5, 3, 0, 0), "cuda")
    sc = table.struct()
    d = PPDims(N=N, F=Fd, Ef=Ef, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=B)
    bd = ctypes.byref(d)
    chunk = 40
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    gi = Guarded.like(torch.from_numpy(ids.astype(np.int32)).cuda())
    ws = Guarded(lib.gib_route_plan_ws_bytes(bd, chunk))
    off = Guarded(4 * (M + 1))
    status = Guarded(4 * PP_STATUS_INTS)
    ctl, slots, s_ids, s_n = Guarded(8), Guarded(8 * B), Guarded(4 * B), Guarded(4 * B)
    on, oe = Guarded(B * N * Fd), Guarded(B * N * N * Ef)
    lik, coef, dl = Guarded(4 * S), Guarded.like(torch.ones(S, device="cuda")), Guarded(4 * B * apd)
    logits = Guarded.like(torch.randn(B, apd, device="cuda", generator=torch.Generator("cuda").manual_seed(1)) * 4)
    bufs = (gn, ge, gi, ws, off, status, ctl, slots, s_ids, s_n, on, oe, lik, coef, dl, logits)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda g: ctypes.c_void_p(g.ptr())
    check(lib.gib_route_plan_scaffold(bd, p(gn), p(ge), M, chunk, ctypes.byref(sc), p(gi), p(ws), p(off), p(status),
                                      st), "gib_route_plan_scaffold")
    sw = status.view(torch.int32, (PP_STATUS_INTS,)).cpu().numpy()
    assert sw[3] == 0 and sw[1] == 0 and sw[5] == S and sw[6] == 0
    assert np.array_equal(off.view(torch.int32, (M + 1,)).cpu().numpy(), offsets)
    raw = logits.view().clone()
    for r in range(-(-S // B)):
        logits.view().copy_(raw)
        check(lib.gib_route_fill_scaffold(bd, p(gn), p(ge), chunk, p(ws), p(off), p(status), p(gi), p(ctl), p(slots),
                                          p(s_ids), p(s_n), p(on), p(oe), st), "gib_route_fill_scaffold")
        check(lib.gib_route_mask_logits(B, N, Ef, apd, ctypes.byref(sc), p(s_ids), p(s_n), p(logits), st),
              "gib_route_mask_logits")
        check(lib.gib_route_probs(B, apd, p(logits), p(slots), p(lik), st), "gib_route_probs")
        check(lib.gib_route_dlogits(B, apd, p(logits), p(slots), p(coef), p(dl), None, st), "gib_route_dlogits")
        check(lib.gib_rl_next_round(ctypes.c_void_p(status.ptr() + 24), st), "gib_rl_next_round")
        sl = slots.view(torch.int32, (2, B)).cpu().numpy()
        live = min(B, S - r * B)
        dst = sl[1]
        assert (dst[:live] >= 0).all() and (dst[live:] == -1).all()
        assert np.array_equal(sl[0][:live], acts[dst[:live]])
        xn, xe = on.view(torch.int8, (B, N, Fd)).cpu().numpy(), oe.view(torch.int8, (B, N, N, Ef)).cpu().numpy()
        assert np.array_equal(xn[:live], X[dst[:live]]) and np.array_equal(xe[:live], E[dst[:live]])
        assert not xn[live:].any() and not xe[live:].any()
        si, sn_ = s_ids.view(torch.int32, (B,)).cpu().numpy(), s_n.view(torch.int32, (B,)).cpu().numpy()
        assert np.array_equal(si[:live], sid[dst[:live]]) and (si[live:] == -1).all()
        want_n = np.where(sid[dst[:live]] >= 0, n_at[dst[:live]], -1)
        assert np.array_equal(sn_[:live], want_n) and (sn_[live:] == -1).all()
        lg = logits.view().cpu()
        assert torch.equal(torch.isinf(lg[:live]), torch.from_numpy(masks[dst[:live]]))
        assert torch.equal(lg[live:], raw[live:].cpu())
        dlv = dl.view(torch.float32, (B, apd)).cpu()
        assert (dlv[:live][torch.from_numpy(masks[dst[:live]])] == 0).all() and torch.isfinite(dlv).all()
    pl = lik.view(torch.float32, (S,)).cpu()
    assert torch.isfinite(pl).all() and (pl > 0).all()
    torch.cuda.synchronize()
    for g in bufs:
        assert g.intact(), g.damage()


# ---- fine-tuning a decorator ---------------------------------------------------------------------------------------
def _eager_conditional_nll(net, X, E, acts, masks, offsets, B):
    """nll per molecule with autograd through `model(nodes, edges)` in capacity mode at the scorer's capacity,
    batches of B padded states, the mask on the logits and ATen's log-softmax gather"""
    from graphinvent_b200.graphed import route_entry_capacity
    S, N, Ef = X.shape[0], X.shape[1], E.shape[3]
    net.entry_capacity = route_entry_capacity(B, N, Ef)
    try:
        lp = []
        for s in range(0, S, B):
            k = min(B, S - s)
            x = torch.zeros(B, *X.shape[1:], device="cuda")
            e = torch.zeros(B, *E.shape[1:], device="cuda")
            x[:k], e[:k] = torch.from_numpy(X[s:s + k]).cuda(), torch.from_numpy(E[s:s + k]).cuda()
            o = net(x, e)[:k].masked_fill(torch.from_numpy(masks[s:s + k]).cuda(), float("-inf"))
            a = torch.from_numpy(acts[s:s + k]).cuda().view(-1, 1)
            lp.append(torch.log_softmax(o, 1).gather(1, a).view(-1))
    finally:
        net.entry_capacity = None
    lp = torch.cat(lp)
    seg = torch.repeat_interleave(torch.arange(offsets.shape[0] - 1), torch.from_numpy(np.diff(offsets))).cuda()
    return -torch.zeros(offsets.shape[0] - 1, device="cuda", dtype=lp.dtype).index_add(0, seg, lp)


def test_fine_tuning_a_decorator_tracks_eager_steps_and_lowers_the_nll():
    from graphinvent_b200.graphed import RouteScorer
    from graphinvent_b200.optim import FlatAdam
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"][:128], z["gdb13_1K_train/edges"][:128]
    sn, se, ids, attach = _case(nodes, edges, seed=7)
    (net, _, _), (twin, _, _), (frozen, _, _) = _net("GGNN", seed=4), _net("GGNN", seed=4), _net("GGNN", seed=4)
    before = RouteScorer(frozen, 256, **GDB13).score(nodes, edges)
    X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, SEGS)
    masks = SR.state_masks(sid, n_at, sn, SR.protect_of(sn, attach), 13, 3, 45)
    opt, opt_e = FlatAdam(net.parameters(), lr=1e-4), FlatAdam(twin.parameters(), lr=1e-4)
    scorer = _scorer(net, 256, sn, se, attach, True)
    losses = []
    for step in range(8):
        opt.zero_grad()
        loss = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True).nll.mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if step < 4:
            opt_e.zero_grad()
            le = _eager_conditional_nll(twin, X, E, acts, masks, offsets, scorer.B).mean()
            le.backward()
            opt_e.step()
            assert abs(losses[-1] - le.item()) <= 1e-4 * abs(le.item()), (step, losses[-1], le.item())
    with torch.no_grad():
        final = scorer.score(nodes, edges, scaffold_ids=ids).nll.mean().item()
    assert final < losses[0], (losses[0], final)
    after = RouteScorer(frozen, 256, **GDB13).score(nodes, edges)
    assert all(torch.equal(a, b) for a, b in zip(before, after))
