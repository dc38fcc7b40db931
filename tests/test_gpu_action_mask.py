"""GPU: the action mask (`gib_action_mask_logits`, `action_mask=` of the generators) -- the kernel against the numpy
rule of tests/action_mask_reference.py entry by entry, its writes confined to its rows, masked generation with the
pretrained gdb13 GGNN and a seeded EMN (no invalid terminations, every molecule within the valence table, the
recorded likelihoods an fp64 masked softmax, eager and captured bit for bit), and the masked RL rollout's
log-likelihoods and gradients against the eager masked rollout."""
import copy
import ctypes
from collections import namedtuple

import numpy as np
import pytest
import torch

from tests import action_mask_reference as R
from tests.conftest import pretrained_path

pytestmark = pytest.mark.gpu

GDB13 = namedtuple("C", "atom_types formal_charge")(["C", "N", "O", "S", "Cl"], [-1, 0, 1])


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _random_states(rng, B, N, A, CH, H, C, Ef):
    """nodes [B, N, F] / edges [B, N, N, Ef] int8 and atom counts: one-hot atoms, random bonds, some pairs with two
    types, empty and full graphs"""
    F = A + CH + H + C
    nodes = np.zeros((B, N, F), np.int8)
    edges = np.zeros((B, N, N, Ef), np.int8)
    n = rng.integers(0, N + 1, B)
    n[:3] = [0, min(1, N), N]                                   # empty, single-atom and full graphs
    for b in range(B):
        for i in range(n[b]):
            nodes[b, i, rng.integers(0, A)] = 1
            nodes[b, i, A + rng.integers(0, CH)] = 1
            if H:
                nodes[b, i, A + CH + rng.integers(0, H)] = 1
            if C:
                nodes[b, i, A + CH + H + rng.integers(0, C)] = 1
            if i:
                for j in set(rng.integers(0, i, 1 + int(rng.random() < 0.4))):
                    t = rng.integers(0, Ef)
                    edges[b, i, j, t] = edges[b, j, i, t] = 1
                    if Ef > 1 and rng.random() < 0.1:
                        edges[b, i, j, (t + 1) % Ef] = edges[b, j, i, (t + 1) % Ef] = 1
    return nodes, edges, n.astype(np.int32)


def _mask(N, A, CH, H, C, Ef, mode, V=None):
    from graphinvent_b200.generation import ActionMask
    apd = N * (A * CH * max(H, 1) * max(C, 1) * Ef + Ef) + 1
    return ActionMask(mode, V, None, (A, CH, H, C), N, A + CH + H + C, Ef, apd, "cuda"), apd


CASES = [(13, 5, 3, 0, 0, 3), (13, 2, 2, 4, 0, 3), (9, 2, 2, 0, 3, 4), (7, 2, 1, 4, 3, 2), (2, 2, 1, 0, 3, 4),
         (1, 1, 2, 2, 0, 3), (38, 4, 3, 0, 0, 4), (127, 1, 1, 0, 0, 1), (64, 2, 1, 3, 0, 2)]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mode", ["structure", "valence"])
@pytest.mark.parametrize("int8", [False, True])
def test_kernel_matches_the_oracle(case, mode, int8):
    N, A, CH, H, C, Ef = case
    rng = np.random.default_rng(4 * CASES.index(case) + 2 * (mode == "valence") + int(int8))
    B = 37 if N < 100 else 6
    V = rng.integers(0, 5, (A, CH)) if mode == "valence" else None
    m, apd = _mask(N, A, CH, H, C, Ef, mode, V)
    nodes, edges, n = _random_states(rng, B, N, A, CH, H, C, Ef)
    logits = torch.randn(B, apd, device="cuda")
    want_keep = logits.clone()
    dt = torch.int8 if int8 else torch.float32
    nd, ed = torch.from_numpy(nodes).cuda().to(dt), torch.from_numpy(edges).cuda().to(dt)
    m.apply(B, logits, torch.from_numpy(n).cuda(), _stream(), nd, ed, int8=int8, first_slot=0)
    got = torch.isneginf(logits).cpu().numpy()
    for b in range(B):
        want = R.forbidden(nodes[b], edges[b], int(n[b]), N, A, CH, H, C, Ef, V, m.bond_orders, m.imp_h)
        assert (got[b] == want).all(), (b, int(n[b]), np.flatnonzero(got[b] != want)[:8])
    keep = ~torch.from_numpy(got).cuda()
    assert torch.equal(logits[keep], want_keep[keep])


@pytest.mark.parametrize("int8", [False, True])
def test_combined_with_the_scaffold_rule_and_the_round_gate(int8):
    """one launch: forbidden = attachment rule OR action rule; slot 0 left alone at first_slot = 1; a gated call
    writes nothing once the batch is done; `row` reads the counts and scaffold ids of one record row (int8: the
    RL backward's launch with attachment points)"""
    from graphinvent_b200._lib import Scaffolds
    N, A, CH, H, C, Ef = 13, 5, 3, 0, 0, 3
    rng = np.random.default_rng(3)
    B, S = 40, 3
    m, apd = _mask(N, A, CH, H, C, Ef, "valence", rng.integers(1, 5, (A, CH)))
    nodes, edges, n = _random_states(rng, B, N, A, CH, H, C, Ef)
    k = np.array([1, 3, 5], np.int32)
    ids = rng.integers(-1, S, B).astype(np.int32)
    protect_bits = np.zeros((S, 128), bool)
    for s in range(S):
        protect_bits[s, :k[s]] = rng.random(k[s]) < 0.6
    words = (protect_bits.reshape(S, 4, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
    protect = torch.from_numpy(words.astype(np.uint32).view(np.int32)).cuda()
    n_atoms = torch.from_numpy(k).cuda()
    sc = Scaffolds(n_atoms=n_atoms.data_ptr(), protect=protect.data_ptr(), S=S)
    per = A * CH * Ef

    def scaffold_rule(b):
        out = np.zeros(apd, bool)
        s = ids[b]
        if s < 0:
            return out
        for i in range(k[s]):
            if protect_bits[s, i]:
                out[i * per:(i + 1) * per] = True
                out[N * per + i * Ef:N * per + (i + 1) * Ef] = True
        if n[b] - 1 < k[s]:
            out[N * per:N * per + N * Ef] = True
        return out

    # two record rows: row 1 holds the real counts / ids, row 0 garbage
    n_rows = torch.from_numpy(np.stack([np.zeros_like(n), n])).cuda()
    id_rows = torch.from_numpy(np.stack([np.full_like(ids, 2), ids])).cuda()
    row = torch.ones(1, dtype=torch.int32, device="cuda")
    logits = torch.randn(B, apd, device="cuda")
    ref = logits.clone()
    dt = torch.int8 if int8 else torch.float32
    m.apply(B, logits, n_rows, _stream(), torch.from_numpy(nodes).cuda().to(dt), torch.from_numpy(edges).cuda().to(dt),
            int8=int8, sc=sc, slot_ids=id_rows, row=row, first_slot=1)
    got = torch.isneginf(logits).cpu().numpy()
    assert torch.equal(logits[0], ref[0])
    for b in range(1, B):
        want = R.forbidden(nodes[b], edges[b], int(n[b]), N, A, CH, H, C, Ef, m.valence, m.bond_orders, m.imp_h)
        want |= scaffold_rule(b)
        assert not want[-1]
        assert (got[b] == want).all(), b
    # the gate: counters[0] >= B (the batch is done) -> nothing written
    state = torch.tensor([3, 0], dtype=torch.int32, device="cuda")
    for counters, writes in ((torch.tensor([B, 0], dtype=torch.int32, device="cuda"), False),
                             (torch.tensor([0, 0], dtype=torch.int32, device="cuda"), True)):
        lg = ref.clone()
        m.apply(B, lg, torch.from_numpy(n).cuda(), _stream(), torch.from_numpy(nodes).cuda().float(),
                torch.from_numpy(edges).cuda().float(), state=state, counters=counters)
        assert bool(torch.isneginf(lg).any()) == writes


def test_writes_stay_inside_the_rows():
    """guard bands of poison around the logits, the state, the counts and the rule table are left as they were, the
    state and the table are not written, and no entry outside the forbidden set changes"""
    N, A, CH, H, C, Ef = 13, 2, 2, 4, 3, 3
    rng = np.random.default_rng(9)
    B, G = 29, 4096
    m, apd = _mask(N, A, CH, H, C, Ef, "valence", rng.integers(0, 5, (A, CH)))
    nodes, edges, n = _random_states(rng, B, N, A, CH, H, C, Ef)

    def banded(a, dtype, poison):
        t = torch.full((G + a.size + G,), poison, dtype=dtype, device="cuda")
        t[G:G + a.size] = torch.from_numpy(a.ravel()).to(dtype).cuda()
        return t, t[G:G + a.size]

    lg_buf, lg = banded(rng.standard_normal(B * apd).astype(np.float32), torch.float32, float("nan"))
    nd_buf, nd = banded(nodes, torch.float32, float("nan"))
    ed_buf, ed = banded(edges, torch.float32, float("nan"))
    n_buf, nn_ = banded(n, torch.int32, -7)
    tb_buf, m.table = banded(m.table.cpu().numpy(), torch.int32, 1 << 30)     # the rule table, banded too
    before = [t.clone() for t in (lg_buf, nd_buf, ed_buf, n_buf, tb_buf)]
    m.apply(B, lg.view(B, apd), nn_, _stream(), nd.view(B, N, -1), ed.view(B, N, N, Ef), first_slot=0)
    torch.cuda.synchronize()
    assert torch.equal(tb_buf, before[4])
    for t, t0 in zip((lg_buf, nd_buf, ed_buf, n_buf), before):
        for part in (slice(0, G), slice(t.numel() - G, t.numel())):
            assert torch.equal(t[part].isnan(), t0[part].isnan()) and torch.equal(
                torch.nan_to_num(t[part]), torch.nan_to_num(t0[part]))
    assert torch.equal(torch.nan_to_num(nd_buf), torch.nan_to_num(before[1]))
    assert torch.equal(torch.nan_to_num(ed_buf), torch.nan_to_num(before[2]))
    changed = (lg != before[0][G:G + B * apd]).view(B, apd)
    assert torch.isneginf(lg.view(B, apd)[changed]).all()


# ---- generation --------------------------------------------------------------------------------------------------
def _pretrained():
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    C = make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    return C, net.cuda().eval()


def _seeded_emn():
    from graphinvent_b200.config import make_constants
    from tests.test_gpu_generation_layouts import _seeded_model
    C = make_constants("EMN")
    net, _ = _seeded_model("EMN", C, 5)
    return C, net.eval()


def _gdb13_valence():
    from graphinvent_b200.config import action_rule_table
    return action_rule_table(5, 3, 3, 0, None, GDB13)[0]


def _eager_masked(model, C, B, U, mode, V, record=False, layout=None):
    """the eager generator's own masked round loop on the uniforms U [2N, B], the model in capacity mode at the graphed
    generator's capacity; record: per round (nodes, edges, n_nodes, raw logits, action, likelihood)"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import entry_capacity
    kw = dict(n_atom_types=5, n_formal_charge=3) if layout is None else {}
    gen = GraphGenerator(model, B, constants=C, action_mask=mode, max_valence=V, **kw)
    st, n, rnd, rec = _stream(), 0, 0, []
    model.entry_capacity = entry_capacity(B, gen.N, gen.Ef)
    try:
        with torch.no_grad():
            while n < B:
                assert rnd < 2 * gen.N
                raw = model(*gen._model_inputs(model)).contiguous()
                out = raw.clone()
                gen._mask(out, st)
                action, lik = Fn.sample_actions(out, uniforms=U[rnd])
                if record:
                    rec.append([t.clone() for t in (gen.nodes, gen.edges, gen.n_nodes, raw, action, lik)])
                gen._round(rnd, action, lik, st)
                n = int(gen._counters[0].item())
                rnd += 1
    finally:
        model.entry_capacity = None
    gen.rounds = rnd
    return gen, rec


def _check_batch(gen, B, mode, V):
    pt = gen.properly_terminated[:B].cpu().numpy()
    assert (pt == 1).all(), f"{int((pt != 1).sum())} of {B} molecules ended on an invalid action"
    if mode == "valence":
        nodes, edges = gen.generated_nodes[:B].cpu().numpy(), gen.generated_edges[:B].cpu().numpy()
        nn_ = gen.generated_n_nodes[:B].cpu().numpy()
        for b in range(B):
            assert R.valence_ok(nodes[b], edges[b], int(nn_[b]), 5, 3, 0, V, (2, 4, 6), ()), b


@pytest.mark.parametrize("which", ["pretrained", "emn"])
@pytest.mark.parametrize("mode", ["structure", "valence"])
def test_masked_generation_is_valid_and_captured_equals_eager(which, mode):
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained() if which == "pretrained" else _seeded_emn()
    V = _gdb13_valence() if mode == "valence" else None
    B = 256
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, action_mask=mode, max_valence=V)
    for seed in range(1, 5):
        U = torch.rand(2 * C.max_n_nodes, B, generator=torch.Generator("cuda").manual_seed(seed), device="cuda")
        n = gen.build_graphs(uniforms=U)
        assert n >= B
        _check_batch(gen, B, mode, V)
        if seed <= 2:
            eager, _ = _eager_masked(net, C, B, U, mode, V)
            assert eager.rounds == gen.rounds
            for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "generated_likelihoods",
                         "properly_terminated", "nodes", "edges", "n_nodes"):
                assert torch.equal(getattr(gen, name), getattr(eager, name)), name


@pytest.mark.parametrize("mode", ["structure", "valence"])
def test_recorded_likelihoods_are_a_masked_softmax(mode):
    """every round's stored likelihood = the fp64 softmax of the model's logits renormalised over the actions the
    oracle allows in the replayed state; the sampled action is always allowed"""
    C, net = _pretrained()
    V = _gdb13_valence() if mode == "valence" else None
    B = 128
    U = torch.rand(2 * C.max_n_nodes, B, generator=torch.Generator("cuda").manual_seed(11), device="cuda")
    _, rec = _eager_masked(net, C, B, U, mode, V, record=True)
    worst = 0.0
    for nodes, edges, n_nodes, raw, action, lik in rec:
        nodes, edges, n_nodes = nodes.cpu().numpy(), edges.cpu().numpy(), n_nodes.cpu().numpy()
        raw, action, lik = raw.double().cpu().numpy(), action.cpu().numpy(), lik.double().cpu().numpy()
        for b in range(1, B):
            f = R.forbidden(nodes[b], edges[b], int(n_nodes[b]), 13, 5, 3, 0, 0, 3, V, (2, 4, 6), ())
            assert not f[action[b]], b
            x = np.where(f, -np.inf, raw[b])
            p = np.exp(x - x.max())
            p /= p.sum()
            worst = max(worst, abs(p[action[b]] - lik[b]) / max(p[action[b]], 1e-30))
    assert worst <= 1e-5, worst


def test_default_generator_is_unchanged():
    """action_mask=None: the same batch as the generator built without the argument, and no mask object"""
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained()
    B = 128
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(4), device="cuda")
    a = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    b = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, action_mask=None)
    assert a.action_mask is None and b.action_mask is None
    a.build_graphs(uniforms=U)
    b.build_graphs(uniforms=U)
    for name in ("generated_nodes", "generated_edges", "generated_likelihoods", "properly_terminated"):
        assert torch.equal(getattr(a, name), getattr(b, name))


# ---- RL ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,frozen_prior", [("structure", False), ("valence", False), ("valence", True)])
def test_masked_rl_rollout_matches_eager(mode, frozen_prior):
    from graphinvent_b200.generation import GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from tests.test_gpu_rl_graphed import _loss
    from tests.test_gpu_generation_layouts import _seeded_model
    C, agent = _pretrained()
    prior, _ = _seeded_model("GGNN", C, 2)
    V = _gdb13_valence() if mode == "valence" else None
    if frozen_prior:
        for p in prior.parameters():
            p.requires_grad_(False)
    B = 96
    gen = GraphedGeneratorRL(agent, B, n_atom_types=5, n_formal_charge=3, action_mask=mode, max_valence=V)
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(3), device="cuda")
    _, agent_ll, prior_ll, pt = gen.sample(agent, prior, uniforms=U)
    assert (pt == 1).all()
    R_ = gen.rounds
    p_a, p_b, acts = gen.p_a[:R_].clone(), gen.p_b[:R_].clone(), gen.act_rec[:R_].clone()
    # the rollout's probabilities against an fp64 softmax of the agent's logits on the recorded states, masked by the
    # numpy rule (independent of the kernel both generators share)
    with torch.no_grad():
        for r in range(R_):
            xs, es = gen.rec_nodes[r].float(), gen.rec_edges[r].float()
            lg = agent(xs, es).double().cpu().numpy()
            xs, es, nr = xs.cpu().numpy(), es.cpu().numpy(), gen.rec_n[r].cpu().numpy()
            a, pr = acts[r].cpu().numpy(), p_a[r].double().cpu().numpy()
            for b in range(1, B, 7):
                f = R.forbidden(xs[b], es[b], int(nr[b]), 13, 5, 3, 0, 0, 3, V, (2, 4, 6), ())
                assert not f[a[b]]
                x = np.where(f, -np.inf, lg[b])
                q = np.exp(x - x.max())
                assert abs(q[a[b]] / q.sum() - pr[b]) <= 1e-4 * pr[b] + 1e-7, (r, b)
    agent.zero_grad()
    _loss(agent_ll, prior_ll).backward()
    assert gen.backward_rounds == [R_, 0 if frozen_prior else R_]
    assert torch.equal(gen.recomputed_p[0][:R_], p_a)
    if not frozen_prior:
        assert torch.equal(gen.recomputed_p[1][:R_], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager = GraphGeneratorRL(agent2, B, n_atom_types=5, n_formal_charge=3, action_mask=mode, max_valence=V)
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eager.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert eager.rounds == R_
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    assert torch.isfinite(ll_a).all() and torch.isfinite(ll_p).all()
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    pairs = [(agent, agent2)] + ([] if frozen_prior else [(prior, prior2)])
    for m, m2 in pairs:
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        assert total > 0
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total
    if frozen_prior:
        assert all(p.grad is None for p in prior.parameters())


def test_masked_generation_in_the_l3_layout():
    """implicit H and chirality: a seeded GGNN, both modes, captured equal to eager, every molecule properly
    terminated and (valence, implicit hydrogens counted) within the table"""
    from graphinvent_b200.graphed import GraphedGenerator
    from tests.test_gpu_generation_layouts import _constants_for, _seeded_model
    C = _constants_for("GGNN", "L3")
    net, _ = _seeded_model("GGNN", C, 7)
    A, CH, H = C.n_atom_types, C.n_formal_charge, C.n_imp_H
    V = np.full((A, CH), 4)
    V[-1] = 2
    B = 128
    for mode in ("structure", "valence"):
        gen = GraphedGenerator(net.eval(), B, constants=C, action_mask=mode, max_valence=V if mode == "valence" else None)
        U = torch.rand(2 * C.max_n_nodes, B, generator=torch.Generator("cuda").manual_seed(5), device="cuda")
        assert gen.build_graphs(uniforms=U) >= B
        assert (gen.properly_terminated[:B] == 1).all()
        eager, _ = _eager_masked(net, C, B, U, mode, V if mode == "valence" else None, layout="L3")
        for name in ("generated_nodes", "generated_edges", "generated_likelihoods", "properly_terminated"):
            assert torch.equal(getattr(gen, name), getattr(eager, name)), (mode, name)
        if mode == "valence":
            nodes, edges = gen.generated_nodes[:B].cpu().numpy(), gen.generated_edges[:B].cpu().numpy()
            nn_ = gen.generated_n_nodes[:B].cpu().numpy()
            for b in range(B):
                assert R.valence_ok(nodes[b], edges[b], int(nn_[b]), A, CH, H, V, (2, 4, 6), np.arange(H)), b


def test_masked_scaffold_rl_rollout_matches_eager():
    """scaffolds with attachment points and the valence mask together: the rollout's one combined launch, and the
    backward's int8 + scaffold + record-row launch, against the eager rollout"""
    from graphinvent_b200.generation import GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from tests.test_gpu_rl_graphed import _loss
    from tests.test_gpu_generation_layouts import _seeded_model
    from tests.test_gpu_scaffold_generation import _gdb13_constants, attachment_lists, gdb13_scaffolds
    C = _gdb13_constants()
    agent, _ = _seeded_model("GGNN", C, 1)
    prior, _ = _seeded_model("GGNN", C, 2)
    sn, se = gdb13_scaffolds()
    att = attachment_lists(sn, seed=1)
    V = _gdb13_valence()
    B = 96
    kw = dict(constants=C, scaffolds=(sn, se), attachment=att, action_mask="valence", max_valence=V)
    gen = GraphedGeneratorRL(agent, B, **kw)
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(2), device="cuda")
    _, agent_ll, prior_ll, pt = gen.sample(agent, prior, uniforms=U)
    assert (pt == 1).all()
    R_ = gen.rounds
    p_a, acts = gen.p_a[:R_].clone(), gen.act_rec[:R_].clone()
    _loss(agent_ll, prior_ll).backward()
    assert torch.equal(gen.recomputed_p[0][:R_], p_a)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager = GraphGeneratorRL(agent2, B, **kw)
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eager.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert torch.equal(eager.generated_scaffolds, gen.generated_scaffolds)
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


# ---- RouteScorer -------------------------------------------------------------------------------------------------
def _route_setup(M=40):
    import os
    from tests.conftest import ROOT
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    z = np.load(os.path.join(ROOT, "tests", "golden", "route_nll_gdb13.npz"))
    nodes, edges = z["nodes"][:M], z["edges"][:M]
    C = O.make_constants("GGNN")
    sd = O.init_state_dict(C, seed=3)
    net = mpnn.create(C)
    net.load_state_dict(sd)
    V = _gdb13_valence()
    ok = [R.valence_ok(nodes[m], edges[m], int(nodes[m].any(-1).sum()), 5, 3, 0, V, (2, 4, 6), ())
          for m in range(nodes.shape[0])]
    return nodes[ok], edges[ok], net.cuda().eval(), sd, C, V


def _oracle_masked(sd, C, nodes, edges, V):
    """fp64: per route state the masked softmax probability of its action, the offsets and the log-p bound"""
    from tests import preprocess_reference as P
    from tests import route_nll_reference as RN
    X, E, acts, offsets = RN.build_order_states(nodes, edges, P.segments(5, 3))
    _, logits = RN.probabilities(sd, C, X, E, acts)
    logits = logits.numpy()
    p = np.empty(len(acts))
    for s in range(len(acts)):
        f = R.forbidden(X[s], E[s], int(X[s].any(-1).sum()), 13, 5, 3, 0, 0, 3, V, (2, 4, 6), ())
        assert not f[acts[s]]
        x = np.where(f, -np.inf, logits[s])
        q = np.exp(x - x.max())
        p[s] = q[acts[s]] / q.sum()
    return p, offsets, RN.log_p_bound(sd, C, X, E, acts, torch.from_numpy(logits)).numpy(), (X, E, acts)


@pytest.mark.parametrize("mode", ["structure", "valence"])
def test_route_scorer_masked_likelihoods_match_the_fp64_masked_softmax(mode):
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, net, sd, C, V = _route_setup()
    Vm = V if mode == "valence" else None
    sc = RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, action_mask=mode, max_valence=Vm, chunk_molecules=16)
    out = sc.score(nodes, edges)
    p, offsets, bound, _ = _oracle_masked(sd, C, nodes, edges, Vm)
    assert out.offsets.cpu().numpy().tolist() == offsets.tolist()
    got = out.likelihoods.double().cpu().numpy()
    assert (np.abs(np.log(got) - np.log(p)) <= bound).all()
    plain = RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, chunk_molecules=16).score(nodes, edges)
    assert (out.likelihoods >= plain.likelihoods * (1 - 1e-5)).all()     # masking only renormalises upwards
    # conditional: every molecule from its own first atom (a one-atom scaffold, no attachment points): the route's
    # states past the first add, scored as the unconditional masked scorer scores them
    k1 = nodes.copy()
    k1[:, 1:] = 0
    e1 = np.zeros_like(edges)
    cs = RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, action_mask=mode, max_valence=Vm, chunk_molecules=16, scaffolds=(k1, e1))
    ids = np.arange(nodes.shape[0], dtype=np.int64)
    ids[::3] = -1
    cond = cs.score(nodes, edges, scaffold_ids=ids)
    o, oc = out.offsets.cpu().numpy(), cond.offsets.cpu().numpy()
    for m in range(nodes.shape[0]):
        want = out.likelihoods[o[m] + (0 if ids[m] < 0 else 1):o[m + 1]]
        assert torch.allclose(cond.likelihoods[oc[m]:oc[m + 1]], want, rtol=2e-5, atol=0), m


def test_route_scorer_refuses_an_over_valent_molecule_by_index():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, net, sd, C, V = _route_setup(24)
    bad = nodes.copy()
    i = int(np.flatnonzero(edges[5].sum((1, 2)) > 0)[0])          # a bonded atom of molecule 5 becomes Cl-
    bad[5, i] = 0
    bad[5, i, 4] = bad[5, i, 5] = 1
    sc = RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, action_mask="valence", max_valence=V, chunk_molecules=8)
    with pytest.raises(ValueError, match=r"molecule 5 \(or a later one in molecules \[0, 8\)\).*over its limit"):
        sc.score(bad, edges)
    assert sc.replays == 0                                         # nothing of the chunk was scored
    RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, action_mask="structure", chunk_molecules=8).score(bad, edges)      # structurally fine
    sc.score(nodes, edges)


def test_route_scorer_masked_gradients_match_eager_autograd():
    """the recomputing backward with the masked logits against autograd through the module forward, the oracle's
    mask as a -inf bias and a log-softmax gather"""
    import copy as _copy
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, net, sd, C, V = _route_setup(32)
    sc = RouteScorer(net, 256, n_atom_types=5, n_formal_charge=3, action_mask="valence", max_valence=V, chunk_molecules=16)
    net.zero_grad()
    w = torch.linspace(0.5, 1.5, nodes.shape[0], device="cuda")
    (w * sc.score(nodes, edges, requires_grad=True).nll).sum().backward()
    net2 = _copy.deepcopy(net)
    net2.zero_grad()
    _, offsets, _, (X, E, acts) = _oracle_masked(sd, C, nodes, edges, V)
    bias = np.zeros((len(acts), sc.apd), np.float32)
    for s in range(len(acts)):
        bias[s][R.forbidden(X[s], E[s], int(X[s].any(-1).sum()), 13, 5, 3, 0, 0, 3, V, (2, 4, 6), ())] = -np.inf
    logits = net2(torch.from_numpy(X).float().cuda(), torch.from_numpy(E).float().cuda()) + torch.from_numpy(bias).cuda()
    logp = torch.log_softmax(logits, 1).gather(1, torch.from_numpy(acts).cuda().view(-1, 1)).view(-1)
    mol = torch.from_numpy(np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))).cuda()
    (-(w[mol] * logp).sum()).backward()
    total = sum(p.grad.norm().item() ** 2 for p in net2.parameters()) ** 0.5
    assert total > 0
    for p, p2 in zip(net.parameters(), net2.parameters()):
        assert (p.grad - p2.grad).norm().item() <= 1e-3 * p2.grad.norm().item() + 1e-5 * total
