"""GPU: constraints (`generation.Constraints`, `constraints=` of the generators and the route scorer) -- the
constrained mask kernel against tests/constraints_reference.py entry by entry, rows that stay sampleable, the
molecule check, the off set bit-identical to the unconstrained launch, constrained generation with the pretrained
gdb13 GGNN (every molecule within the set but for dead ends, captured equal to eager), set_constraints without a
recapture, the RL rollout and its backward, the route scorer, guarded buffers and determinism."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from tests import constraints_reference as R
from tests.guarded import Guarded
from tests.test_gpu_action_mask import GDB13, _gdb13_valence, _pretrained, _random_states

pytestmark = pytest.mark.gpu

GEN_STATE = ("generated_nodes", "generated_edges", "generated_n_nodes", "generated_likelihoods",
             "properly_terminated")
CASES = [(13, 5, 3, 0, 0, 3), (13, 2, 2, 4, 0, 3), (9, 2, 2, 0, 3, 4), (7, 2, 1, 4, 3, 2), (12, 3, 2, 0, 0, 1),
         (38, 4, 3, 0, 0, 4), (127, 1, 1, 0, 0, 1)]


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _mask(N, A, CH, H, C, Ef, mode, V=None, cons=None):
    from graphinvent_b200.generation import ActionMask
    apd = N * (A * CH * max(H, 1) * max(C, 1) * Ef + Ef) + 1
    return ActionMask(mode, V, None, (A, CH, H, C), N, A + CH + H + C, Ef, apd, "cuda", cons), apd


def _random_set(rng, N, A, CH, Ef, n_mean):
    """a Constraints by index whose bounds sit near a state of n_mean atoms, so that every field fires somewhere"""
    from graphinvent_b200.generation import Constraints
    pick = lambda p, lo, hi: (int(rng.integers(lo, hi + 1)) if rng.random() < p else None)
    mx = pick(0.5, max(1, n_mean - 2), N)
    mn = pick(0.5, 0, mx if mx is not None else N)
    types, budget = {}, mx if mx is not None else N
    for t in range(A):
        lo = pick(0.3, 0, 2)
        lo = lo if lo is not None and lo <= budget else None
        hi = pick(0.4, lo or 0, (lo or 0) + 3)
        if lo is not None:
            budget -= lo
        if lo is not None or hi is not None:
            types[t] = (lo, hi)
    charges = {c: int(rng.integers(0, 4)) for c in range(CH) if rng.random() < 0.3}
    bonds = {e: int(rng.integers(0, n_mean + 1)) for e in range(Ef) if rng.random() < 0.4}
    rmax = pick(0.4, 0, 3)
    rmin = pick(0.3, 0, rmax if rmax is not None else 3)
    ring = int(rng.choice([0, 3, 4, 5, 6, 8])) if rng.random() < 0.6 else None
    return Constraints(atoms=(mn, mx), atom_types=types, charges=charges, bonds=bonds, rings=(rmin, rmax),
                       min_ring_size=ring)


def _ring_states(rng, B, N, A, CH, H, C, Ef):
    """_random_states with extra bonds closing rings of every size"""
    nodes, edges, n = _random_states(rng, B, N, A, CH, H, C, Ef)
    for b in range(B):
        for _ in range(int(rng.integers(0, 3))):
            if n[b] >= 3:
                i, j = rng.choice(n[b], 2, replace=False)
                if not edges[b, i, j].any():
                    t = rng.integers(0, Ef)
                    edges[b, i, j, t] = edges[b, j, i, t] = 1
    return nodes, edges, n


def _protect(rng, S, k):
    bits = np.zeros((S, 128), bool)
    for s in range(S):
        bits[s, :k[s]] = rng.random(k[s]) < 0.5
    words = (bits.reshape(S, 4, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
    return bits, torch.from_numpy(words.astype(np.uint32).view(np.int32)).cuda()


# ---- 1. the kernel against the restatement --------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mode", ["structure", "valence"])
@pytest.mark.parametrize("int8", [False, True])
@pytest.mark.parametrize("attach", [False, True])
def test_kernel_matches_the_restatement(case, mode, int8, attach):
    from graphinvent_b200._lib import Scaffolds
    N, A, CH, H, C, Ef = case
    seed = 16 * CASES.index(case) + 8 * (mode == "valence") + 4 * int8 + 2 * attach
    rng = np.random.default_rng(seed)
    B = 29 if N < 100 else 5
    V = rng.integers(1, 5, (A, CH)) if mode == "valence" else None
    cons = _random_set(rng, N, A, CH, Ef, min(N, 8))
    m, apd = _mask(N, A, CH, H, C, Ef, mode, V, cons)
    t = R.table_dict(m.cons_table.cpu().numpy(), A, CH, Ef)
    nodes, edges, n = _ring_states(rng, B, N, A, CH, H, C, Ef)
    sc, ids, scaffold = None, None, [None] * B
    if attach:
        S = 3
        k = np.minimum(np.array([1, 3, 5], np.int32), N)
        bits, protect = _protect(rng, S, k)
        n_atoms = torch.from_numpy(k).cuda()
        sc = Scaffolds(n_atoms=n_atoms.data_ptr(), protect=protect.data_ptr(), S=S)
        ids_np = rng.integers(-1, S, B).astype(np.int32)
        ids = torch.from_numpy(ids_np).cuda()
        scaffold = [(int(k[s]), bits[s]) if s >= 0 else None for s in ids_np]
    logits = torch.randn(B, apd, device="cuda")
    keep0 = logits.clone()
    dt = torch.int8 if int8 else torch.float32
    nd, ed = torch.from_numpy(nodes).cuda().to(dt), torch.from_numpy(edges).cuda().to(dt)
    m.apply(B, logits, torch.from_numpy(n).cuda(), _stream(), nd, ed, int8=int8, sc=sc, slot_ids=ids, first_slot=0)
    got = torch.isneginf(logits).cpu().numpy()
    fired = 0
    for b in range(B):
        want = R.mask(t, nodes[b], edges[b], int(n[b]), N, A, CH, H, C, Ef, V, m.bond_orders, m.imp_h, scaffold[b])
        assert (got[b] == want).all(), (b, int(n[b]), np.flatnonzero(got[b] != want)[:8])
        assert not got[b].all()                                      # the row stays sampleable
        fired += int(want[-1])
    keep = ~torch.from_numpy(got).cuda()
    assert torch.equal(logits[keep], keep0[keep])


def test_every_field_fires_and_the_dead_end_keeps_terminate():
    """hand states on the gdb13 layout: a saturated 3-ring under min_atoms under 'valence' keeps terminate (dead
    end); the same state with a free valence masks it"""
    from graphinvent_b200.generation import Constraints
    N, A, CH, Ef = 13, 5, 3, 3
    V = _gdb13_valence()
    cons = Constraints(atoms=(6, None), constants=GDB13)
    m, apd = _mask(N, A, CH, 0, 0, Ef, "valence", V, cons)
    nodes = np.zeros((2, N, A + CH), np.int8)
    edges = np.zeros((2, N, N, Ef), np.int8)
    for b in range(2):
        for i in range(3):
            nodes[b, i, 0] = 1                                       # carbon
            nodes[b, i, A + 1] = 1                                   # neutral
        for i, j in ((0, 1), (1, 2), (0, 2)):
            edges[b, i, j, 1] = edges[b, j, i, 1] = 1                # double bonds: each C at 4 -- saturated
    edges[1, 0, 2, 1] = edges[1, 2, 0, 1] = 0
    edges[1, 0, 2, 0] = edges[1, 2, 0, 0] = 1                        # one single bond: C0 and C2 at 3
    n = torch.tensor([3, 3], dtype=torch.int32, device="cuda")
    logits = torch.zeros(2, apd, device="cuda")
    m.apply(2, logits, n, _stream(), torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda(), int8=True,
            first_slot=0)
    row = torch.isneginf(logits).cpu().numpy()
    assert row[0, :-1].all() and not row[0, -1]                      # a dead end: terminate stays
    assert row[1, -1] and not row[1, :-1].all()                      # an add survives: terminate is masked
    flags = m.check(torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda(), n).cpu().numpy()
    assert flags.tolist() == [R.DEAD_END, R.UNDER_MIN]


# ---- 2. the molecule check --------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES[:5])
@pytest.mark.parametrize("mode", ["structure", "valence"])
def test_check_matches_the_restatement(case, mode):
    N, A, CH, H, C, Ef = case
    rng = np.random.default_rng(100 + CASES.index(case) + 50 * (mode == "valence"))
    B = 41
    V = rng.integers(1, 5, (A, CH)) if mode == "valence" else None
    cons = _random_set(rng, N, A, CH, Ef, min(N, 8))
    m, apd = _mask(N, A, CH, H, C, Ef, mode, V, cons)
    t = R.table_dict(m.cons_table.cpu().numpy(), A, CH, Ef)
    nodes, edges, n = _ring_states(rng, B, N, A, CH, H, C, Ef)
    for dt in (torch.float32, torch.int8):
        nd, ed = torch.from_numpy(nodes).cuda().to(dt), torch.from_numpy(edges).cuda().to(dt)
        for cnt in (torch.from_numpy(n).cuda(), None):
            got = m.check(nd, ed, cnt).cpu().numpy()
            for b in range(B):
                want = R.check(t, nodes[b], edges[b], int(n[b]), N, A, CH, H, C, Ef, V, m.bond_orders, m.imp_h)
                assert got[b] == want, (b, int(n[b]), int(got[b]), want)


# ---- 3. off means off --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["structure", "valence"])
def test_off_set_equals_the_unconstrained_launch(mode):
    from graphinvent_b200.generation import Constraints
    N, A, CH, H, C, Ef = 13, 5, 3, 0, 0, 3
    rng = np.random.default_rng(7)
    V = rng.integers(1, 5, (A, CH)) if mode == "valence" else None
    plain, apd = _mask(N, A, CH, H, C, Ef, mode, V)
    off, _ = _mask(N, A, CH, H, C, Ef, mode, V, Constraints())
    assert off.constraints.off
    nodes, edges, n = _ring_states(rng, 300, N, A, CH, H, C, Ef)
    nd, ed, nn = (torch.from_numpy(x).cuda() for x in (nodes, edges, n))
    x = torch.randn(300, apd, device="cuda")
    a, b = x.clone(), x.clone()
    plain.apply(300, a, nn, _stream(), nd, ed, int8=True, first_slot=0)
    off.apply(300, b, nn, _stream(), nd, ed, int8=True, first_slot=0)
    assert torch.equal(a, b)


# ---- 4. generation with the pretrained gdb13 GGNN ----------------------------------------------------------------
def _pretrained_or_seeded():
    """the reference's pretrained gdb13 GGNN, or the seeded GGNN the tools fall back to without it"""
    try:
        return _pretrained()
    except pytest.skip.Exception:
        from graphinvent_b200.config import make_constants
        from tests.test_gpu_generation_layouts import _seeded_model
        C = make_constants("GGNN")
        net, _ = _seeded_model("GGNN", C, 1)
        return C, net.eval()


# atoms=(13, 13) cannot finish a batch: B - 1 slots make B molecules, so one slot makes two of at least 14 rounds
# each, past the 2N = 26-round limit (the batch raises, as any batch over the limit does)
SETS = [dict(atoms=(10, 10)), dict(atom_types={"N": (None, 2), "O": (None, 2), "S": (0, 0), "Cl": (0, 0)}, bonds={"TRIPLE": 0}),
        dict(rings=(0, 2), min_ring_size=5), dict(atoms=(8, 11), rings=(1, None), charges={1: 0, -1: 0})]


@pytest.mark.parametrize("spec", SETS)
def test_generated_molecules_respect_the_set(spec):
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained_or_seeded()
    B = 1000
    cons = Constraints(**spec, constants=GDB13)
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, constraints=cons)
    assert gen.action_mask.mode == "structure"                       # constraints bring the structural rule
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(5), device="cuda")
    gen.build_graphs(uniforms=U)
    pt = gen.properly_terminated[:B].cpu().numpy()
    assert (pt == 1).all()                                           # the structural rule: no invalid action
    flags = gen.constraints.check(gen.generated_nodes[:B], gen.generated_edges[:B],
                                  gen.generated_n_nodes[:B]).cpu().numpy()
    assert not (flags & (R.OVER_MAX | R.SMALL_RING | R.UNDER_MIN)).any(), np.unique(flags)
    if spec == SETS[0]:
        nn_ = gen.generated_n_nodes[:B].cpu().numpy()
        assert ((nn_ == 10) | ((flags & R.DEAD_END) != 0)).all()
        assert (nn_ == 10).mean() > 0.5


def _eager(model, C, B, U, **kw):
    """the eager generator's round loop on uniforms U, the model in capacity mode at the captured capacity"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import entry_capacity
    gen = GraphGenerator(model, B, constants=C, n_atom_types=5, n_formal_charge=3, **kw)
    st, n, rnd = _stream(), 0, 0
    model.entry_capacity = entry_capacity(B, gen.N, gen.Ef)
    try:
        with torch.no_grad():
            while n < B:
                assert rnd < 2 * gen.N
                out = model(*gen._model_inputs(model)).contiguous()
                gen._mask(out, st)
                action, lik = Fn.sample_actions(out, uniforms=U[rnd], **gen._policy_kw())
                gen._round(rnd, action, lik, st)
                n = int(gen._counters[0].item())
                rnd += 1
    finally:
        model.entry_capacity = None
    gen.rounds = rnd
    return gen


@pytest.mark.parametrize("kw", [dict(), dict(action_mask="valence", temperature=1.3, top_k=10, top_p=0.9)])
def test_captured_equals_eager(kw):
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained_or_seeded()
    kw = dict(kw)
    if kw.get("action_mask") == "valence":
        kw["max_valence"] = _gdb13_valence()
    cons = Constraints(atoms=(9, 12), atom_types={"N": (1, None)}, min_ring_size=5, constants=GDB13)
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(8), device="cuda")
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, constraints=cons, **kw)
    gen.build_graphs(uniforms=U)
    eager = _eager(net, C, B, U, constraints=cons, **kw)
    assert eager.rounds == gen.rounds
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name


def test_set_constraints_reuses_the_captured_round():
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained_or_seeded()
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(9), device="cuda")
    a, b = Constraints(atoms=(10, 12), constants=GDB13), Constraints(atoms=(5, 7), constants=GDB13)
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, constraints=a)
    gen.build_graphs(uniforms=U)
    graph = gen.graph
    gen.set_constraints(b)
    assert gen.constraints == b and gen.constraints_version == 1
    gen.build_graphs(uniforms=U)
    assert gen.graph is graph                                        # no recapture
    fresh = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, constraints=b)
    fresh.build_graphs(uniforms=U)
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), getattr(fresh, name)), name
    nn_ = gen.generated_n_nodes[:B].cpu().numpy()
    flags = gen.constraints.check(gen.generated_nodes[:B], gen.generated_edges[:B],
                                  gen.generated_n_nodes[:B]).cpu().numpy()
    assert ((nn_ <= 7) & ((nn_ >= 5) | ((flags & R.DEAD_END) != 0))).all()
    # built without constraints: the first set_constraints captures once more, and the result is the constrained one
    plain = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    plain.build_graphs(uniforms=U)
    plain.set_constraints(b)
    assert plain.graph is None
    plain.build_graphs(uniforms=U)
    for name in GEN_STATE:
        assert torch.equal(getattr(plain, name), getattr(fresh, name)), name


# ---- 5. RL -----------------------------------------------------------------------------------------------------
def test_rl_rollout_and_backward_match_eager():
    from graphinvent_b200.generation import Constraints, GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from tests.test_gpu_generation_layouts import _seeded_model
    from tests.test_gpu_rl_graphed import _loss
    C, agent = _pretrained_or_seeded()
    prior, _ = _seeded_model("GGNN", C, 2)
    B = 96
    cons = Constraints(atoms=(8, 12), atom_types={"O": (1, None)}, rings=(0, 2), min_ring_size=5, constants=GDB13)
    gen = GraphedGeneratorRL(agent, B, n_atom_types=5, n_formal_charge=3, constraints=cons)
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(3), device="cuda")
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    R_ = gen.rounds
    p_a, p_b, acts = gen.p_a[:R_].clone(), gen.p_b[:R_].clone(), gen.act_rec[:R_].clone()
    agent.zero_grad()
    prior.zero_grad()
    _loss(agent_ll, prior_ll).backward()
    assert gen.backward_rounds == [R_, R_]
    assert torch.equal(gen.recomputed_p[0][:R_], p_a) and torch.equal(gen.recomputed_p[1][:R_], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eager = GraphGeneratorRL(agent2, B, n_atom_types=5, n_formal_charge=3, constraints=cons)
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eager.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert eager.rounds == R_
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eager, name)), name
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        assert total > 0
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total
    # a set_constraints between a rollout and its backward
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    gen.set_constraints(Constraints(atoms=(5, 9)))
    with pytest.raises(RuntimeError, match="set_constraints"):
        _loss(agent_ll, prior_ll).backward()


# ---- 6. the route scorer ---------------------------------------------------------------------------------------
def test_route_scorer_scores_under_the_constraints_and_refuses_probability_zero():
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator, RouteScorer
    from tests import route_nll_reference as RN
    C, net = _pretrained_or_seeded()
    cons = Constraints(atoms=(9, 12), rings=(0, 2), min_ring_size=5, constants=GDB13)
    B = 256
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, constraints=cons)
    gen.build_graphs(generator=torch.Generator("cuda").manual_seed(4))
    nodes, edges = gen.generated_nodes[:B].to(torch.int8), gen.generated_edges[:B].to(torch.int8)
    flags = gen.constraints.check(nodes, edges).cpu().numpy()
    keep = np.flatnonzero(flags == 0)[:64]
    nodes, edges = nodes[keep], edges[keep]
    scorer = RouteScorer(net, 300, n_atom_types=5, n_formal_charge=3, constraints=cons)
    out = scorer.score(nodes, edges)
    # fp64: each route state's masked softmax under the restated rule
    from tests import preprocess_reference as P
    t = R.table_dict(scorer.action_mask.cons_table.cpu().numpy(), 5, 3, 3)
    X, E, acts, off = RN.build_order_states(nodes.cpu().numpy(), edges.cpu().numpy(), P.segments(5, 3))
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    _, logits = RN.probabilities(sd, C, X, E, acts)
    logits = logits.numpy()
    want = np.zeros(len(acts))
    for s in range(len(acts)):
        f = R.mask(t, X[s], E[s], int(X[s].any(-1).sum()), 13, 5, 3, 0, 0, 3)
        assert not f[acts[s]]
        z = np.where(f, -np.inf, logits[s])
        z = np.exp(z - z.max())
        want[s] = z[acts[s]] / z.sum()
    assert out.offsets.cpu().numpy().tolist() == off.tolist()
    got = out.likelihoods.double().cpu().numpy()
    assert np.abs(np.log(got) - np.log(want)).max() < 1e-3
    # gradients: score(requires_grad) and backward run under the same mask, and change with set_constraints raises
    net.zero_grad()
    sc = scorer.score(nodes, edges, requires_grad=True)
    sc.nll.sum().backward()
    assert sum(p.grad.norm().item() for p in net.parameters()) > 0
    sc = scorer.score(nodes, edges, requires_grad=True)
    scorer.set_constraints(Constraints(atoms=(9, 12), constants=GDB13))
    with pytest.raises(RuntimeError, match="set_constraints"):
        sc.nll.sum().backward()
    # a molecule over a maximum is refused by name
    tight = RouteScorer(net, 300, n_atom_types=5, n_formal_charge=3,
                        constraints=Constraints(atoms=(None, 9), constants=GDB13))
    big = int(np.flatnonzero((nodes.cpu().numpy() != 0).any(-1).sum(-1) > 9)[0])
    with pytest.raises(ValueError, match=f"molecule {big} .*probability 0"):
        tight.score(nodes, edges)


def test_route_scorer_gradients_match_an_unconstrained_scorer_where_nothing_is_masked():
    """an off set scores and differentiates bit for bit as the structural mask alone"""
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator, RouteScorer
    C, net = _pretrained_or_seeded()
    gen = GraphedGenerator(net, 128, n_atom_types=5, n_formal_charge=3, action_mask="structure")
    gen.build_graphs(generator=torch.Generator("cuda").manual_seed(6))
    nodes, edges = gen.generated_nodes[:128].to(torch.int8), gen.generated_edges[:128].to(torch.int8)
    grads = []
    for cons in (None, Constraints()):
        scorer = RouteScorer(net, 300, n_atom_types=5, n_formal_charge=3, action_mask="structure", constraints=cons)
        net.zero_grad()
        out = scorer.score(nodes, edges, requires_grad=True)
        out.nll.sum().backward()
        grads.append((out.nll.detach().clone(), [p.grad.clone() for p in net.parameters()]))
    assert torch.equal(grads[0][0], grads[1][0])
    for g0, g1 in zip(grads[0][1], grads[1][1]):
        assert torch.equal(g0, g1)


# ---- 7. buffers and determinism -------------------------------------------------------------------------------
def test_kernels_stay_inside_their_buffers():
    from graphinvent_b200._lib import check, lib
    N, A, CH, H, C, Ef = 13, 5, 3, 0, 0, 3
    rng = np.random.default_rng(21)
    B = 67
    cons = _random_set(rng, N, A, CH, Ef, 8)
    m, apd = _mask(N, A, CH, H, C, Ef, "valence", rng.integers(1, 5, (A, CH)), cons)
    nodes, edges, n = _ring_states(rng, B, N, A, CH, H, C, Ef)
    g_nodes, g_edges = Guarded.like(torch.from_numpy(nodes).cuda()), Guarded.like(torch.from_numpy(edges).cuda())
    g_n, g_tab = Guarded.like(torch.from_numpy(n).cuda()), Guarded.like(m.cons_table)
    g_val = Guarded.like(m.table)
    x = torch.randn(B, apd, device="cuda")
    g_x = Guarded.like(x)
    before = [g.raw.clone() for g in (g_nodes, g_edges, g_n, g_tab, g_val)]
    p = lambda g: ctypes.c_void_p(g.ptr())
    st = _stream()
    check(lib.gib_action_mask_logits_constrained(B, N, A + CH, Ef, A, CH, H, C, apd, 2, p(g_val), None, None,
                                                 p(g_nodes), p(g_edges), p(g_n), None, None, None, None, None,
                                                 p(g_x), 0, st, p(g_tab)), "gib_action_mask_logits_constrained")
    flags = Guarded(4 * B)
    check(lib.gib_constraints_check(B, N, A + CH, Ef, A, CH, H, C, 2, p(g_val), None, None, p(g_nodes), p(g_edges),
                                    p(g_n), None, None, p(g_tab), p(flags), st), "gib_constraints_check")
    torch.cuda.synchronize()
    for g, b0 in zip((g_nodes, g_edges, g_n, g_tab, g_val), before):
        assert torch.equal(g.raw, b0)
    assert g_x.intact(), g_x.damage()
    assert flags.intact(), flags.damage()
    y = x.clone()
    m.apply(B, y, torch.from_numpy(n).cuda(), st, torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda(),
            int8=True, first_slot=0)
    assert torch.equal(g_x.view(torch.float32, (B, apd)), y)
    assert torch.equal(flags.view(torch.int32, (B,)),
                       m.check(torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda(),
                               torch.from_numpy(n).cuda()))


def test_replays_are_deterministic():
    from graphinvent_b200.generation import Constraints
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _pretrained_or_seeded()
    B = 256
    U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(19), device="cuda")
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3, temperature=0.9,
                           constraints=Constraints(atoms=(9, None), min_ring_size=5, constants=GDB13))
    gen.build_graphs(uniforms=U)
    keep = {name: getattr(gen, name).clone() for name in GEN_STATE}
    gen.build_graphs(uniforms=U)
    for name in GEN_STATE:
        assert torch.equal(getattr(gen, name), keep[name]), name


def test_setter_refuses_bad_tables_before_any_launch():
    from graphinvent_b200._lib import lib
    from tests.constraints_reference import off_values
    A, CH, Ef, N = 5, 3, 3, 13
    tab = torch.zeros(8 + 2 * A + CH + Ef, dtype=torch.int32, device="cuda")
    for edit in ({1: 14}, {0: 5, 1: 4}, {4: 2}, {4: 1}, {2: 3, 3: 2}, {8: -1}, {8 + A: -2}, {8: 7, 9: 7, 1: 12},
                 {0: 14}):
        v = off_values(A, CH, Ef)
        for k, x in edit.items():
            v[k] = x
        assert lib.gib_constraints_set(ctypes.c_void_p(tab.data_ptr()), v.ctypes.data_as(ctypes.c_void_p), N, A, CH,
                                       Ef, _stream()) != 0, edit
    v = off_values(A, CH, Ef)
    assert lib.gib_constraints_set(None, v.ctypes.data_as(ctypes.c_void_p), N, A, CH, Ef, _stream()) != 0
    assert lib.gib_constraints_set(ctypes.c_void_p(tab.data_ptr()), None, N, A, CH, Ef, _stream()) != 0
    assert lib.gib_constraints_set(ctypes.c_void_p(tab.data_ptr()), v.ctypes.data_as(ctypes.c_void_p), N, A, CH, Ef,
                                   _stream()) == 0
    got = tab.cpu().numpy()
    assert got[5:8].tolist() == [A, CH, Ef]
