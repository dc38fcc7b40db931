"""GPU: scaffold decoration (generation.ScaffoldTable, include/gib200.h `gib_scaffolds`).

The round kernels with the scaffold reset against the scaffold oracle (tests/scaffold_oracle.py) on random action
streams in the gdb13 layout and in L3; the attachment mask over a batch of 1000 with a seeded model; the captured
generator against the eager one, bit for bit, across an in-place `set_scaffolds` and one that recaptures; the
scaffold refusals; the unchanged default."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import molecules_reference as MR
from tests import scaffold_oracle as SO
from tests.conftest import ROOT
from tests.test_gpu_molecules import check_batch, ref  # noqa: F401  (the reference fixture)
from tests.test_gpu_generation_layouts import _layout_constants, _layout_stream, _seeded_model

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden")
N, A, CH, EF = 13, 5, 3, 3
STATE = ("nodes", "edges", "n_nodes", "likelihoods", "generated_nodes", "generated_edges", "generated_n_nodes",
         "generated_likelihoods", "properly_terminated")


def gdb13_scaffolds(sizes=(1, 2, 4, 6, 9, 12)):
    """int8 (nodes [S, 13, 8], edges [S, 13, 13, 3]): one decoding-route state of gdb13_1K per atom count in `sizes`,
    taken from the first 256 training rows (real partial molecules, in route order); 12 = N - 1"""
    from graphinvent_b200 import data
    nodes, edges, _ = data.read_hdf5_raw(os.path.join(GOLDEN, "gdb13_train_head256.h5"), N, 8, EF, 625)
    k = (nodes != 0).any(-1).sum(-1)
    rows = [int(np.flatnonzero(k == s)[0]) for s in sizes]
    return nodes[rows].copy(), edges[rows].copy()


def with_segments(nodes, H, C):
    """gdb13 scaffolds widened to the L1-L3 node features: implicit-H and chirality index 0 on every atom"""
    atoms = (nodes != 0).any(-1, keepdims=True)
    extra = [np.concatenate([atoms, np.zeros(atoms.shape[:-1] + (w - 1,), bool)], -1) for w in (H, C) if w]
    return np.concatenate([nodes] + [e.astype(np.int8) for e in extra], -1)


def attachment_lists(nodes, seed=0):
    """a seeded choice of attachment points per scaffold: at least one (the last atom), some scaffolds more"""
    rng = np.random.default_rng(seed)
    k = (nodes != 0).any(-1).sum(-1)
    return [sorted({int(n - 1)} | {int(i) for i in np.flatnonzero(rng.random(n) < 0.3)}) for n in k]


def _gdb13_constants(n=N):
    return _layout_constants(n, A, CH, 0, 0, EF)


def _round(gen, rnd, a, lik):
    gen._round(rnd, a, lik, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("seed,H,C,B", [(0, 0, 0, 200), (1, 4, 3, 200), (2, 0, 0, 37), (3, 4, 0, 96)])
def test_scaffold_rounds_match_the_oracle_on_random_action_streams(seed, H, C, B):
    """the state after every round, then the finished buffers and generated_scaffolds, starting from gdb13 route
    states (one single-atom scaffold, one with N - 1 atoms)"""
    from graphinvent_b200.generation import GraphGenerator
    sn, se = gdb13_scaffolds()
    sn = with_segments(sn, H, C)
    rng = np.random.default_rng(seed)
    st = SO.ScaffoldState(B, N, A, CH, EF, H, C, sn, se)
    gen = GraphGenerator(None, B, constants=_layout_constants(N, A, CH, H, C, EF), scaffolds=(sn, se))
    assert (gen.n_nodes.cpu().numpy() == st.n_nodes).all() and (gen.nodes.cpu().numpy() == st.nodes).all()
    for rnd in range(2 * N - 1):
        if st.n_generated > B:
            break
        a, _ = _layout_stream(rng, st)
        lik = rng.random(B).astype(np.float32)
        SO.generation_round(st, rnd, a, lik)
        _round(gen, rnd, torch.from_numpy(a).cuda(), torch.from_numpy(lik).cuda())
        for name in ("nodes", "edges", "n_nodes", "likelihoods"):
            assert (getattr(gen, name).cpu().numpy() == getattr(st, name)).all(), (rnd, name)
        assert int(gen._counters[0]) == st.n_generated
        assert (gen._slot_ids.cpu().numpy() == st.slot_ids).all() and int(gen._started) == st.started
    for name in STATE[4:]:
        assert (getattr(gen, name).cpu().numpy() == getattr(st, name)).all(), name
    assert (gen._gen_scaffolds.cpu().numpy() == st.generated_scaffolds).all()
    assert st.n_generated > B // 4 and len(set(st.generated_scaffolds[:st.n_generated].tolist())) == len(sn)


def _forbidden(logits_shape, per_node, k, protect, slot_ids, n_nodes):
    """vectorised scaffold_oracle.forbidden over a batch: bool [B, apd]"""
    B, apd = logits_shape
    len_add = N * per_node
    m = np.zeros((B, apd), bool)
    for b in range(1, B):
        s = int(slot_ids[b])
        for i in np.flatnonzero(protect[s][:k[s]]):
            m[b, i * per_node:(i + 1) * per_node] = True
            m[b, len_add + i * EF:len_add + (i + 1) * EF] = True
        if n_nodes[b] - 1 < k[s]:
            m[b, len_add:len_add + N * EF] = True
    return m


def test_attachment_mask_over_a_batch_of_1000(monkeypatch):
    """no forbidden action is drawn, each recorded likelihood is the masked softmax in fp64 to fp32 rounding, every
    molecule keeps its scaffold in rows 0..k-1, and protected atoms gain no bond"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    sn, se = gdb13_scaffolds()
    att = attachment_lists(sn)
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 3)
    B = 1000
    gen = GraphGenerator(net.eval(), B, constants=C, scaffolds=(sn, se), attachment=att)
    k = gen.scaffolds.n_atoms
    protect = SO.protect_of(k, att, N)
    rounds = []
    net.register_forward_pre_hook(lambda m, i: rounds.append([gen._slot_ids.cpu().numpy(), gen.n_nodes.cpu().numpy()]))
    net.register_forward_hook(lambda m, i, o: rounds[-1].append(o.detach().double().cpu().numpy()))
    real = Fn.sample_actions

    def record(out, **kw):
        a, lik = real(out, **kw)
        rounds[-1] += [a.cpu().numpy(), lik.cpu().numpy()]
        return a, lik
    monkeypatch.setattr(Fn, "sample_actions", record)
    (nodes, edges, n_nodes), flat, final, proper = gen.sample(generator=torch.Generator("cuda").manual_seed(0))
    per_node = A * CH * EF
    drawn_masked = 0
    for ids, n, logits, a, lik in rounds:
        m = _forbidden(logits.shape, per_node, k, protect, ids, n)
        assert not m[np.arange(1, B), a[1:]].any()
        drawn_masked += int(m[1:].any(1).sum())
        x = np.where(m, -np.inf, logits)
        p = np.exp(x - x.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        want = p[np.arange(B), a]
        assert np.allclose(lik[1:], want[1:], rtol=1e-5, atol=0)
    assert drawn_masked > 0
    ids = gen.generated_scaffolds.cpu().numpy()
    assert ids.shape == (B,) and (ids >= 0).all()
    nodes, edges = nodes.cpu().numpy(), edges.cpu().numpy()
    for p in range(B):
        s, ks = ids[p], k[ids[p]]
        assert (nodes[p, :ks] == sn[s, :ks]).all()
        assert (edges[p, :ks, :ks] == se[s, :ks, :ks]).all()
        for i in np.flatnonzero(protect[s][:ks]):
            assert (edges[p, i] == se[s, i]).all(), (p, i)
    assert torch.isfinite(final).all()


def test_scaffold_molecules_convert(ref):
    """decorated molecules go through MoleculeBatch / generation_graphs as the reference's graph_to_graph reads them"""
    from graphinvent_b200.generation import GraphGenerator
    sn, se = gdb13_scaffolds()
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 4)
    gen = GraphGenerator(net.eval(), 64, constants=C, scaffolds=(sn, se), attachment=attachment_lists(sn))
    (nodes, edges, n_nodes), flat, final, term = gen.sample(generator=torch.Generator("cuda").manual_seed(1))
    assert (n_nodes.cpu().numpy() >= gen.scaffolds.n_atoms[gen.generated_scaffolds.cpu().numpy()]).all()
    check_batch(ref, nodes, edges, n_nodes, MR.constants("L0", device="cuda"), term=term)


def _eager(model, C, B, U, sc, att):
    """the eager generator's loop on given uniforms, the model in capacity mode at the captured generator's capacity"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import scaffold_entry_capacity
    gen = GraphGenerator(model, B, constants=C, scaffolds=sc, attachment=att)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    model.entry_capacity = scaffold_entry_capacity(B, gen.N, gen.Ef, gen.scaffolds.m_max)
    n, rnd = 0, 0
    try:
        with torch.no_grad():
            while n < B:
                out = model(*gen._model_inputs(model)).contiguous()
                if gen.masked:
                    gen._mask(out, st)
                action, lik = Fn.sample_actions(out, uniforms=U[rnd])
                gen._round(rnd, action, lik, st)
                n = int(gen._counters[0].item())
                rnd += 1
    finally:
        model.entry_capacity = None
    gen.rounds = rnd
    return gen


@pytest.mark.parametrize("masked", [False, True])
def test_captured_scaffold_generation_equals_the_eager_loop(masked):
    from graphinvent_b200.graphed import GraphedGenerator, scaffold_entry_capacity
    sn, se = gdb13_scaffolds()
    att = attachment_lists(sn) if masked else None
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 5)
    net.eval()
    B = 300
    graphed = GraphedGenerator(net, B, constants=C, scaffolds=(sn, se), attachment=att)
    assert graphed.entry_capacity == scaffold_entry_capacity(B, N, EF, graphed.scaffolds.m_max)
    g = torch.Generator(device="cuda").manual_seed(7)
    sets = [(sn, se, att),
            (sn[::-1].copy(), se[::-1].copy(), att[::-1] if masked else None),       # in place: same S and m_max
            (sn[:4].copy(), se[:4].copy(), att[:4] if masked else None)]            # another S: recaptured
    for i, (n_, e_, a_) in enumerate(sets):
        if i:
            before = graphed.graph
            graphed.set_scaffolds((n_, e_), a_)
            assert (graphed.graph is before) == (i == 1)
        U = torch.rand(2 * N, B, generator=g, device="cuda")
        got = graphed.build_graphs(uniforms=U)
        eager = _eager(net, C, B, U, (n_, e_), a_)
        assert got == int(eager._counters[0]) and graphed.rounds == eager.rounds
        for name in STATE:
            assert torch.equal(getattr(graphed, name), getattr(eager, name)), (i, name)
        assert torch.equal(graphed.generated_scaffolds, eager._gen_scaffolds[:B]), i


def test_default_is_unchanged_after_scaffolds_are_dropped():
    """set_scaffolds(None) returns the captured generator to the plain one: the same bits as a generator that never
    had scaffolds"""
    from graphinvent_b200.graphed import GraphedGenerator, entry_capacity
    sn, se = gdb13_scaffolds()
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 6)
    net.eval()
    B = 128
    plain = GraphedGenerator(net, B, constants=C)
    was = GraphedGenerator(net, B, constants=C, scaffolds=(sn, se))
    U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(3), device="cuda")
    was.build_graphs(uniforms=U)
    was.set_scaffolds(None)
    assert was.entry_capacity == entry_capacity(B, N, EF) and was.generated_scaffolds is not None
    plain.build_graphs(uniforms=U)
    was.build_graphs(uniforms=U)
    assert was.generated_scaffolds is None
    for name in STATE:
        assert torch.equal(getattr(plain, name), getattr(was, name)), name


@pytest.mark.parametrize("case", ["not_one_hot", "gap", "asymmetric", "two_types", "disconnected", "empty",
                                  "too_many_atoms"])
def test_malformed_scaffolds_are_refused_by_name(case):
    from graphinvent_b200.generation import GraphGenerator
    sn, se = gdb13_scaffolds()
    sn, se = sn.copy(), se.copy()
    s = 3                                           # 6 atoms
    if case == "not_one_hot":
        sn[s, 1, 0:2] = 1
    elif case == "gap":
        sn[s, 6] = sn[s, 5]
        sn[s, 5] = 0
    elif case == "asymmetric":
        i, j = np.argwhere(se[s].any(-1))[0]
        se[s, i, j] = 0
    elif case == "two_types":
        i, j = np.argwhere(se[s].any(-1))[0]
        se[s, i, j] = se[s, j, i] = 1
    elif case == "disconnected":
        se[s, :, 5] = 0
        se[s, 5, :] = 0
    elif case == "empty":
        sn[s] = 0
        se[s] = 0
    C = _gdb13_constants()
    if case == "too_many_atoms":
        C = _gdb13_constants(8)
        with pytest.raises(ValueError, match="scaffold 4 holds 9 atoms"):
            GraphGenerator(None, 8, constants=C, scaffolds=(sn, se))
        return
    with pytest.raises(ValueError, match=f"invalid scaffold.*molecule {s}"):
        GraphGenerator(None, 8, constants=C, scaffolds=(sn, se))


# ---- the reference generator's scaffold traces ----------------------------------------------------------------
@pytest.mark.parametrize("name", ["L0", "L0_attach", "L3", "L3_attach"])
def test_replay_reproduces_the_reference_scaffold_traces_bit_exactly(name):
    """eager GraphGenerator(scaffolds=) replaying the reference's recorded draws: every buffer, generated_scaffolds
    included"""
    from graphinvent_b200.generation import GraphGenerator
    from tests.test_generation_layouts import assert_matches_trace
    from tests.test_scaffold_generation_host import scaffold_trace
    z = scaffold_trace(name)
    H, C = int(z["n_imp_H"]), int(z["n_chirality"])
    sn, se = z["scaffold_nodes"], z["scaffold_edges"]
    k = (sn != 0).any(-1).sum(-1)
    att = (np.arange(N)[None] < k[:, None]) & ~z["protect"] if bool(z["attachment"]) else None
    gen = GraphGenerator(None, int(z["batch"]), constants=_layout_constants(N, A, CH, H, C, EF), scaffolds=(sn, se),
                         attachment=att)
    if att is not None:
        assert (gen.scaffolds.protect_mask == z["protect"]).all()
    got = gen.build_graphs(replay=[(torch.from_numpy(a.astype(np.int32)), torch.from_numpy(lk))
                                   for a, lk in zip(z["actions"], z["likelihoods"])])
    assert got == int(z["n_generated"]) and gen.rounds == int(z["rounds"])
    assert_matches_trace(z, *(t.cpu().numpy() for t in (gen.generated_nodes, gen.generated_edges,
                                                        gen.generated_n_nodes, gen.generated_likelihoods,
                                                        gen.properly_terminated, gen.nodes, gen.edges, gen.n_nodes,
                                                        gen.likelihoods)))
    assert (gen._gen_scaffolds.cpu().numpy() == z["generated_scaffolds"]).all()
    assert (gen.generated_scaffolds.cpu().numpy() == z["generated_scaffolds"][:int(z["batch"])]).all()
    assert (gen._slot_ids.cpu().numpy() == z["final_slot_ids"]).all() and int(gen._started) == int(z["started"])


# ---- the entry capacity's worst case --------------------------------------------------------------------------
def _worst_case_actions(B, sn, se, rounds):
    """[rounds, B] actions that add a bond in every slot whenever one can be added: the dummy slot adds onto a new
    (bond_to, bond type) pair each round; a scaffold slot adds an atom onto atom 0 until the graph is full, then
    connects its newest atom to the lowest atom it is not bonded to, and terminates only when no bond is left (it
    restarts from the scaffold).  Returns the actions and the most bond entries any model call of the captured
    generator sees: the state before each round and after the last one"""
    st = SO.ScaffoldState(B, N, A, CH, EF, 0, 0, sn, se)
    per_node = A * CH * EF
    len_add = N * per_node
    acts, peak = [], int((st.edges != 0).sum())
    for r in range(rounds):
        if st.n_generated >= B:
            break
        a = np.full(B, len_add + N * EF, np.int32)                # terminate
        a[0] = (r % N) * per_node + (r // N) % EF
        for b in range(1, B):
            n = int(st.n_nodes[b])
            if n < N:
                a[b] = 0
                continue
            free = [j for j in range(n - 1) if st.edges[b, j, n - 1].sum() == 0]
            if free:
                a[b] = len_add + free[0] * EF
        SO.generation_round(st, r, a, np.ones(B, np.float32))
        acts.append(a)
        peak = max(peak, int((st.edges != 0).sum()))
    return np.stack(acts), peak


def test_entry_capacity_holds_the_scripted_worst_case():
    """the largest scaffold in every slot, then only bond-adding actions, through the captured rollout (recorded
    actions, K0 in capacity mode): no overflow at scaffold_entry_capacity, which no real batch can reach (a slot can
    only connect its newest atom, so it cannot add a bond in every one of 2N rounds); the overflow is raised at the
    peak the script reaches minus one"""
    from graphinvent_b200.graphed import GraphedGeneratorRL, scaffold_entry_capacity
    sn, se = gdb13_scaffolds(sizes=(12,))
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 8)
    B = 64
    acts, peak = _worst_case_actions(B, sn, se, 2 * N)
    gen = GraphedGeneratorRL(net, B, constants=C, scaffolds=(sn, se))
    bound = scaffold_entry_capacity(B, N, EF, int(se[0].sum()) // 2)
    assert gen.entry_capacity == bound and peak <= bound
    with torch.no_grad():
        gen.sample(net, net, actions=torch.from_numpy(acts).cuda())
    assert gen.rounds == acts.shape[0]
    gen._set_capacity(peak)
    gen._invalidate_graphs()
    with torch.no_grad():
        gen.sample(net, net, actions=torch.from_numpy(acts).cuda())      # exactly the peak fits
    gen._set_capacity(peak - 1)
    gen._invalidate_graphs()
    with pytest.raises(RuntimeError, match="bond entries"), torch.no_grad():
        gen.sample(net, net, actions=torch.from_numpy(acts).cuda())


# ---- scaffolds=None: the same bits as a generator built before scaffolds existed ------------------------------
def test_default_generators_are_unchanged_by_a_scaffold_round_trip():
    """each of the four generators after set_scaffolds(table) then set_scaffolds(None) equals a fresh one"""
    from graphinvent_b200.generation import GraphGenerator, GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    sn, se = gdb13_scaffolds()
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 9)
    net.eval()
    B = 64
    U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(5), device="cuda")
    for cls in (GraphGenerator, GraphGeneratorRL, GraphedGeneratorRL):
        fresh, was = cls(net, B, constants=C), cls(net, B, constants=C, scaffolds=(sn, se))
        was.set_scaffolds(None)
        assert was.scaffolds is None
        outs = []
        for gen in (fresh, was):
            with torch.no_grad():
                if cls is GraphGenerator:
                    outs.append(gen.sample(generator=torch.Generator("cuda").manual_seed(2)))
                elif cls is GraphGeneratorRL:
                    outs.append(gen.sample(net, net, generator=torch.Generator("cuda").manual_seed(2)))
                else:
                    outs.append(_run_or_error(lambda: gen.sample(net, net, uniforms=U)))
            assert gen.generated_scaffolds is None
        for name in STATE:
            assert torch.equal(getattr(fresh, name), getattr(was, name)), (cls.__name__, name)


def _run_or_error(fn):
    try:
        return fn()
    except RuntimeError as e:
        return e
