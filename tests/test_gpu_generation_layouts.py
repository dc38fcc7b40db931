"""The implicit-H and chirality action layouts of the device generator (reference parameters/constants.py:23-95).

The round kernels behind `gib_generation_round_layout` against the reference's own traces
(tests/golden/generation_layout_traces.npz) and against the layout oracle (tests/generation_layout_oracle.py) on
synthetic action streams; the generators and the models at these node-feature widths end to end."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_generation_layouts import A, CH, EF, LAYOUTS, N, _constants, _trace, assert_matches_trace


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _run_round(gen, rnd, a, lik, H, C, entry="layout"):
    """one round through the C-ABI on the generator's buffers"""
    from graphinvent_b200._lib import check, lib
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    bufs = (_ptr(a), _ptr(lik), _ptr(gen.nodes), _ptr(gen.edges), _ptr(gen.n_nodes), _ptr(gen.likelihoods),
            _ptr(gen.generated_nodes), _ptr(gen.generated_edges), _ptr(gen.generated_n_nodes),
            _ptr(gen.generated_likelihoods), _ptr(gen.properly_terminated), gen.capacity, _ptr(gen._counters),
            _ptr(gen._scratch), st)
    if entry == "layout":
        check(lib.gib_generation_round_layout(gen.batch_size, gen.N, gen.F, gen.Ef, gen.A, gen.CH, H, C, rnd, *bufs),
              "gib_generation_round_layout")
    else:
        check(lib.gib_generation_round(gen.batch_size, gen.N, gen.F, gen.Ef, gen.A, gen.CH, rnd, *bufs),
              "gib_generation_round")


def _layout_stream(rng, st):
    """like tests/test_generation.py::_action_stream, with every add index drawn uniformly inside its node's block
    (atom, charge, implicit H, chirality, bond type): adds bond to an existing atom, so graphs grow to max_n_nodes and
    the next add goes into a full graph; the remaining 0.6/N of the draws are connects among existing atoms,
    connects to a random position, terminates and uniformly random indices"""
    from tests.generation_layout_oracle import add_dims
    B, N_, Ef = st.B, st.N, st.Ef
    per_node = int(np.prod(add_dims(st)[1:]))
    len_add = N_ * per_node
    apd = len_add + N_ * Ef + 1
    q = 0.6 / N_
    u = rng.random(B)
    n = st.n_nodes
    bond_to = np.where(n > 0, rng.integers(0, 1 << 30, B) % np.maximum(n, 1), 0)
    add = bond_to * per_node + rng.integers(0, per_node, B)
    conn_in = len_add + bond_to * Ef + rng.integers(0, Ef, B)
    conn_any = len_add + rng.integers(0, N_, B) * Ef + rng.integers(0, Ef, B)
    a = np.where(u < 1 - q, add,
                 np.where(u < 1 - 0.5 * q, conn_in,
                          np.where(u < 1 - 0.3 * q, conn_any, np.where(u < 1 - 0.15 * q, apd - 1,
                                                                       rng.integers(0, apd, B)))))
    return a.astype(np.int32), len_add


def _layout_constants(N_, A_, CH_, H, C, Ef):
    from graphinvent_b200.config import make_constants
    return make_constants("GGNN", max_n_nodes=N_, n_node_features=A_ + CH_ + H + C, n_edge_features=Ef,
                          len_f_add_per_node=A_ * CH_ * max(H, 1) * max(C, 1) * Ef, len_f_conn_per_node=Ef,
                          n_atom_types=A_, n_formal_charge=CH_, n_imp_H=H, n_chirality=C)


def _assert_state_equal(gen, st, what):
    assert int(gen._counters[0].item()) == st.n_generated, what
    assert (gen.nodes.cpu().numpy() == st.nodes).all(), what
    assert (gen.edges.cpu().numpy() == st.edges).all(), what
    assert (gen.n_nodes.cpu().numpy() == st.n_nodes).all(), what
    assert (gen.likelihoods.cpu().numpy() == st.likelihoods).all(), what


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
def test_replay_reproduces_the_reference_layout_trace_bit_exactly(layout):
    from graphinvent_b200.generation import GraphGenerator
    z = _trace(layout)
    gen = GraphGenerator(model=None, batch_size=int(z["batch"]), constants=_constants(layout))
    assert (gen.n_imp_H, gen.n_chirality) == (int(z["n_imp_H"]), int(z["n_chirality"]))
    got = gen.build_graphs(replay=[(torch.from_numpy(a), torch.from_numpy(lk))
                                   for a, lk in zip(z["actions"], z["likelihoods"])])
    assert got == int(z["n_generated"]) and gen.rounds == int(z["rounds"])
    assert_matches_trace(z, *(t.cpu().numpy() for t in (gen.generated_nodes, gen.generated_edges,
                                                        gen.generated_n_nodes, gen.generated_likelihoods,
                                                        gen.properly_terminated, gen.nodes, gen.edges, gen.n_nodes,
                                                        gen.likelihoods)))


@pytest.mark.gpu
@pytest.mark.parametrize("seed,N_,A_,CH_,H,C,Ef,B", [
    (0, 13, 5, 3, 4, 0, 3, 200),      # L1
    (1, 13, 5, 3, 0, 3, 3, 200),      # L2
    (2, 13, 5, 3, 4, 3, 3, 200),      # L3
    (3, 5, 2, 1, 1, 0, 2, 64),        # L1, H = 1, small N
    (4, 4, 2, 2, 0, 1, 3, 64),        # L2, C = 1
    (5, 3, 3, 1, 1, 1, 2, 64),        # L3, H = C = 1, N = 3
    (6, 2, 2, 1, 2, 3, 3, 48),        # L3, chirality >= max_n_nodes: the reference's "max nodes" rule fires on it
    (7, 2, 2, 2, 3, 0, 3, 48),        # L1, bond type >= max_n_nodes: the same rule on the bond type
    (8, 38, 9, 3, 4, 3, 3, 96),       # L3, N = 38
    (9, 38, 4, 3, 4, 0, 3, 96),       # L1, N = 38
])
def test_layout_round_kernels_match_the_oracle_on_random_action_streams(seed, N_, A_, CH_, H, C, Ef, B):
    """the state after every round, then the finished buffers; the streams include adds into full graphs (an invalid
    action here, an IndexError in the reference) and every other validity rule"""
    from graphinvent_b200.generation import GraphGenerator
    from tests import generation_layout_oracle as L
    rng = np.random.default_rng(seed)
    rounds = 2 * N_ - 1
    liks = rng.random((rounds, B)).astype(np.float32)
    st = L.LayoutState(B, N_, A_, CH_, Ef, H, C)
    gen = GraphGenerator(model=None, batch_size=B, constants=_layout_constants(N_, A_, CH_, H, C, Ef))
    into_full = 0
    for rnd in range(rounds):
        if st.n_generated > B:          # a round writes at most B-1 graphs: stay inside the 2B output buffers
            break
        a, len_add = _layout_stream(rng, st)
        into_full += int(((a[1:] < len_add) & (st.n_nodes[1:] == N_)).sum())
        L.generation_round(st, rnd, a, liks[rnd])
        _run_round(gen, rnd, torch.from_numpy(a).cuda(), torch.from_numpy(liks[rnd]).cuda(), H, C)
        _assert_state_equal(gen, st, rnd)
    assert (gen.generated_nodes.cpu().numpy() == st.generated_nodes).all()
    assert (gen.generated_edges.cpu().numpy() == st.generated_edges).all()
    assert (gen.generated_n_nodes.cpu().numpy() == st.generated_n_nodes).all()
    assert (gen.generated_likelihoods.cpu().numpy() == st.generated_likelihoods).all()
    assert (gen.properly_terminated.cpu().numpy() == st.properly_terminated).all()
    assert st.n_generated > B // 4
    if not (H and C > N_):   # chirality >= N voids a third of the adds: that stream ends before a graph fills up
        assert into_full > 0 and int(st.generated_n_nodes.max()) == N_


@pytest.mark.gpu
@pytest.mark.parametrize("seed,N_,B", [(0, 13, 200), (1, 5, 64)])
def test_layout_entry_point_without_segments_equals_the_gdb13_entry_point(seed, N_, B):
    from graphinvent_b200.generation import GraphGenerator
    from tests import generation_layout_oracle as L
    rng = np.random.default_rng(seed)
    C = _layout_constants(N_, A, CH, 0, 0, EF)
    old, new = (GraphGenerator(model=None, batch_size=B, constants=C) for _ in range(2))
    st = L.LayoutState(B, N_, A, CH, EF)
    for rnd in range(2 * N_ - 1):
        if st.n_generated > B:
            break
        a, _ = _layout_stream(rng, st)
        lik = torch.from_numpy(rng.random(B).astype(np.float32)).cuda()
        L.generation_round(st, rnd, a, lik.cpu().numpy())
        ad = torch.from_numpy(a).cuda()
        _run_round(old, rnd, ad, lik, 0, 0, entry="gdb13")
        _run_round(new, rnd, ad, lik, 0, 0)
        _assert_state_equal(new, st, rnd)
    for name in ("nodes", "edges", "n_nodes", "likelihoods", "generated_nodes", "generated_edges",
                 "generated_n_nodes", "generated_likelihoods", "properly_terminated", "_counters"):
        assert torch.equal(getattr(old, name), getattr(new, name)), name


def _oracle_constants(C):
    from oracle import mpnn_oracle as O
    return O.make_constants(**dict(C._asdict(), device="cpu"))


def _seeded_model(model, C, seed):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    sd = O.init_state_dict(_oracle_constants(C), seed=seed)
    net = mpnn.create(C)
    net.load_state_dict(sd)
    return net.cuda(), sd


def _constants_for(model, layout="L3"):
    from graphinvent_b200.config import layout_dims, make_constants
    from tests.test_generation_layouts import FLAGS
    return make_constants(model, **layout_dims(A, CH, EF, **FLAGS[layout]))


@pytest.mark.gpu
def test_rl_generator_at_l3_dims_matches_the_oracle_two_stream_mode():
    """GraphGeneratorRL with a random-init GGNN agent and prior, replaying the actions of the L3 trace: the buffers and
    both likelihood streams equal the layout oracle fed with the same per-round probabilities, and the
    log-likelihoods back-propagate into both models"""
    from graphinvent_b200.generation import GraphGeneratorRL
    from tests import generation_layout_oracle as L
    z = _trace("L3")
    B, R = int(z["batch"]), int(z["rounds"])
    C = _constants_for("GGNN")
    agent, _ = _seeded_model("GGNN", C, 1)
    prior, _ = _seeded_model("GGNN", C, 2)
    outs = {"agent": [], "prior": []}
    agent.register_forward_hook(lambda m, i, o: outs["agent"].append(o.detach()))
    prior.register_forward_hook(lambda m, i, o: outs["prior"].append(o.detach()))
    gen = GraphGeneratorRL(None, B, constants=C)
    (nodes, edges, n_nodes), agent_ll, prior_ll, proper = gen.sample(
        agent, prior, replay=[torch.from_numpy(a) for a in z["actions"]])
    assert gen.rounds == R and int(gen._counters[0]) == int(z["n_generated"])
    assert len(outs["agent"]) == R == len(outs["prior"])
    st = L.LayoutState(B, N, A, CH, EF, 4, 3, rl=True)
    for r in range(R):
        idx = torch.from_numpy(z["actions"][r]).long().cuda().unsqueeze(1)
        la, lp = (torch.softmax(outs[k][r], dim=1).gather(1, idx).squeeze(1).cpu().numpy() for k in ("agent", "prior"))
        L.generation_round(st, r, z["actions"][r], la, lp)
    assert (gen.generated_nodes.cpu().numpy() == st.generated_nodes).all()
    assert (gen.generated_edges.cpu().numpy() == st.generated_edges).all()
    assert (gen.generated_n_nodes.cpu().numpy() == st.generated_n_nodes).all()
    assert (gen.properly_terminated.cpu().numpy() == st.properly_terminated).all()
    assert (gen.generated_agent_likelihoods.detach().cpu().numpy() == st.generated_likelihoods).all()
    assert (gen.generated_prior_likelihoods.detach().cpu().numpy() == st.generated_prior_likelihoods).all()
    assert (gen.generated_nodes.cpu().numpy().astype(np.int8) == z["generated_nodes"]).all()
    assert torch.isfinite(agent_ll).all() and torch.isfinite(prior_ll).all()
    (agent_ll.sum() + 0.5 * prior_ll.sum()).backward()
    for net in (agent, prior):
        grads = [p.grad for p in net.parameters()]
        assert all(g is not None and torch.isfinite(g).all() for g in grads)
        assert sum(float(g.norm()) for g in grads) > 0


def _segments(H, C):
    return np.cumsum([0, A, CH] + ([H] if H else []) + ([C] if C else []))


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["GGNN", "EMN"])
def test_sampling_at_l3_dims_builds_well_formed_molecules(model):
    """end to end with a seeded model: every stored atom has exactly one hot feature in each of its four segments
    (the first one with chirality index 0), rows past the atom count are empty, and the bonds are symmetric"""
    from graphinvent_b200.generation import GraphGenerator
    C = _constants_for(model)
    net, _ = _seeded_model(model, C, 5)
    gen = GraphGenerator(net.eval(), batch_size=128, constants=C)
    g = torch.Generator(device="cuda").manual_seed(0)
    (nodes, edges, n_nodes), flat, final, proper = gen.sample(generator=g)
    nodes, edges, n_nodes = nodes.cpu().numpy(), edges.cpu().numpy(), n_nodes.cpu().numpy()
    assert nodes.shape == (128, N, A + CH + 4 + 3) and torch.isfinite(final).all() and (flat > 0).all()
    atoms = np.arange(N)[None] < n_nodes[:, None]
    assert ((nodes.sum(-1) > 0) == atoms).all()
    bounds = _segments(4, 3)
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        assert (nodes[..., lo:hi].sum(-1)[atoms] == 1).all()
    assert (nodes[n_nodes > 0, 0, A + CH + 4] == 1).all()
    assert (edges == edges.transpose(0, 2, 1, 3)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["GGNN", "MNN", "AttGGNN", "EMN"])
def test_model_forward_at_l3_feature_width_matches_the_oracle(model):
    """F = 15 node features (not a multiple of 4) on generated states of the L3 trace (finished molecules and the live
    batch without the dummy slot): logits within 1e-4 of the CPU oracle, same argmax"""
    from oracle import mpnn_oracle as O
    z = _trace("L3")
    n_gen = int(z["n_generated"])
    nodes = torch.from_numpy(np.concatenate([z["generated_nodes"][:n_gen], z["final_nodes"][1:]])).float()
    edges = torch.from_numpy(np.concatenate([z["generated_edges"][:n_gen], z["final_edges"][1:]])).float()
    C = _constants_for(model)
    net, sd = _seeded_model(model, C, 9)
    with torch.no_grad():
        out = net.eval()(nodes.cuda(), edges.cuda()).cpu()
        ref = O.forward(sd, _oracle_constants(C), nodes, edges)
    assert out.shape == ref.shape == (nodes.shape[0], N * (540 + EF) + 1)
    assert (out - ref).abs().max().item() <= 1e-4
    assert torch.equal(out.argmax(1), ref.argmax(1))
