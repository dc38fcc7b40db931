"""GPU: generation as replays of one captured round (graphinvent_b200.graphed.GraphedGenerator) against the eager
loop of `generation.GraphGenerator` -- forward, `sample_actions` on the same uniforms, one round kernel call -- bit
for bit: finished molecules, live state, counters, rounds.

The eager loop runs the model in capacity mode at the generator's entry capacity.  Exact mode is not bit-identical
at generation's small bond counts: there exact mode runs some message GEMMs on the fp32 SIMT kernel, while capacity
mode always uses the 3xTF32 tensor-core kernel (device-side row counts), so the sampled likelihoods can differ in
their last bits."""
import ctypes

import numpy as np
import pytest
import torch

from tests.conftest import MODELS, load_small, pretrained_path
from tests.test_generation_graphed_host import scripted_worst_case
from tests.test_gpu_generation_layouts import _constants_for, _layout_constants, _seeded_model

pytestmark = pytest.mark.gpu

STATE = ("nodes", "edges", "n_nodes", "likelihoods", "generated_nodes", "generated_edges", "generated_n_nodes",
         "generated_likelihoods", "properly_terminated")
LIMIT = "more than 2\\*max_n_nodes rounds"


def _eager(model, C, B, U, **kw):
    """the reference loop on the eager generator, the model in capacity mode at the graphed generator's entry
    capacity: returns (generator, n_generated or the RuntimeError raised)"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import entry_capacity
    gen = GraphGenerator(model, B, constants=C, **kw)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n, rnd = 0, 0
    model.entry_capacity = entry_capacity(B, gen.N, gen.Ef)
    try:
        with torch.no_grad():
            while n < B:
                if rnd >= 2 * gen.N:
                    gen.rounds = rnd
                    return gen, RuntimeError("generation needs more than 2*max_n_nodes rounds")
                out = model(*gen._model_inputs(model))
                action, lik = Fn.sample_actions(out, uniforms=U[rnd])
                gen._round(rnd, action, lik, st)
                n = int(gen._counters[0].item())
                rnd += 1
    finally:
        model.entry_capacity = None
    gen.rounds = rnd
    return gen, n


def _graphed_batch(gen, U):
    try:
        return gen.build_graphs(uniforms=U)
    except RuntimeError as e:
        return e


def _assert_same(graphed, got, eager, want):
    if isinstance(want, Exception):
        assert isinstance(got, RuntimeError) and "2*max_n_nodes" in str(got), got
    else:
        assert got == want
    assert graphed.rounds == eager.rounds
    assert graphed.inert_rounds == 1
    for name in STATE:
        assert torch.equal(getattr(graphed, name), getattr(eager, name)), name
    assert torch.equal(graphed._counters, eager._counters)
    status = 0 if not isinstance(want, Exception) else 1
    assert graphed._state.tolist() == [eager.rounds, status]


def _uniforms(N, B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(2 * N, B, generator=g, device="cuda")


def _small(model, seed=0):
    """the golden fixtures' small hidden dims with a consistent action layout (3 atom types, 1 charge)"""
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C0 = load_small(model)["C"]._asdict()
    C0.update(n_node_features=4, len_f_add_per_node=9, n_atom_types=3, n_formal_charge=1)
    for k in ("model", "edge_features", "edge_embedding_size"):
        C0.pop(k, None)
    C = make_constants(model, **dict(C0, device="cuda"))
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(O.make_constants(**dict(C._asdict(), device="cpu")), seed=seed))
    return C, net.cuda().eval()


@pytest.mark.parametrize("model", MODELS)
def test_graphed_generator_equals_the_eager_loop_small_dims(model):
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _small(model)
    B = 96
    U = _uniforms(C.max_n_nodes, B, 1)
    gen = GraphedGenerator(net, B, constants=C)
    got = _graphed_batch(gen, U)
    eager, want = _eager(net, C, B, U)
    _assert_same(gen, got, eager, want)


def test_graphed_generator_equals_the_eager_loop_pretrained_gdb13():
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator
    C = make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    net = net.cuda().eval()
    B = 256
    U = _uniforms(C.max_n_nodes, B, 2)
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    got = _graphed_batch(gen, U)
    eager, want = _eager(net, C, B, U, n_atom_types=5, n_formal_charge=3)
    assert not isinstance(want, Exception) and want >= B
    _assert_same(gen, got, eager, want)
    assert 8.0 <= gen.generated_n_nodes[:B].float().mean().item() <= 12.5


@pytest.mark.parametrize("model", ["GGNN", "AttGGNN"])
def test_graphed_generator_equals_the_eager_loop_l3_layout(model):
    from graphinvent_b200.graphed import GraphedGenerator
    C = _constants_for(model, "L3")
    net, _ = _seeded_model(model, C, 5)
    net.eval()
    B = 128
    U = _uniforms(C.max_n_nodes, B, 3)
    gen = GraphedGenerator(net, B, constants=C)
    assert (gen.n_imp_H, gen.n_chirality, gen.F) == (4, 3, 15)
    got = _graphed_batch(gen, U)
    eager, want = _eager(net, C, B, U)
    _assert_same(gen, got, eager, want)


def test_batches_pick_up_new_weights_and_keep_earlier_results():
    from graphinvent_b200.graphed import GraphedGenerator
    from oracle import mpnn_oracle as O
    C, net = _small("GGNN", seed=0)
    B = 64
    gen = GraphedGenerator(net, B, constants=C)
    U1, U2, U3 = (_uniforms(C.max_n_nodes, B, s) for s in (10, 11, 12))
    first = gen.sample(uniforms=U1)
    eager, want = _eager(net, C, B, U1)
    _assert_same(gen, int(gen._counters[0]), eager, want)
    kept = [t.clone() for t in first[0]] + [first[3].clone()]
    # a load_state_dict between batches
    net.load_state_dict(O.init_state_dict(O.make_constants(**dict(C._asdict(), device="cpu")), seed=7))
    got = _graphed_batch(gen, U2)
    eager, want = _eager(net, C, B, U2)
    _assert_same(gen, got, eager, want)
    # an in-place optimizer step
    opt = torch.optim.SGD(net.parameters(), lr=0.05)
    for p in net.parameters():
        p.grad = torch.randn_like(p)
    opt.step()
    got = _graphed_batch(gen, U3)
    eager, want = _eager(net, C, B, U3)
    _assert_same(gen, got, eager, want)
    # the first batch's results were copies
    for a, b in zip(kept, list(first[0]) + [first[3]]):
        assert torch.equal(a, b)


def test_scripted_worst_case_fits_the_capacity_and_ends_at_the_round_limit():
    """a model whose APD output Linears are zeroed gives logits that are exactly 0: u = (a + 0.5) / apd then selects
    action a.  Every slot grows a chain of N atoms, connects its last atom to every other atom, then adds into its
    full graph: the most bonds a batch can hold, and a batch that needs round 2N"""
    from graphinvent_b200._lib import FLAG_OVERFLOW
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator
    from oracle import generation_oracle as G
    N, B = 5, 64
    C = _layout_constants(N, 5, 3, 0, 0, 3)
    torch.manual_seed(4)
    net = mpnn.create(C)
    with torch.no_grad():
        for mlp in (net.APDReadout.fAddNet2, net.APDReadout.fConnNet2, net.APDReadout.fTermNet2):
            last = [m for m in mlp.modules() if isinstance(m, torch.nn.Linear)][-1]
            last.weight.zero_()
            last.bias.zero_()
    net = net.cuda().eval()
    apd = N * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
    st = G.GenerationState(B, N, 5, 3, 3)
    actions = []
    for rnd in range(2 * N):
        a = scripted_worst_case(st, rnd)
        actions.append(a)
        G.generation_round(st, rnd, a, np.full(B, 1.0 / apd, np.float32))
    U = torch.from_numpy(((np.stack(actions).astype(np.float64) + 0.5) / apd).astype(np.float32)).cuda()
    gen = GraphedGenerator(net, B, constants=C)
    with pytest.raises(RuntimeError, match=LIMIT):
        gen.build_graphs(uniforms=U)
    assert int(gen._flags) & FLAG_OVERFLOW == 0
    eager, want = _eager(net, C, B, U)
    assert isinstance(want, RuntimeError)
    _assert_same(gen, RuntimeError(LIMIT.replace("\\", "")), eager, want)
    assert gen.rounds == 2 * N and int(gen._counters[0]) == B - 1
    assert (gen.edges.cpu().numpy() == st.edges).all() and (gen.generated_edges.cpu().numpy() == st.generated_edges).all()
    assert int((gen.generated_edges[: B - 1] != 0).sum()) == 2 * (B - 1) * (2 * N - 3)


def test_replay_loop_makes_no_blocking_torch_call():
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _small("EMN")
    B = 64
    gen = GraphedGenerator(net, B, constants=C)
    U = _uniforms(C.max_n_nodes, B, 5)
    first = _graphed_batch(gen, U)                   # the round is captured here
    ref = {name: getattr(gen, name).clone() for name in STATE}
    g = torch.Generator(device="cuda").manual_seed(6)
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = _graphed_batch(gen, U)
        again = {name: getattr(gen, name).clone() for name in STATE}
        try:
            third = gen.build_graphs(generator=g)
        except RuntimeError as e:
            third = e
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for r in (first, second, third):
        assert not isinstance(r, Exception) or "synchroniz" not in str(r), r
    assert type(second) is type(first) and (isinstance(first, Exception) or second == first)
    assert all(torch.equal(again[name], ref[name]) for name in STATE)
