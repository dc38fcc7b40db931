"""GPU: gib_molecule_table / gib_graph_statistics and graphinvent_b200.molecules against the numpy restatement
(tests/molecules_reference.py) and against the reference's own graph_to_graph and get_molecular_properties run live on
the same CUDA tensors (stubbed rdkit: identical call logs; properties equal bit for bit and type for type).

Inputs: the recorded generation traces in the four action layouts, GraphedGenerator batches of the four models, and
adversarial batches (empty molecules, N atoms, hubs of degree > 10, isolated atoms, malformed rows, n_nodes outside
[0, N], NaN / inf above and below the diagonal; B 1..2000, N up to 90, Ef 1..4)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import molecules_reference as R
from tests.conftest import MODELS
from tests.guarded import Guarded

pytestmark = pytest.mark.gpu


@pytest.fixture
def ref(monkeypatch):
    ns = R.load_reference(R.constants("L0"), setitem=monkeypatch.setitem)
    if ns is None:
        pytest.skip("oracle/_ref lacks the reference's MolecularGraph / GraphGenerator / Analyzer: run build()")
    return ns


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same_properties(got, want):
    if isinstance(want, Exception):
        assert type(got) is type(want), (got, want)
        return
    assert list(got) == list(want)
    for k in want:
        a, b = got[k], want[k]
        assert type(a) is type(b), (k, type(a), type(b))
        if isinstance(b, torch.Tensor):
            assert (a.dtype, a.device, a.shape) == (b.dtype, b.device, b.shape), k
            assert torch.equal(_bits(a), _bits(b)), (k, a, b)
        elif isinstance(b, float) and np.isnan(b):
            assert np.isnan(a), k
        else:
            assert a == b, (k, a, b)


def _properties(batch, graphs, key, term):
    try:
        return batch.properties(key, term, graphs)
    except Exception as ex:            # noqa: BLE001 -- compared with the reference's outcome
        return ex


def check_batch(ref, nodes, edges, n_nodes, C, term=None, live=True):
    """one batch on the device: table and statistics against numpy, then (live) graphs and properties against the
    reference run on the same tensors.  Returns the MoleculeBatch."""
    from graphinvent_b200.molecules import MoleculeBatch
    nodes, edges, n_nodes = nodes.cuda(), edges.cuda(), n_nodes.cuda()
    batch = MoleculeBatch(nodes, edges, n_nodes, C)
    header, body, stats = R.table(nodes.cpu().numpy(), edges.cpu().numpy(), n_nodes.cpu().numpy(), C)
    assert np.array_equal(batch.header, header)
    assert np.array_equal(batch.body, body)
    assert np.array_equal(batch.stats.cpu().numpy(), stats, equal_nan=True)
    if not live:
        return batch
    R.set_constants(ref, C)
    want, want_log = R.reference_graphs(ref, nodes, edges, n_nodes)
    R.LOG.clear()
    try:
        got = batch.generation_graphs()
    except Exception as ex:            # noqa: BLE001
        got = ex
    assert list(R.LOG) == want_log
    assert R.describe(got) == R.describe(want)
    if isinstance(want, Exception):
        return batch
    term = term.cuda() if term is not None else (torch.arange(nodes.shape[0], device=nodes.device) % 3 != 0).to(torch.int8)
    for key in ("Epoch 3", "Training set"):
        want_p, want_log = R.reference_properties(ref, want, key, term)
        R.LOG.clear()
        got_p = _properties(batch, got, key, term)
        assert_same_properties(got_p, want_p)
        if not isinstance(want_p, Exception):
            assert list(R.LOG) == want_log
    return batch


def _gpu_constants(layout, N, Ef):
    return R.constants(layout, N=N, Ef=Ef, device="cuda")


@pytest.mark.parametrize("layout", ["L0", "L1", "L2", "L3"])
def test_generation_traces(ref, layout):
    from tests.test_molecules_host import _trace_batches
    (_, nodes, edges, n_nodes, term), = [t for t in _trace_batches() if t[0] == layout]
    batch = check_batch(ref, nodes, edges, n_nodes, _gpu_constants(layout, 13, 3), term=term)
    assert batch.decodes.sum() > 0


def adversarial(C, B, seed, nan=False):
    """a seeded batch of edge cases.  nan=False keeps graph_to_graph from raising (so that the statistics can be
    compared); nan=True adds NaN / inf entries, bonds to missing atoms and duplicate bond types"""
    rng = np.random.default_rng(seed)
    N, F, Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
    h, c = C.n_imp_H, C.n_chirality
    nodes = np.zeros((B, N, F), np.float32)
    edges = np.zeros((B, N, N, Ef), np.float32)
    n_nodes = np.zeros(B, np.int8)
    for b in range(B):
        kind = rng.integers(0, 9)
        n = {0: 0, 1: N, 2: min(N, 127)}.get(kind, int(rng.integers(1, N + 1)))
        for a in range(n):
            nodes[b, a, rng.integers(0, C.n_atom_types)] = 1
            nodes[b, a, C.n_atom_types + rng.integers(0, C.n_formal_charge)] = 1
            if h:
                nodes[b, a, C.n_atom_types + C.n_formal_charge + rng.integers(0, h)] = 1
            if c:
                nodes[b, a, F - c + rng.integers(0, c)] = 1
        if n > 1:
            if kind in (1, 3):                      # a hub: atom 0 bonded to every other atom
                for j in range(1, n):
                    t = rng.integers(0, Ef)
                    edges[b, 0, j, t] = edges[b, j, 0, t] = 1
            else:                                   # a random sparse graph: some atoms stay isolated
                for _ in range(int(rng.integers(0, n + 1))):
                    i, j = sorted(rng.choice(n, 2, replace=False))
                    if edges[b, i, j].sum() == 0:
                        t = rng.integers(0, Ef)
                        edges[b, i, j, t] = edges[b, j, i, t] = rng.choice([1.0, 2.0, 0.5])
        if kind == 4 and n > 0:                     # a malformed row
            a = rng.integers(0, n)
            nodes[b, a] = 0
            nodes[b, a, rng.choice(F, int(rng.integers(0, 4)), replace=False)] = 1
        if kind == 5:
            n = int(rng.choice([-1, -100, min(127, N + 1 + int(rng.integers(0, 3)))]))
        if kind == 6 and n > 0:                     # features past n_nodes (read by the node histogram only)
            nodes[b, n:, 0] = 1
        if nan and kind in (7, 8) and n > 2:
            i, j = sorted(rng.choice(n, 2, replace=False))
            v = rng.choice([np.nan, np.inf, -np.inf, 1.0])
            if kind == 7:
                edges[b, i, j, rng.integers(0, Ef)] = v
            else:
                edges[b, j, i, rng.integers(0, Ef)] = v
            if rng.random() < 0.3:
                edges[b, i, rng.integers(0, N), rng.integers(0, Ef)] = 1
        n_nodes[b] = n
    return torch.from_numpy(nodes), torch.from_numpy(edges), torch.from_numpy(n_nodes)


@pytest.mark.parametrize("layout,B,N,Ef", [("L0", 1, 13, 3), ("L1", 7, 13, 1), ("L2", 64, 38, 4), ("L3", 48, 90, 4),
                                           ("L0", 300, 13, 2), ("L3", 2000, 13, 3)])
def test_adversarial_batches(ref, layout, B, N, Ef):
    C = _gpu_constants(layout, N, Ef)
    live = B <= 300                       # the reference's per-atom reads take minutes at B = 2000
    check_batch(ref, *adversarial(C, B, seed=B + N), C, live=live)


@pytest.mark.parametrize("layout", ["L0", "L3"])
def test_adversarial_batches_with_nan_and_raising_molecules(ref, layout):
    C = _gpu_constants(layout, 13, 3)
    outcomes = set()
    for seed in range(24):
        nodes, edges, n_nodes = adversarial(C, 3, seed=seed, nan=True)
        batch = check_batch(ref, nodes, edges, n_nodes, C)
        try:
            graphs = batch.generation_graphs()
        except Exception as ex:           # noqa: BLE001
            outcomes.add(type(ex).__name__)
            continue
        p = _properties(batch, graphs, "Epoch 1", torch.ones(3, dtype=torch.int8).cuda())
        outcomes.add(type(p).__name__)
    assert {"dict", "ValueError"} <= outcomes, outcomes


def _launch(B, N, F, Ef, C, nodes, edges, n_nodes, table, out, ws):
    from graphinvent_b200._lib import check, lib
    from graphinvent_b200.molecules import mol_layout
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lay = mol_layout(C)
    check(lib.gib_molecule_table(B, N, F, Ef, ctypes.byref(lay), nodes.data_ptr(), edges.data_ptr(),
                                 n_nodes.data_ptr(), table, st), "gib_molecule_table")
    check(lib.gib_graph_statistics(B, N, F, Ef, nodes.data_ptr(), edges.data_ptr(), table, out, ws, st),
          "gib_graph_statistics")
    torch.cuda.synchronize()


@pytest.mark.parametrize("layout,B,N,Ef", [("L1", 37, 13, 3), ("L3", 5, 90, 4)])
def test_buffers_poisoned_and_guard_banded(layout, B, N, Ef):
    """no band byte is written; the table's header and used records and the statistics are the same on poisoned and on
    zeroed buffers, and the table's unused tail keeps the fill"""
    from graphinvent_b200._lib import lib
    C = _gpu_constants(layout, N, Ef)
    nodes, edges, n_nodes = (t.cuda() for t in adversarial(C, B, seed=5))
    F = C.n_node_features
    sizes = (lib.gib_molecule_table_bytes(B, N, F, Ef), lib.gib_graph_statistics_bytes(N, F, Ef),
             lib.gib_graph_statistics_ws_bytes(B, N, F, Ef))
    runs = {}
    for fill in ("poison", "zero"):
        bufs = [Guarded(n, fill=fill) for n in sizes]
        _launch(B, N, F, Ef, C, nodes, edges, n_nodes, *(g.ptr() for g in bufs))
        for g in bufs:
            assert g.intact(), (fill, g.damage())
        table = bufs[0].view(torch.int32)
        used = 8 + 6 * B + 3 * int(table[0]) + int(table[1])
        assert bool((bufs[0].t[4 * used:] == (0xFF if fill == "poison" else 0)).all())
        runs[fill] = (table[:used].clone(), bufs[1].view(torch.int32).clone())
    assert torch.equal(runs["poison"][0], runs["zero"][0]) and torch.equal(runs["poison"][1], runs["zero"][1])


def _d2h_copies(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sum(1 for e in prof.events() if "Memcpy DtoH" in e.name and e.device_type.name == "CUDA")


def test_at_most_two_device_to_host_copies_per_batch(ref):
    from graphinvent_b200.molecules import MoleculeBatch
    from tests.test_molecules_host import _trace_batches
    C = _gpu_constants("L0", 13, 3)
    R.set_constants(ref, C)
    _, nodes, edges, n_nodes, term = _trace_batches()[0]
    nodes, edges, n_nodes, term = nodes.cuda(), edges.cuda(), n_nodes.cuda(), term.cuda()
    MoleculeBatch(nodes, edges, n_nodes, C).generation_graphs()              # warm-up (module load, allocator)
    (batch, graphs), n = _d2h_copies(lambda: (lambda b: (b, b.generation_graphs()))(
        MoleculeBatch(nodes, edges, n_nodes, C)))
    assert n == 2, n
    _, n = _d2h_copies(lambda: batch.properties("Epoch 1", term, graphs))
    assert n == 1, n                                                          # termination, read once
    _, n = _d2h_copies(lambda: R.reference_graphs(ref, nodes, edges, n_nodes))
    assert n > 50 * nodes.shape[0]                                            # the reference's per-atom reads


def _ref_constants_for(C, Ef):
    """reference constants for the small-dims generators of tests/test_gpu_generation_graphed.py (3 atom types, one
    formal charge)"""
    RC = R.constants("L0", N=C.max_n_nodes, Ef=Ef, device="cuda")
    return RC._replace(n_atom_types=3, atom_types=["C", "N", "O"], n_formal_charge=1, formal_charge=[0],
                       n_node_features=4, dim_nodes=[C.max_n_nodes, 4])


@pytest.mark.parametrize("model", MODELS)
def test_graphed_generator_sample_molecules(ref, model):
    from graphinvent_b200.graphed import GraphedGenerator
    from tests.test_gpu_generation_graphed import _small, _uniforms
    C, net = _small(model)
    B = 96
    RC = _ref_constants_for(C, C.n_edge_features)
    gen = GraphedGenerator(net, B, constants=C)
    for seed in range(1, 6):
        U = _uniforms(C.max_n_nodes, B, seed)
        try:
            (nodes, edges, n_nodes), flat, final, term = gen.sample(uniforms=U)
        except RuntimeError:
            continue
        graphs, flat2, final2, term2 = gen.sample_molecules(uniforms=U, constants=RC)
        assert torch.equal(flat, flat2) and torch.equal(final, final2) and torch.equal(term, term2)
        batch = check_batch(ref, nodes, edges, n_nodes, RC, term=term)
        assert R.describe(graphs)[0][:2] == R.describe(batch.generation_graphs())[0][:2]
        assert [g.n_nodes for g in graphs] == [g.n_nodes for g in batch.generation_graphs()]
        return
    pytest.skip("no batch finished within the round limit")


@pytest.mark.parametrize("model", ["GGNN", "AttGGNN"])
def test_eager_generator_sample_molecules(ref, model):
    from graphinvent_b200.generation import GraphGenerator
    from tests.test_gpu_generation_graphed import _small
    C, net = _small(model)
    B = 64
    RC = _ref_constants_for(C, C.n_edge_features)
    gen = GraphGenerator(net, B, constants=C)
    for seed in range(1, 6):
        try:
            (nodes, edges, n_nodes), flat, final, term = gen.sample(
                generator=torch.Generator(device="cuda").manual_seed(seed))
        except RuntimeError:
            continue
        nodes, edges, n_nodes = nodes.clone(), edges.clone(), n_nodes.clone()
        graphs, flat2, final2, term2 = gen.sample_molecules(
            generator=torch.Generator(device="cuda").manual_seed(seed), constants=RC)
        assert torch.equal(flat, flat2) and torch.equal(final, final2) and torch.equal(term, term2)
        assert torch.equal(gen.molecules.nodes, nodes) and torch.equal(gen.molecules.n_nodes, n_nodes)
        R.set_constants(ref, RC)
        want, _ = R.reference_graphs(ref, gen.molecules.nodes, gen.molecules.edges, gen.molecules.n_nodes)
        assert R.describe(graphs) == R.describe(want)
        return
    pytest.skip("no batch finished within the round limit")


@pytest.mark.parametrize("model", ["GGNN", "EMN"])
def test_rl_sample_molecules_keeps_the_gradient(ref, model):
    from tests.test_gpu_rl_graphed import _finished_rollout, _grads, _loss
    C, agent, prior, gen, U = _finished_rollout(model)
    RC = _ref_constants_for(C, C.n_edge_features)
    _, agent_ll, prior_ll, term = gen.sample(agent, prior, uniforms=U)
    agent.zero_grad()
    prior.zero_grad()
    _loss(agent_ll, prior_ll).backward()
    want = _grads(agent) + _grads(prior)
    agent.zero_grad()
    prior.zero_grad()
    graphs, agent_ll2, prior_ll2, term2 = gen.sample_molecules(agent, prior, uniforms=U, constants=RC)
    assert agent_ll2.requires_grad and prior_ll2.requires_grad
    assert torch.equal(agent_ll, agent_ll2) and torch.equal(prior_ll, prior_ll2) and torch.equal(term, term2)
    _loss(agent_ll2, prior_ll2).backward()
    got = _grads(agent) + _grads(prior)
    assert any(g is not None and bool(g.abs().sum() > 0) for g in got)
    for a, b in zip(got, want):
        assert (a is None and b is None) or torch.equal(a, b)
    R.set_constants(ref, RC)
    want_graphs, _ = R.reference_graphs(ref, gen.molecules.nodes, gen.molecules.edges, gen.molecules.n_nodes, rl=True)
    assert R.describe(graphs) == R.describe(want_graphs)
