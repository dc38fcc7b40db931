"""GPU: decoding routes chosen on the device (graphinvent_b200.preprocess.reorder, csrc/preprocess.cu reorder_kernel) and
the loader that trains on a fresh random route of every molecule each pass (graphinvent_b200.loader.RandomRouteLoader).

  1. reorder against the reference's own BFS / DFS orders (tests/golden/route_orders.npz): orders equal and the
     reordered stacks' digest equal, gdb13 and N = 38; the four action layouts and N = 181 with one bond type against
     the restatement (tests/route_order_reference.py), with the device-drawn rankings;
  2. the refusals: disconnected, empty, a bad ranking, a molecule `groups` refuses;
  3. the drawn rankings: permutations, a function of (seed, epoch, molecule) only, a uniform start atom, and torch's
     default generator untouched;
  4. the loader: each pass equal to DeviceBlockLoader over the file the reference's preprocessing writes for that
     pass's molecules (built on the host path), its len, total_batches and set_epoch;
  5. train_epoch over a pass bit-identical to train_epoch over the equivalent DeviceBlockLoader.
"""
import copy
import hashlib
import os
import time
import types

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_order_reference as RO
from tests.conftest import GOLDEN
from tests.test_gpu_preprocess import LAYOUTS, complete_graph, graphs

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(GOLDEN, "route_orders.npz")
GDB13 = LAYOUTS["gdb13"]


def _fixture(name):
    z = np.load(FIXTURE)
    return z, z[f"{name}/nodes"], z[f"{name}/edges"], z[f"{name}/rankings"], z[f"{name}/orders"]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the orders
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["gdb13", "synthetic38"])
@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_reorder_equals_the_reference(name, route):
    from graphinvent_b200 import preprocess as PP
    z, nodes, edges, rankings, orders = _fixture(name)
    M, R, N = rankings.shape
    # every (molecule, ranking) pair as one molecule of the stack, in [M, R] order
    X = np.repeat(nodes, R, axis=0)
    E = np.repeat(edges, R, axis=0)
    on, oe, order = PP.reorder(X, E, route, rankings=rankings.reshape(M * R, N), layout=GDB13)
    want = orders[:, :, 0 if route == "bfs" else 1].reshape(M * R, N)
    assert np.array_equal(order.cpu().numpy(), want)
    assert hashlib.sha256(on.cpu().numpy().tobytes() + oe.cpu().numpy().tobytes()).hexdigest() == \
        str(z[f"{name}/sha256_{route}"])


def _check_against_restatement(nodes, edges, route, layout, **kw):
    from graphinvent_b200 import preprocess as PP
    on, oe, order = PP.reorder(nodes, edges, route, seed=7, epoch=3, layout=layout, **kw)
    n_atoms = [RO.n_atoms(x) for x in nodes]
    rk = PP.rankings(n_atoms, nodes.shape[1], seed=7, epoch=3).cpu().numpy()
    on, oe, order = on.cpu().numpy(), oe.cpu().numpy(), order.cpu().numpy()
    for m in range(nodes.shape[0]):
        o, X, E = RO.node_remap(nodes[m], edges[m], rk[m, :n_atoms[m]].tolist(), route)
        assert np.array_equal(order[m], o), m
        assert np.array_equal(on[m], X) and np.array_equal(oe[m], E), m


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_action_layouts(layout, route):
    nodes, edges = graphs(60, 38, LAYOUTS[layout], seed=4)
    _check_against_restatement(nodes, edges, route, LAYOUTS[layout])


@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_n181_one_bond_type(route):
    """N = 181, Ef = 1: sparse molecules up to 181 atoms and complete graphs, whose BFS layers of up to 180 atoms grow
    the set table to 512 slots"""
    nodes, edges = graphs(6, 181, GDB13, Ef=1, seed=9, min_atoms=150)
    full = [complete_graph(n, 181, GDB13, 1, seed=n) for n in (181, 97, 40)]
    nodes = np.concatenate([nodes, np.stack([f[0] for f in full])])
    edges = np.concatenate([edges, np.stack([f[1] for f in full])])
    _check_against_restatement(nodes, edges, route, GDB13)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_refusals(route):
    from graphinvent_b200 import preprocess as PP
    nodes, edges = graphs(12, 13, GDB13, seed=3, min_atoms=4)
    n3 = RO.n_atoms(nodes[3])
    bad = edges.copy()                                   # molecule 3: its last atom cut off
    bad[3, n3 - 1, :, :] = 0
    bad[3, :, n3 - 1, :] = 0
    t0 = time.perf_counter()
    with pytest.raises(ValueError, match=r"molecule 3 .*disconnected"):
        PP.reorder(nodes, bad, route, layout=GDB13)
    assert time.perf_counter() - t0 < 30
    empty = nodes.copy()
    empty[5] = 0
    e5 = edges.copy()
    e5[5] = 0
    with pytest.raises(ValueError, match=r"molecule 5 .*no atoms"):
        PP.reorder(empty, e5, route, layout=GDB13)
    rk = PP.rankings([RO.n_atoms(x) for x in nodes], 13).cpu().numpy()
    rk[7, 1] = rk[7, 0]                                  # not a permutation
    with pytest.raises(ValueError, match=r"molecule 7 .*ranking"):
        PP.reorder(nodes, edges, route, rankings=rk, layout=GDB13)
    rk = PP.rankings([RO.n_atoms(x) for x in nodes], 13).cpu().numpy()
    rk[2, 0] = 13                                        # out of range
    with pytest.raises(ValueError, match=r"molecule 2 .*ranking"):
        PP.reorder(nodes, edges, route, rankings=rk, layout=GDB13)
    two = nodes.copy()                                   # two atom types on one atom: groups refuses it too
    two[9, 0, :5] = 1
    with pytest.raises(ValueError, match=r"molecule 9 .*one-hot"):
        PP.reorder(two, edges, route, layout=GDB13)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the drawn rankings
# ---------------------------------------------------------------------------------------------------------------------
def test_drawn_rankings():
    from scipy.stats import chisquare

    from graphinvent_b200 import preprocess as PP
    n_atoms = np.random.default_rng(0).integers(1, 39, 3000)
    state = torch.get_rng_state(), torch.cuda.get_rng_state()
    a = PP.rankings(n_atoms, 38, seed=11, epoch=2).cpu().numpy()
    assert torch.equal(torch.get_rng_state(), state[0]) and torch.equal(torch.cuda.get_rng_state(), state[1])
    for m, n in enumerate(n_atoms):
        assert sorted(a[m, :n]) == list(range(n)) and (a[m, n:] == -1).all()
    pieces = [PP.rankings(n_atoms[s:s + 700], 38, seed=11, epoch=2, first=s).cpu().numpy()
              for s in range(0, 3000, 700)]
    assert np.array_equal(np.concatenate(pieces), a)
    assert np.array_equal(PP.rankings(n_atoms, 38, seed=11, epoch=2).cpu().numpy(), a)
    b = PP.rankings(n_atoms, 38, seed=11, epoch=3).cpu().numpy()
    assert (a != b).any(1).mean() > 0.9                 # 1- and 2-atom molecules have one or two rankings
    assert not np.array_equal(PP.rankings(n_atoms, 38, seed=12, epoch=2).cpu().numpy(), a)
    # the start atom (ranking[0]) of a 6-atom molecule is uniform
    start = PP.rankings(np.full(60000, 6), 6, seed=5, epoch=0).cpu().numpy()[:, 0]
    assert chisquare(np.bincount(start, minlength=6)).pvalue > 1e-3
    # reorder's own draws are these rankings, and leave torch's generators alone
    nodes, edges = graphs(50, 13, GDB13, seed=1)
    state = torch.get_rng_state(), torch.cuda.get_rng_state()
    _, _, order = PP.reorder(nodes, edges, "bfs", seed=3, epoch=1, layout=GDB13)
    assert torch.equal(torch.get_rng_state(), state[0]) and torch.equal(torch.cuda.get_rng_state(), state[1])
    rk = PP.rankings([RO.n_atoms(x) for x in nodes], 13, seed=3, epoch=1)
    assert torch.equal(PP.reorder(nodes, edges, "bfs", rankings=rk, layout=GDB13)[2], order)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the loader contract
# ---------------------------------------------------------------------------------------------------------------------
def _host_file(nodes, edges, B, route, seed, epoch, layout=GDB13):
    """the file the reference's preprocessing writes for the pass's reordered molecules, built on the host path:
    reorder -> groups -> assemble -> the final resize"""
    from graphinvent_b200 import preprocess as PP
    on, oe, _ = PP.reorder(nodes, edges, route, seed=seed, epoch=epoch, layout=layout)
    on, oe = on.cpu().numpy(), oe.cpu().numpy()
    gs = [dict(init_idx=g.init_idx, nodes=g.nodes, edges=g.edges, apds=g.apds.astype(np.int64), size=g.dataset_size)
          for g in PP.groups(on, oe, B, *layout)]
    N, F, Ef = on.shape[1], on.shape[2], oe.shape[3]
    apd_len = P.apd_length(N, Ef, P.segments(*layout))
    n, e, a = P.assemble(gs, P.total_subgraphs(oe), N, F, Ef, apd_len)
    size = gs[-1]["size"]
    return types.SimpleNamespace(nodes=n[:size], edges=e[:size], apds=a[:size])


def _gdb13_molecules():
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]


@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_passes_equal_device_block_loader_over_the_file(route):
    from graphinvent_b200.loader import DeviceBlockLoader, RandomRouteLoader
    nodes, edges = _gdb13_molecules()
    B, K = 250, 4000
    loader = RandomRouteLoader(nodes, edges, batch_size=B, block_size=K, route=route, seed=21, n_atom_types=5,
                               n_formal_charge=3)
    lens = []
    for epoch in (0, 1):
        ds = _host_file(nodes, edges, B, route, 21, epoch)
        ref = DeviceBlockLoader(ds, batch_size=B, block_size=K)
        assert loader.epoch == epoch
        assert len(loader) == len(ref) and loader.n_rows == ds.nodes.shape[0]
        lens.append(len(ref))
        assert np.array_equal(loader.dataset.apds.cpu().numpy(), ds.apds)
        torch.manual_seed(5 + epoch)
        got = [tuple(t.clone() for t in b) for b in loader]
        rand = torch.rand(3)
        torch.manual_seed(5 + epoch)
        want = list(ref)
        assert torch.equal(torch.rand(3), rand)
        assert len(got) == len(want) == lens[-1]
        for g, w in zip(got, want):
            for x, y in zip(g, w):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert loader.epoch == 2
    assert loader.total_batches(0, 2) == sum(lens)
    assert loader.total_batches(1, 1) == lens[1]
    # set_epoch repeats a pass: its rows, and with the same seed its batches
    loader.set_epoch(0)
    ds = _host_file(nodes, edges, B, route, 21, 0)
    assert len(loader) == lens[0]
    assert np.array_equal(loader.dataset.edges.cpu().numpy(), ds.edges)


def test_device_rows_equal_the_file_layouts():
    """file_rows against the host path: chunk boundaries inside groups, a last group that cuts rows, layouts"""
    from graphinvent_b200 import preprocess as PP
    for layout, B, chunk in (("gdb13", 7, 7), ("imp_H", 40, 64), ("imp_H+chirality", 1000, 4096)):
        nodes, edges = graphs(130, 38, LAYOUTS[layout], seed=2)
        ds = _host_file(nodes, edges, B, "bfs", 0, 0, LAYOUTS[layout])
        on, oe, _ = PP.reorder(nodes, edges, "bfs", layout=LAYOUTS[layout])
        rows, size = PP.file_rows(on, oe, B, *LAYOUTS[layout], chunk_molecules=chunk)
        assert size == ds.nodes.shape[0] and PP.file_rows(on, oe, B, *LAYOUTS[layout], keep=False)[1] == size
        for got, want in zip(rows, (ds.nodes, ds.edges, ds.apds)):
            assert np.array_equal(got.cpu().numpy(), want), layout


# ---------------------------------------------------------------------------------------------------------------------
# 5. training
# ---------------------------------------------------------------------------------------------------------------------
def test_train_epoch_equals_device_block_loader():
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.loader import DeviceBlockLoader, RandomRouteLoader
    from graphinvent_b200.optim import FlatAdam
    from oracle import mpnn_oracle as O
    from tests.test_gpu_partial_and_eval import _capacity
    nodes, edges = _gdb13_molecules()
    nodes, edges = nodes[:300], edges[:300]
    C = O.make_constants("GGNN")
    base = mpnn.create(C)
    base.load_state_dict(O.init_state_dict(C, seed=0))
    base = base.cuda()
    B = 100
    cap = _capacity(torch.from_numpy(edges).cuda(), C)
    steps = []
    for _ in range(2):
        net = copy.deepcopy(base)
        opt = FlatAdam(net.parameters(), lr=1e-3)
        steps.append((TrainStep(net, opt, batch_size=B, entry_capacity=cap, input_dtype=torch.int8),
                      torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-2, total_steps=200)))
    loader = RandomRouteLoader(nodes, edges, batch_size=B, block_size=1000, seed=4, constants=types.SimpleNamespace(
        n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, use_explicit_H=False, ignore_H=True,
        use_chirality=False))
    seen = []
    for epoch in (0, 1):
        ref = DeviceBlockLoader(_host_file(nodes, edges, B, "bfs", 4, epoch), batch_size=B, block_size=1000)
        torch.manual_seed(epoch)
        got = steps[0][0].train_epoch(loader, steps[0][1])
        torch.manual_seed(epoch)
        want = steps[1][0].train_epoch(ref, steps[1][1])
        assert torch.equal(got.view(1).view(torch.int32), want.view(1).view(torch.int32)), (float(got), float(want))
        for p, q in zip(steps[0][0].model.parameters(), steps[1][0].model.parameters()):
            assert torch.equal(p.detach().view(torch.int32), q.detach().view(torch.int32))
        seen.append(loader.dataset.edges[:loader.n_rows].cpu().numpy())
    assert seen[0].shape != seen[1].shape or not np.array_equal(seen[0], seen[1])
