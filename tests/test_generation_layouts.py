"""The implicit-H and chirality action layouts of the generator (reference parameters/constants.py:23-95), on CPU.

Pin: tests/golden/generation_layout_traces.npz, recorded from the unmodified reference `GraphGenerator` by
tests/golden/make_generation_layout_traces.py in three layouts (L1 implicit H, L2 chirality, L3 both; N = 13, A = 5,
CH = 3, H = 4, C = 3, Ef = 3): draws and stored likelihoods of every round, final buffers and live state."""
import ctypes
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN
from tests.hostshim import _view

N, A, CH, EF = 13, 5, 3, 3
LAYOUTS = ("L1", "L2", "L3")
FLAGS = {"L0": dict(), "L1": dict(ignore_H=False), "L2": dict(use_chirality=True),
         "L3": dict(ignore_H=False, use_chirality=True)}


def _trace(layout):
    z = np.load(os.path.join(GOLDEN, "generation_layout_traces.npz"))
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(layout + "/")}


def _replay_oracle(z):
    from tests import generation_layout_oracle as L
    st = L.LayoutState(int(z["batch"]), N, A, CH, EF, int(z["n_imp_H"]), int(z["n_chirality"]))
    for rnd, (a, lik) in enumerate(zip(z["actions"], z["likelihoods"])):
        L.generation_round(st, rnd, a, lik)
    return st


def assert_matches_trace(z, generated_nodes, generated_edges, generated_n_nodes, generated_likelihoods,
                         properly_terminated, nodes, edges, n_nodes, likelihoods):
    """every buffer of the reference's generator after its last round, bit for bit (numpy arrays)"""
    assert (generated_nodes.astype(np.int8) == z["generated_nodes"]).all()
    assert (generated_edges.astype(np.int8) == z["generated_edges"]).all()
    assert (generated_n_nodes == z["generated_n_nodes"]).all()
    assert (generated_likelihoods == z["generated_likelihoods"]).all()
    assert (properly_terminated == z["properly_terminated"]).all()
    assert (nodes.astype(np.int8) == z["final_nodes"]).all() and (edges.astype(np.int8) == z["final_edges"]).all()
    assert (n_nodes.astype(np.int8) == z["final_n_nodes"]).all() and (likelihoods == z["final_likelihoods"]).all()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_layout_trace_fixture_is_self_consistent(layout):
    z = _trace(layout)
    B, n_gen, R = int(z["batch"]), int(z["n_generated"]), int(z["rounds"])
    H, C = int(z["n_imp_H"]), int(z["n_chirality"])
    assert (H, C) == {"L1": (4, 0), "L2": (0, 3), "L3": (4, 3)}[layout]
    assert z["actions"].shape == (R, B) and z["likelihoods"].shape == (R, B) and B <= n_gen <= 2 * B
    nn = z["generated_n_nodes"][:n_gen]
    g = z["generated_nodes"][:n_gen]
    assert g.shape[-1] == A + CH + H + C and int(nn.max()) == N
    atoms = g.sum(-1) > 0
    assert (atoms.sum(-1) == nn).all()
    bounds = np.cumsum([0, A, CH] + ([H] if H else []) + ([C] if C else []))
    for lo, hi in zip(bounds[:-1], bounds[1:]):              # one hot feature per segment on every stored atom
        assert (g[..., lo:hi].sum(-1)[atoms] == 1).all()
    if H and C:                                               # quirk 1: every first atom stored with chirality 0
        assert (g[nn > 0, 0, A + CH + H] == 1).all()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_layout_oracle_replays_the_reference_trace_bit_exactly(layout):
    z = _trace(layout)
    st = _replay_oracle(z)
    assert st.n_generated == int(z["n_generated"])
    assert_matches_trace(z, st.generated_nodes, st.generated_edges, st.generated_n_nodes, st.generated_likelihoods,
                         st.properly_terminated, st.nodes, st.edges, st.n_nodes, st.likelihoods)


def test_layout_oracle_without_segments_replays_the_gdb13_traces():
    """H = C = 0 is the gdb13 oracle: both of its reference traces (plain and RL) replay bit-exactly"""
    from tests import generation_layout_oracle as L
    z = np.load(os.path.join(GOLDEN, "generation_trace.npz"))
    st = L.LayoutState(int(z["batch"]), N, A, CH, EF)
    for rnd, (a, lik) in enumerate(zip(z["actions"], z["likelihoods"])):
        L.generation_round(st, rnd, a, lik)
    assert st.n_generated == int(z["n_generated"])
    assert_matches_trace(z, st.generated_nodes, st.generated_edges, st.generated_n_nodes, st.generated_likelihoods,
                         st.properly_terminated, st.nodes, st.edges, st.n_nodes, st.likelihoods)
    z = np.load(os.path.join(GOLDEN, "generation_rl_trace.npz"))
    st = L.LayoutState(int(z["batch"]), N, A, CH, EF, rl=True)
    for r in range(int(z["rounds"])):
        L.generation_round(st, r, z["actions"][r], z["agent_likelihoods"][r], z["prior_likelihoods"][r])
    assert (st.generated_nodes.astype(np.int8) == z["generated_nodes"]).all()
    assert (st.generated_likelihoods == z["generated_agent_likelihoods"]).all()
    assert (st.generated_prior_likelihoods == z["generated_prior_likelihoods"]).all()


def test_layout_dims_restate_the_reference_constants():
    from graphinvent_b200.config import layout_dims
    want = {"L0": (8, 45, 0, 0), "L1": (12, 180, 4, 0), "L2": (11, 135, 0, 3), "L3": (15, 540, 4, 3)}
    for layout, flags in FLAGS.items():
        d = layout_dims(A, CH, EF, **flags)
        assert (d["n_node_features"], d["len_f_add_per_node"], d["n_imp_H"], d["n_chirality"]) == want[layout]
    # explicit H is the gdb13 layout with H among the atom types; it cannot be combined with ignore_H
    assert layout_dims(6, CH, EF, use_explicit_H=True, ignore_H=False)["n_node_features"] == 9
    with pytest.raises(ValueError):
        layout_dims(A, CH, EF, use_explicit_H=True, ignore_H=True)


def _constants(layout, **overrides):
    from graphinvent_b200.config import layout_dims, make_constants
    d = dict(layout_dims(A, CH, EF, **FLAGS[layout]), **overrides)
    return make_constants("GGNN", **d)


@pytest.mark.parametrize("overrides,kw", [
    (dict(n_node_features=14), {}),                        # F != A + CH + H + C
    (dict(len_f_add_per_node=180), {}),                    # the add segment of L1, with L3 node features
    (dict(n_chirality=0), {}),                             # node features of L3, counts of L1
    ({}, dict(n_imp_H=0)),                                 # an explicit count that contradicts the constants
    ({}, dict(n_chirality=-3, n_imp_H=10)),
    (dict(n_atom_types=0, n_node_features=10, len_f_add_per_node=0), {}),
    (dict(n_imp_H=256, n_node_features=267, len_f_add_per_node=5 * 3 * 256 * 3 * 3), {}),
])
def test_generator_refuses_inconsistent_layout_dims_before_allocating(monkeypatch, overrides, kw):
    from graphinvent_b200.generation import GraphGenerator, GraphGeneratorRL

    def no_allocation(self):
        raise AssertionError("allocated before validating the layout")
    monkeypatch.setattr(GraphGenerator, "_allocate", no_allocation)
    C = _constants("L3", **overrides)
    for cls in (GraphGenerator, GraphGeneratorRL):
        with pytest.raises(ValueError, match="inconsistent action layout"):
            cls(None, 8, constants=C, device="cpu", **kw)


def _fake_generation_round_layout(B, N_, F, Ef, A_, CH_, H, C, rnd, action, lik, nodes, edges, n_nodes, likelihoods,
                                  g_nodes, g_edges, g_n_nodes, g_lik, proper, cap, counters, scratch, stream):
    """`gib_generation_round_layout` played by the layout oracle in place on the caller's CPU tensors"""
    from tests import generation_layout_oracle as L
    st = L.LayoutState.__new__(L.LayoutState)
    st.B, st.N, st.A, st.CH, st.H, st.C, st.Ef, st.F, st.rl = B, N_, A_, CH_, H, C, Ef, F, False
    f32, i32, i8 = (ctypes.c_float, np.float32), (ctypes.c_int32, np.int32), (ctypes.c_int8, np.int8)
    st.nodes = _view(nodes, (B, N_, F), *f32)
    st.edges = _view(edges, (B, N_, N_, Ef), *f32)
    st.n_nodes = _view(n_nodes, (B,), *i32)
    st.likelihoods = _view(likelihoods, (B, 2 * N_), *f32)
    st.generated_nodes = _view(g_nodes, (cap, N_, F), *f32)
    st.generated_edges = _view(g_edges, (cap, N_, N_, Ef), *f32)
    st.generated_n_nodes = _view(g_n_nodes, (cap,), *i8)
    st.generated_likelihoods = _view(g_lik, (cap, 2 * N_), *f32)
    st.properly_terminated = _view(proper, (cap,), *i8)
    cnt = _view(counters, (2,), *i32)
    st.n_generated = int(cnt[0])
    written = L.generation_round(st, rnd, _view(action, (B,), *i32), _view(lik, (B,), *f32))
    cnt[0], cnt[1] = st.n_generated, written
    return 0


@pytest.mark.parametrize("layout", LAYOUTS)
def test_generator_host_logic_replays_the_layout_trace_on_cpu_shims(monkeypatch, layout):
    """GraphGenerator's own plumbing for the new layouts (dims from the constants, the layout entry point and its
    argument order) with the round played by the layout oracle; the gdb13 entry point must not be called"""
    from tests import hostshim
    from graphinvent_b200 import generation as gen_mod
    hostshim.install_generation_shims(monkeypatch)
    calls = []

    def layout_entry(*args):
        calls.append(args[6:8])
        return _fake_generation_round_layout(*args)
    monkeypatch.setattr(gen_mod, "lib", types.SimpleNamespace(
        gib_generation_round=None, gib_generation_round_layout=layout_entry, gib_generation_scratch_bytes=lambda B: 64))
    z = _trace(layout)
    gen = gen_mod.GraphGenerator(None, int(z["batch"]), constants=_constants(layout), device="cpu")
    got = gen.build_graphs(replay=[(torch.from_numpy(a), torch.from_numpy(lk))
                                   for a, lk in zip(z["actions"], z["likelihoods"])])
    assert got == int(z["n_generated"]) and gen.rounds == int(z["rounds"])
    assert set(calls) == {(int(z["n_imp_H"]), int(z["n_chirality"]))}
    assert_matches_trace(z, *(t.numpy() for t in (gen.generated_nodes, gen.generated_edges, gen.generated_n_nodes,
                                                  gen.generated_likelihoods, gen.properly_terminated, gen.nodes,
                                                  gen.edges, gen.n_nodes, gen.likelihoods)))


def _reference_generator_module(monkeypatch, C):
    """the unmodified reference GraphGenerator.py from oracle/_ref/, imported with the stub modules of
    tests/golden/make_generation_trace.py (rdkit, MolecularGraph, parameters.constants)"""
    from tests import refimpl
    path = os.path.join(refimpl.REF_ROOT, "GraphGenerator.py")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref absent: run __graft_entry__.build() with a checkout of the reference")
    for name in ("rdkit", "rdkit.Chem"):
        monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
    mg = types.ModuleType("MolecularGraph")
    mg.GenerationGraph = type("GenerationGraph", (), {"__init__": lambda self, **kw: None})
    monkeypatch.setitem(sys.modules, "MolecularGraph", mg)
    pkg, pc = types.ModuleType("parameters"), types.ModuleType("parameters.constants")
    pkg.__path__ = []
    pc.constants = C
    pkg.constants = pc
    monkeypatch.setitem(sys.modules, "parameters", pkg)
    monkeypatch.setitem(sys.modules, "parameters.constants", pc)
    spec = importlib.util.spec_from_file_location("_reference_GraphGenerator", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("layout", ["L1", "L3"])
def test_reference_add_into_a_full_graph_raises_index_error(monkeypatch, layout):
    """the one deliberate deviation: outside the gdb13 layout the reference's "max nodes" rule looks at bond_type or
    chirality instead of bond_from (GraphGenerator.py:618), so an add into a graph that already holds max_n_nodes atoms
    is applied at nodes[b, max_n_nodes] and raises.  The device generator terminates such a slot as invalid."""
    spec = importlib.util.spec_from_file_location("_make_layout_traces",
                                                  os.path.join(GOLDEN, "make_generation_layout_traces.py"))
    script = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script)               # the constants the fixtures were recorded with
    C = script.layout_constants(*script.LAYOUTS[layout])
    GG = _reference_generator_module(monkeypatch, C)
    B = 4
    apd = N * (C.len_f_add_per_node + EF) + 1

    class Fixed(torch.nn.Module):               # all mass on add(bond_to=0, index 0 of every other segment)
        def forward(self, nodes, edges):
            out = torch.full((nodes.shape[0], apd), -1e4)
            out[:, 0] = 0.0
            return out

    with torch.no_grad():
        gen = GG.GraphGenerator(model=Fixed(), batch_size=B)
        gen.n_nodes[1] = N                      # slot 1 holds a full molecule
        gen.nodes[1, :, 0] = 1
        gen.nodes[1, :, A] = 1
        with pytest.raises(IndexError):
            gen.build_graphs()


def test_layout_entry_point_refuses_inconsistent_arguments():
    """refused on the host, before any launch: F != A + CH + H + C, a count above 255 or below 0, a bad round"""
    from graphinvent_b200._lib import lib
    for (F, H, C, rnd) in ((14, 4, 3, 0), (16, 4, 3, 0), (15, 4, 4, 0), (5 + 3 + 256 + 3, 256, 3, 0),
                           (5 + 3 + 4 - 1, 4, -1, 0), (15, 4, 3, 2 * N)):
        rc = lib.gib_generation_round_layout(8, N, F, EF, A, CH, H, C, rnd, *([None] * 11), 16, None, None, None)
        assert rc == -1 and b"gib_generation_round" in lib.gib_last_error(), (F, H, C, rnd)
    # the gdb13 entry point is the layout entry point without segments: it refuses the same way
    assert lib.gib_generation_round(8, N, 9, EF, A, CH, 0, *([None] * 11), 16, None, None, None) == -1
    assert lib.gib_generation_round(8, N, 8, 256, A, CH, 0, *([None] * 11), 16, None, None, None) == -1
