"""CPU: the conditional route scorer's C-ABI (symbols, argument refusals) and the rule it implements: the numpy
restatement's conditional states (tests/scaffold_route_reference.py) against the live reference's
get_decoding_route_state routes of gdb13_1K molecules for every prefix k, their first state against the scaffold
oracle's start state, and their mask decisions against scaffold_oracle.forbidden."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from tests import preprocess_reference as P
from tests import scaffold_oracle as SO
from tests import scaffold_route_reference as SR
from tests.conftest import GOLDEN

NEW_SYMBOLS = ("gib_route_plan_scaffold", "gib_route_fill_scaffold", "gib_route_mask_logits")
SEGS = P.segments(5, 3)
N, EF, PER_NODE = 13, 3, 5 * 3 * 3


def _dims(**kw):
    from graphinvent_b200._lib import PPDims
    d = dict(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=100)
    d.update(kw)
    return PPDims(**d)


def test_symbols_are_declared_exported_and_bound_and_the_abi_is_unchanged():
    from graphinvent_b200 import _lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    for name in NEW_SYMBOLS:
        assert getattr(_lib.lib, name).argtypes is not None
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "gib200.h")).read()
    assert all(f"{name}(" in header for name in NEW_SYMBOLS)
    assert "GIB_ROUTE_NOT_PREFIX = 1, GIB_ROUTE_MASKED = 2, GIB_ROUTE_BAD_ID = 4" in header
    assert (_lib.ROUTE_NOT_PREFIX, _lib.ROUTE_MASKED, _lib.ROUTE_BAD_ID) == (1, 2, 4)
    assert _lib.lib.gib_version() == 206


def test_entry_points_refuse_bad_arguments():
    from graphinvent_b200._lib import Scaffolds, lib
    d = _dims()
    bd = ctypes.byref(d)
    p, a16 = ctypes.c_void_p(64), ctypes.c_void_p(64)
    sc = Scaffolds(nodes=64, edges=64, n_atoms=64, protect=64, S=2)
    scb = ctypes.byref(sc)
    plan = lambda *a: lib.gib_route_plan_scaffold(bd, *a, None)
    err = lambda: lib.gib_last_error()
    assert plan(p, p, 0, 10, scb, p, p, p, p) < 0 and b"gib_route_plan_scaffold" in err() and b"n_molecules" in err()
    assert plan(p, p, 11, 10, scb, p, p, p, p) < 0 and b"n_molecules" in err()
    assert plan(p, p, 5, 10, scb, None, p, p, p) < 0 and b"null" in err()
    assert plan(p, p, 5, 10, None, p, p, p, p) < 0 and b"scaffold table" in err()
    assert plan(p, p, 5, 10, ctypes.byref(Scaffolds(nodes=64, edges=64, n_atoms=64, S=0)), p, p, p, p) < 0
    assert b"S >= 1" in err()
    assert plan(p, p, 5, 10, ctypes.byref(Scaffolds(nodes=64, edges=None, n_atoms=64, S=1)), p, p, p, p) < 0
    assert plan(p, p, 5, 0, scb, p, p, p, p) < 0 and b"max_molecules" in err()
    assert lib.gib_route_plan_scaffold(ctypes.byref(_dims(F=9)), p, p, 5, 10, scb, p, p, p, p, None) < 0
    fill = lambda *a: lib.gib_route_fill_scaffold(bd, *a, None)
    assert fill(p, p, 10, p, p, p, None, p, p, p, p, a16, a16) < 0 and b"null" in err()
    assert fill(p, p, 10, p, p, p, p, p, p, p, None, a16, a16) < 0 and b"gib_route_fill_scaffold: null" in err()
    assert fill(ctypes.c_void_p(65), p, 10, p, p, p, p, p, p, p, p, a16, a16) < 0 and b"16-byte" in err()
    assert fill(p, p, 10, p, p, p, p, p, p, p, p, a16, ctypes.c_void_p(72)) < 0 and b"16-byte" in err()
    assert fill(p, p, 0, p, p, p, p, p, p, p, p, a16, a16) < 0 and b"max_molecules" in err()
    mask = lambda *a: lib.gib_route_mask_logits(*a, None)
    apd = N * (PER_NODE + EF) + 1
    assert mask(0, N, EF, apd, scb, p, p, p) < 0 and b"gib_route_mask_logits" in err()
    assert mask(4, N, EF, apd + 1, scb, p, p, p) < 0 and b"apd - 1" in err()
    assert mask(4, N, EF, apd, None, p, p, p) < 0
    assert mask(4, N, EF, apd, scb, None, p, p) < 0
    assert mask(4, N, EF, apd, scb, p, p, None) < 0
    # a table without attachment points masks nothing: no launch, success
    assert mask(4, N, EF, apd, ctypes.byref(Scaffolds(nodes=64, edges=64, n_atoms=64, S=2)), p, p, p) == 0


def _live_routes(monkeypatch, nodes, edges):
    """per molecule the live reference's decoding-route states (X, E, action), in the reference's own order"""
    from tests import molecules_reference as MR
    spec = importlib.util.spec_from_file_location("_make_route_nll", os.path.join(GOLDEN, "make_route_nll.py"))
    maker = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(maker)
    ref = MR.load_reference(maker.route_constants(), monkeypatch.setitem)
    if ref is None:
        pytest.skip("oracle/_ref holds no MolecularGraph.py (run __graft_entry__.build() with the reference)")
    G = ref.MolecularGraph.PreprocessingGraph
    out = []
    for m in range(nodes.shape[0]):
        g = G.__new__(G)
        g.constants = maker.route_constants()
        g.node_features, g.edge_features = nodes[m].astype(np.float64), edges[m].astype(np.float64)
        g.n_nodes = P.n_atoms(nodes[m])
        states = []
        for k in range(g.get_decoding_route_length()):
            (X, E), apd = g.get_decoding_route_state(k)
            states.append((np.asarray(X).astype(np.int8), np.asarray(E).astype(np.int8),
                           int(np.argmax(np.asarray(apd).ravel()))))
        out.append(states)
    return out


def test_conditional_route_is_the_tail_of_the_live_reference_route(monkeypatch):
    """for every molecule of the first 40 of gdb13_1K/train and every k = 1..n: the restatement's conditional
    states are the last n_bonds - m_k + 1 of the live reference's route, reversed; the first is byte-equal to the
    scaffold oracle's start state of the k-atom prefix; and every mask decision equals scaffold_oracle.forbidden"""
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"][:40], z["gdb13_1K_train/edges"][:40]
    live = _live_routes(monkeypatch, nodes, edges)
    checked = 0
    for m in range(nodes.shape[0]):
        n = P.n_atoms(nodes[m])
        ks = np.arange(1, n + 1)
        sn, se = SR.prefix_scaffolds(np.repeat(nodes[m:m + 1], n, 0), np.repeat(edges[m:m + 1], n, 0), ks)
        for s, k in enumerate(ks):
            X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes[m:m + 1], edges[m:m + 1], [s], sn, SEGS)
            m_k = SR.n_bonds(se[s])
            kept = SR.n_bonds(edges[m]) - m_k + 1
            assert X.shape[0] == kept == offsets[-1]
            tail = live[m][:kept][::-1]                 # the reference's order runs from the full graph back
            for i, (x, e, a) in enumerate(tail):
                assert np.array_equal(X[i], x) and np.array_equal(E[i], e) and acts[i] == a, (m, k, i)
            # the start state the generator writes for this scaffold (the float 0/1 table rows)
            st = SO.ScaffoldState(2, N, 5, 3, EF, 0, 0, sn[s:s + 1], se[s:s + 1])
            assert np.array_equal(st.nodes[1].astype(np.int8), X[0]) and np.array_equal(st.edges[1].astype(np.int8), E[0])
            assert st.n_nodes[1] == k == n_at[0]
            # the mask: with the decoration's own attachment points nothing it takes is forbidden; with every
            # scaffold atom protected the rule decides as the oracle's
            for attach in (SR.decoration_points(nodes[m], edges[m], int(k)), []):
                protect = SR.protect_of(sn[s:s + 1], [attach])
                ours = SR.state_masks(sid * 0, n_at, sn[s:s + 1], protect, N, EF, PER_NODE)
                for i in range(X.shape[0]):
                    st.n_nodes[1] = n_at[i]
                    assert np.array_equal(ours[i], SO.forbidden(st, 1, protect)), (m, k, i)
                if attach:
                    assert not ours[np.arange(X.shape[0]), acts].any(), (m, k)
            checked += 1
    assert checked > 300


def test_restatement_refuses_nothing_it_should_score():
    """a molecule is its own scaffold (k = n): one state, the terminate action; k = 1: every state but the empty one"""
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"][:4], z["gdb13_1K_train/edges"][:4]
    for m in range(4):
        n = P.n_atoms(nodes[m])
        sn, se = SR.prefix_scaffolds(nodes[m:m + 1].repeat(2, 0), edges[m:m + 1].repeat(2, 0), [n, 1])
        X, _, acts, offsets, _, _ = SR.conditional_states(nodes[m:m + 1].repeat(2, 0), edges[m:m + 1].repeat(2, 0),
                                                          [0, 1], sn, SEGS)
        assert offsets.tolist() == [0, 1, 1 + SR.n_bonds(edges[m]) + 1]
        assert acts[0] == N * (PER_NODE + EF) and np.array_equal(X[0], nodes[m])
