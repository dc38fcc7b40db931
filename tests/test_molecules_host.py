"""CPU: the molecule table / statistics entry points (size queries, refusals), the numpy restatement of both against
hand-computed batches in the four action layouts and against the reference's Analyzer, and the host builder of
graphinvent_b200.molecules against the reference's own graph_to_graph (stubbed rdkit, identical call logs)."""
import os

import numpy as np
import pytest
import torch

from tests import molecules_reference as R
from tests.conftest import GOLDEN

NEW_SYMBOLS = ("gib_molecule_table_bytes", "gib_molecule_table", "gib_graph_statistics_bytes",
               "gib_graph_statistics_ws_bytes", "gib_graph_statistics")


@pytest.fixture
def ref(monkeypatch):
    ns = R.load_reference(R.constants("L0"), setitem=monkeypatch.setitem)
    if ns is None:
        pytest.skip("oracle/_ref lacks the reference's MolecularGraph / GraphGenerator / Analyzer: run build()")
    return ns


def test_symbols_and_size_queries():
    from graphinvent_b200 import _lib
    from graphinvent_b200._lib import lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    B, N, F, Ef = 1000, 13, 8, 3
    assert lib.gib_molecule_table_bytes(B, N, F, Ef) == 4 * (8 + 6 * B + 3 * B * N + B * N * N * Ef)
    assert lib.gib_graph_statistics_bytes(N, F, Ef) == 4 * (N + 1 + F + 10 + Ef + 2)
    assert lib.gib_graph_statistics_ws_bytes(B, N, F, Ef) == 4 * B * (F + Ef + 12)
    assert lib.gib_molecule_table_bytes(2000, 90, 20, 4) == 4 * (8 + 6 * 2000 + 3 * 2000 * 90 + 2000 * 90 * 90 * 4)
    for dims in ((0, N, F, Ef), (B, 0, F, Ef), (B, 256, F, Ef), (B, N, 0, Ef), (B, N, 32768, Ef), (B, N, F, 0),
                 (B, N, F, 17)):
        assert lib.gib_molecule_table_bytes(*dims) == 0
        assert b"unsupported dims" in lib.gib_last_error()
        assert lib.gib_graph_statistics_ws_bytes(*dims) == 0
    assert lib.gib_graph_statistics_bytes(256, F, Ef) == 0
    # refused before anything is launched: null stream and null buffers are never touched
    assert lib.gib_molecule_table(B, 300, F, Ef, None, None, None, None, None, None) == -1
    assert lib.gib_molecule_table(B, N, F, Ef, None, None, None, None, None, None) == -1
    assert b"null argument" in lib.gib_last_error()
    assert lib.gib_graph_statistics(B, N, F, 0, None, None, None, None, None, None) == -1


def _atom(C, a, charge, h=None, chi=None):
    """one node feature row: atom type a, formal charge index, implicit-H index, chirality index"""
    row = np.zeros(C.n_node_features, np.float32)
    row[a] = 1
    row[C.n_atom_types + charge] = 1
    off = C.n_atom_types + C.n_formal_charge
    if C.n_imp_H:
        row[off + h] = 1
        off += C.n_imp_H
    if C.n_chirality:
        row[off + chi] = 1
    return row


@pytest.mark.parametrize("layout", ["L0", "L1", "L2", "L3"])
def test_table_and_statistics_of_a_hand_computed_batch(layout):
    """three molecules: C(neutral)-N(+1) with a single bond and a double bond N=O (3 atoms), an empty graph, and one
    atom whose row holds its atom-type bit only (it does not decode)"""
    C = R.constants(layout, N=4)
    F = C.n_node_features
    nodes = np.zeros((3, 4, F), np.float32)
    edges = np.zeros((3, 4, 4, 3), np.float32)
    nodes[0, 0] = _atom(C, 0, 1, 2, 1)
    nodes[0, 1] = _atom(C, 1, 2, 0, 0)
    nodes[0, 2] = _atom(C, 2, 1, 1, 2)
    for i, j, t in ((0, 1, 0), (1, 2, 1)):
        edges[0, i, j, t] = edges[0, j, i, t] = 1
    nodes[2, 0, 3] = 1
    n_nodes = np.array([3, 0, 1], np.int8)
    header, body, stats = R.table(nodes, edges, n_nodes, C)
    h, c = R.LAYOUTS[layout]
    s = C.n_atom_types + C.n_formal_charge        # start of the implicit-H segment
    x = s + h                                     # start of the chirality segment

    def rec(a, q, hh, cc):
        idx = [a, 5 + q] + ([s + hh] if h else []) + ([x + cc] if c else [])
        return [len(idx)] + (idx + [-1, -1])[:3] + [idx[-1], 0]

    want_atoms = [rec(0, 1, 2, 1), rec(1, 2, 0, 0), rec(2, 1, 1, 2), [1, 3, -1, -1, 3, 0]]
    assert header[:8].tolist() == [4, 2, -1, 0, 0, 0, 0, 0]
    assert header[8:].reshape(3, 6).tolist() == [[3, 3, 2, 0, 0, R.DECODES], [0, 0, 0, 3, 2, R.DECODES],
                                                 [1, 1, 0, 3, 2, 0]]
    assert body[:12].view(np.int16).reshape(4, 6).tolist() == want_atoms
    assert body[12:].view(np.uint8).reshape(2, 4).tolist() == [[0, 1, 0, 0], [1, 2, 1, 0]]
    # statistics: n_nodes 3, 0 and 0 (the third molecule does not decode); per-atom degrees 1, 2, 1
    col = nodes.sum((0, 1))
    want = np.concatenate([[2, 0, 0, 1, 0], col, [2, 1, 0, 0, 0, 0, 0, 0, 0, 0], [1, 1, 0], [3, 4]])
    assert stats.tolist() == want.astype(np.float32).tolist()


def _trace_batches():
    """(layout, nodes, edges, n_nodes, terminated) of the reference's recorded generation traces in the four layouts"""
    z = np.load(os.path.join(GOLDEN, "generation_trace.npz"))
    out = [("L0", z["generated_nodes"], z["generated_edges"], z["generated_n_nodes"], z["properly_terminated"],
            int(z["batch"]))]
    zl = np.load(os.path.join(GOLDEN, "generation_layout_traces.npz"))
    for name in ("L1", "L2", "L3"):
        out.append((name, zl[f"{name}/generated_nodes"], zl[f"{name}/generated_edges"],
                    zl[f"{name}/generated_n_nodes"], zl[f"{name}/properly_terminated"], int(zl[f"{name}/batch"])))
    return [(L, torch.from_numpy(n[:b]).float(), torch.from_numpy(e[:b]).float(), torch.from_numpy(nn[:b]),
             torch.from_numpy(t[:b])) for L, n, e, nn, t, b in out]


def _host_graphs(nodes, edges, n_nodes, C):
    from graphinvent_b200.molecules import graphs_from_table
    header, body, _ = R.table(nodes.numpy(), edges.numpy(), n_nodes.numpy(), C)
    R.LOG.clear()
    try:
        graphs = graphs_from_table(header, body, nodes, edges, C)
    except Exception as ex:                 # noqa: BLE001 -- compared with the reference's outcome
        graphs = ex
    return graphs, list(R.LOG)


def _assert_same_outcome(ref, nodes, edges, n_nodes, C, rl=False):
    R.set_constants(ref, C)
    want, want_log = R.reference_graphs(ref, nodes, edges, n_nodes, rl=rl)
    got, got_log = _host_graphs(nodes, edges, n_nodes, C)
    assert got_log == want_log
    assert R.describe(got) == R.describe(want)
    return got, want


@pytest.mark.parametrize("rl", [False, True])
def test_host_builder_matches_graph_to_graph_on_the_generation_traces(ref, rl):
    for layout, nodes, edges, n_nodes, _ in _trace_batches():
        C = R.constants(layout)
        got, want = _assert_same_outcome(ref, nodes, edges, n_nodes, C, rl=rl)
        assert isinstance(got, list) and sum(g.molecule is not None for g in got) > 0, layout


def test_numpy_statistics_match_the_reference_analyzer(ref):
    for layout, nodes, edges, n_nodes, term in _trace_batches():
        C = R.constants(layout)
        R.set_constants(ref, C)
        graphs, _ = R.reference_graphs(ref, nodes, edges, n_nodes)
        props, _ = R.reference_properties(ref, graphs, "Epoch 1", term)
        n_eff = np.array([g.n_nodes for g in graphs])
        stats, err = R.statistics(nodes.numpy(), edges.numpy(), n_eff)
        assert err is None
        N, F = C.max_n_nodes, C.n_node_features
        k = lambda name: props[("Epoch 1", name)]       # noqa: E731
        assert stats[:N + 1].tolist() == k("n_nodes_hist").tolist()
        assert stats[N + 1 + F:N + 11 + F].tolist() == k("n_edges_hist").tolist()
        assert stats[N + 11 + F:N + 14 + F].tolist() == k("edge_feature_hist").tolist()
        assert stats[N + 1:N + 1 + C.n_atom_types].tolist() == k("atom_type_hist").tolist()
        assert np.float32(stats[-2] / np.float32(len(graphs))) == pytest.approx(float(k("avg_n_nodes")), rel=1e-6)


def _malformed_cases(C):
    """(name, nodes [1,N,F], edges [1,N,N,Ef], n_nodes [1]) covering each way graph_to_graph fails or wraps"""
    N, F, Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
    h, c = C.n_imp_H, C.n_chirality
    base = np.zeros((N, F), np.float32)
    base[0] = _atom(C, 0, 1, 1 if h else None, 0 if c else None)
    base[1] = _atom(C, 1, 1, 0 if h else None, 1 if c else None)
    e0 = np.zeros((N, N, Ef), np.float32)
    e0[0, 1, 0] = e0[1, 0, 0] = 1
    cases = []

    def case(name, rows=None, edges=None, n=2):
        nd = base.copy()
        for i, r in (rows or {}).items():
            nd[i] = r
        cases.append((name, torch.from_numpy(nd[None]), torch.from_numpy((e0 if edges is None else edges)[None]),
                      torch.tensor([n], dtype=torch.int8)))

    z = np.zeros(F, np.float32)
    case("valid")
    case("empty row", {1: z})
    one = z.copy()
    one[2] = 1
    case("one non-zero", {1: one})
    two_types = z.copy()
    two_types[[0, 1]] = 1                           # charge index 1 - A: negative, out of range
    case("two atom-type bits", {1: two_types})
    wrap = z.copy()
    wrap[[0, 3]] = 1                                # charge index 3 - 5 = -2: wraps to a valid charge
    if h:
        wrap[C.n_atom_types + C.n_formal_charge] = 1
    case("negative charge index wraps", {1: wrap})
    if h:
        no_h = _atom(C, 1, 1, 0, 0 if c else None)
        no_h[C.n_atom_types + C.n_formal_charge:C.n_atom_types + C.n_formal_charge + h] = 0
        case("missing implicit-H bit", {1: no_h})
    if c:
        last = z.copy()
        last[[0, 6]] = 1
        if h:
            last[C.n_atom_types + C.n_formal_charge + 1] = 1
        case("chirality index from the H segment", {1: last})
    nan_row = base[1].copy()
    nan_row[F - 1] = np.nan
    case("NaN feature", {1: nan_row})
    case("n_nodes above N", n=N + 1)
    case("negative n_nodes", n=-3)
    case("n_nodes 0 with bonds", n=0)
    e = e0.copy()
    e[0, 2, 1] = e[2, 0, 1] = 1
    case("bond to an atom >= n_nodes", edges=e)
    e = e0.copy()
    e[0, 1, 2] = e[1, 0, 2] = 1
    case("one pair with two bond types", edges=e)
    e = e0.copy()
    e[1, 0, 1] = np.nan
    case("NaN below the diagonal", edges=e)
    e = e0.copy()
    e[1, 1, 0] = np.inf
    case("inf on the diagonal", edges=e)
    e = np.zeros((N, N, Ef), np.float32)
    e[0, 1, 0] = np.nan
    case("NaN above the diagonal", edges=e)
    return cases


@pytest.mark.parametrize("layout", ["L0", "L1", "L2", "L3"])
def test_malformed_rows_raise_or_wrap_as_the_reference_does(ref, layout):
    C = R.constants(layout, N=5)
    outcomes = set()
    for name, nodes, edges, n_nodes in _malformed_cases(C):
        got, want = _assert_same_outcome(ref, nodes, edges, n_nodes, C)
        outcomes.add(R.describe(got) if isinstance(got, Exception) else
                     "mol" if got[0].molecule is not None else "None")
        header, _, _ = R.table(nodes.numpy(), edges.numpy(), n_nodes.numpy(), C)
        flags = header[8 + 5]
        if isinstance(want, list):      # the decodes bit says whether graph_to_graph built a molecule
            assert bool(flags & R.DECODES) == (want[0].molecule is not None), name
        elif isinstance(want, KeyError):
            assert flags & R.KEY_ERROR, name
        else:
            assert flags & R.DUPLICATE, name
    assert outcomes == {"mol", "None", "KeyError", "RuntimeError"}


def test_statistics_errors_follow_the_reference(ref):
    """a NaN / inf row sum of an atom makes the reference's int() raise, a large negative one its histogram index;
    the value sits below the diagonal, so graph_to_graph lists it as a new bond (2, 0) (NaN and inf) or not at all"""
    C = R.constants("L0", N=4)
    R.set_constants(ref, C)
    for value, exc, kind in ((np.nan, ValueError, 1), (np.inf, OverflowError, 2), (-40.0, IndexError, 3),
                             (-5.0, None, None)):
        nodes = np.zeros((2, 4, 8), np.float32)
        for a in range(3):
            nodes[:, a] = _atom(C, a, 1)
        edges = np.zeros((2, 4, 4, 3), np.float32)
        edges[:, 0, 1, 0] = edges[:, 1, 0, 0] = 1
        edges[1, 2, 0, 1] = value
        n_nodes = torch.tensor([3, 3], dtype=torch.int8)
        graphs, _ = R.reference_graphs(ref, torch.from_numpy(nodes), torch.from_numpy(edges), n_nodes)
        assert isinstance(graphs, list)
        props, _ = R.reference_properties(ref, graphs, "Epoch 1", torch.ones(2, dtype=torch.int8))
        _, err = R.statistics(nodes, edges, np.array([g.n_nodes for g in graphs]))
        if exc is None:
            assert err is None and isinstance(props, dict)
        else:
            assert isinstance(props, exc) and err == (1, kind, 2), (value, props, err)
