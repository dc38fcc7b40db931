"""CPU: the training-set properties of the device preprocessing pass -- the numpy restatement of each group's integer
statistics (tests/ts_properties_reference.py) through `preprocess.ts_properties` / `merge_ts_properties` -- against
the live reference `Analyzer.get_molecular_properties` / `combine_ts_properties` run as `get_ts_properties` runs them,
type for type and bit for bit; the CSV against the shipped gdb13_1K train.csv; the gib_preprocess_group_statistics
C-ABI and its argument refusals."""
import ctypes
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

from oracle.reference_install import REF
from tests import molecules_reference as MR
from tests import preprocess_reference as P
from tests import ts_properties_reference as TR
from tests.conftest import GOLDEN

LAYOUTS = TR.LAYOUTS
SYMBOLS = ("gib_preprocess_group_statistics_bytes", "gib_preprocess_group_statistics_ws_bytes",
           "gib_preprocess_group_statistics")


def test_symbols():
    from graphinvent_b200 import _lib
    assert set(SYMBOLS) <= set(_lib.exported_symbols())


def _dims(**kw):
    from graphinvent_b200._lib import PPDims
    d = dict(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=20)
    d.update(kw)
    return PPDims(**d)


def test_sizes_and_refusals():
    from graphinvent_b200._lib import lib
    d = _dims()
    assert lib.gib_preprocess_group_statistics_bytes(ctypes.byref(d), 7) == 4 * 7 * (4 + 14 + 8 + 10 + 3)
    assert lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(d), 7) == 4 * 7 * (8 + 3 + 12)
    for bad in (_dims(F=9), _dims(batch_size=0), _dims(N=13, Ef=17)):
        assert lib.gib_preprocess_group_statistics_bytes(ctypes.byref(bad), 7) == 0
        assert lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(bad), 7) == 0
    assert b"Ef" in lib.gib_last_error()
    assert lib.gib_preprocess_group_statistics_bytes(None, 7) == 0 and b"null" in lib.gib_last_error()
    assert lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(d), 0) == 0
    p = ctypes.c_void_p(64)
    assert lib.gib_preprocess_group_statistics(ctypes.byref(d), p, p, 0, 10, p, p, p, p, None) < 0
    assert b"n_molecules" in lib.gib_last_error()
    assert lib.gib_preprocess_group_statistics(ctypes.byref(d), p, p, 11, 10, p, p, p, p, None) < 0
    assert lib.gib_preprocess_group_statistics(ctypes.byref(d), p, p, 5, 10, p, p, None, p, None) < 0
    assert b"null" in lib.gib_last_error()


# ---- molecules --------------------------------------------------------------------------------------------------
def synthetic(M, N, layout, Ef=3, seed=0):
    """seeded molecules of graphinvent_b200.synthetic with the layout's implicit-H / chirality segments"""
    from graphinvent_b200 import synthetic as S
    A, Fc, H, C = layout
    nodes, edges = S.random_graphs(M, N, A, Fc, n_edge_features=Ef, seed=seed, min_atoms=1)
    rng = np.random.default_rng(seed + 1)
    extra = []
    for w in (H, C):
        if w:
            seg = np.zeros((M, N, w), np.int8)
            present = nodes.any(2)
            seg[present, rng.integers(0, w, int(present.sum()))] = 1
            extra.append(seg)
    return np.concatenate([nodes] + extra, axis=2), edges


def single_atom(N, layout, Ef=3, atom=1):
    F = sum(layout)
    nodes, edges = np.zeros((1, N, F), np.int8), np.zeros((1, N, N, Ef), np.int8)
    nodes[0, 0, atom] = nodes[0, 0, layout[0] + 1] = 1
    for j, w in enumerate(layout[2:]):
        if w:
            nodes[0, 0, sum(layout[:2 + j])] = 1
    return nodes, edges


def hub(N, layout, leaves, Ef=3, bond=0):
    """atom 0 bonded to atoms 1..leaves: more than 10 bonds for leaves > 10"""
    nodes, edges = single_atom(N, layout, Ef, atom=0)
    for v in range(1, leaves + 1):
        nodes[0, v] = nodes[0, 0]
        edges[0, 0, v, bond] = edges[0, v, 0, bond] = 1
    return nodes, edges


def cases():
    return ["single_atoms_and_hubs", "cut_groups", "short_last_group", "one_group", "unique_smiles"] + \
        [k for k in LAYOUTS if k != "gdb13"]


def make_case(case):
    """(layout name, nodes, edges, batch_size, SMILES keys or None)"""
    layout, N, Ef, B, keys = "gdb13", 13, 3, 9, None
    if case == "single_atoms_and_hubs":
        parts = [synthetic(6, N, LAYOUTS[layout], seed=1), single_atom(N, LAYOUTS[layout]), hub(N, LAYOUTS[layout], 12),
                 hub(N, LAYOUTS[layout], 11, bond=2), single_atom(N, LAYOUTS[layout], atom=3),
                 synthetic(5, N, LAYOUTS[layout], seed=2), hub(N, LAYOUTS[layout], 10, bond=1)]
        nodes, edges = (np.concatenate(x) for x in zip(*parts))
        B = 11
    elif case == "cut_groups":
        nodes, edges = synthetic(40, N, LAYOUTS[layout], seed=3)
    elif case == "short_last_group":
        nodes, edges = synthetic(23, N, LAYOUTS[layout], seed=4)
        B = 40
    elif case == "one_group":
        nodes, edges = synthetic(15, N, LAYOUTS[layout], seed=5)
        B = 1000
    elif case == "unique_smiles":
        nodes, edges = synthetic(30, N, LAYOUTS[layout], seed=6)
        keys = [None if m % 7 == 3 else f"M{m % 5}" for m in range(30)]
        B = 25
    else:
        layout, N, B = case, 16, 25
        nodes, edges = synthetic(40, N, LAYOUTS[layout], Ef=Ef, seed=sum(map(ord, case)))
    return layout, nodes, edges, B, keys


@pytest.fixture
def ref(monkeypatch):
    r = MR.load_reference(TR.constants("gdb13"), monkeypatch.setitem)
    if r is None:
        pytest.skip("oracle/_ref holds no Analyzer.py (run __graft_entry__.build() with the reference)")
    return r


def restated_ts_properties(ref, C, nodes, edges, spans, smiles):
    """the device path's dicts and merge (graphinvent_b200.preprocess) on the restated group statistics"""
    from graphinvent_b200 import preprocess as PP
    analyzer = ref.Analyzer.Analyzer.__new__(ref.Analyzer.Analyzer)
    out = None
    for start, stop in spans:
        stats = PP.Statistics(*TR.statistics(nodes[start:stop], edges[start:stop]))
        out = PP.merge_ts_properties(analyzer, out, PP.ts_properties(stats, smiles[start:stop], C), C.batch_size)
    return out


@pytest.mark.parametrize("case", cases())
def test_restatement_matches_the_live_reference(ref, case):
    layout, nodes, edges, B, keys = make_case(case)
    C = TR.constants(layout, nodes.shape[1], edges.shape[3], B)
    MR.set_constants(ref, C)
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges, keys)
    gs = list(P.groups(nodes, edges, B, P.segments(*LAYOUTS[layout])))
    spans = [(g["start"], g["stop"]) for g in gs]
    want = TR.reference_ts_properties(ref, graphs, spans, B)
    got = restated_ts_properties(ref, C, nodes, edges, spans, [g.get_smiles() for g in graphs])
    TR.assert_identical(got, want)
    if case == "one_group":
        assert len(spans) == 1 and len(got) == 13       # written unmerged
    else:
        assert len(spans) > 1 and len(got) == 11
    if case == "cut_groups":                            # a group that reached batch_size before its molecules ran out
        assert any(g["full"] and g["stop"] - g["start"] < B for g in gs)
    if case == "short_last_group":
        assert not gs[-1]["full"] and gs[-1]["stop"] - gs[-1]["start"] < B
    if case == "single_atoms_and_hubs":                 # bin 9 holds the clamped hubs and the bond-less single atoms
        assert TR.statistics(nodes, edges)[2][9] >= 4
    if case == "unique_smiles":
        assert 0 < float(got[("Training set", "fraction_unique")]) < 1


def test_gdb13_train_csv(ref, tmp_path):
    """gdb13_1K/train's full graphs (tests/golden/preprocess_gdb13.npz) give the values of the shipped train.csv
    (tests/golden/gdb13_1K_train.csv; numpy 2 writes its values with another repr, so values are compared)"""
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges, B = z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"], int(z["gdb13_1K_train/batch_size"])
    C = TR.constants("gdb13", 13, 3, B)
    MR.set_constants(ref, C)
    gs = list(P.groups(nodes, edges, B, P.segments(*LAYOUTS["gdb13"])))
    spans = [(g["start"], g["stop"]) for g in gs]
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges)
    smiles = [g.get_smiles() for g in graphs]
    assert set(smiles) == {None}                        # PreprocessingGraph keeps no molecule: fraction_unique 0.0
    got = restated_ts_properties(ref, C, nodes, edges, spans, smiles)
    TR.assert_identical(got, TR.reference_ts_properties(ref, graphs, spans, B))
    TR.write_ts_properties(tmp_path / "train.csv", got)
    assert TR.parse_csv(tmp_path / "train.csv") == TR.parse_csv(os.path.join(GOLDEN, "gdb13_1K_train.csv"))


def _reference_util(monkeypatch, C):
    src = os.path.join(REF, "graphinvent", "util.py")
    if not os.path.exists(src):
        pytest.skip("the reference's util.py is not present")
    monkeypatch.setattr(sys.modules["rdkit"], "RDLogger", types.SimpleNamespace(), raising=False)
    spec = importlib.util.spec_from_file_location("reference_util", src)
    util = importlib.util.module_from_spec(spec)
    util.plt = types.SimpleNamespace(axes=object)       # a name its annotations use without importing it
    spec.loader.exec_module(util)
    util.constants = C
    return util


@pytest.mark.parametrize("case", ["one_group", "cut_groups", "imp_H+chirality"])
def test_csv_rule_matches_the_reference_writer(ref, monkeypatch, tmp_path, case):
    """the tests' CSV writer (used where the reference's util.py is not installed) writes the bytes its
    write_ts_properties writes, for an unmerged dict (tensors) and a merged one (numpy arrays)"""
    layout, nodes, edges, B, keys = make_case(case)
    C = TR.constants(layout, nodes.shape[1], edges.shape[3], B, training_set=str(tmp_path / "train.smi"))
    MR.set_constants(ref, C)
    util = _reference_util(monkeypatch, C)
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges, keys)
    spans = [(g["start"], g["stop"]) for g in P.groups(nodes, edges, B, P.segments(*LAYOUTS[layout]))]
    props = restated_ts_properties(ref, C, nodes, edges, spans, [g.get_smiles() for g in graphs])
    util.write_ts_properties(training_set_properties=props)
    TR.write_ts_properties(tmp_path / "mine.csv", props)
    assert (tmp_path / "train.csv").read_bytes() == (tmp_path / "mine.csv").read_bytes()
