"""CPU: the numpy restatement of the training-set construction (tests/preprocess_reference.py) against the reference's
shipped gdb13 files and its live `DataProcesser.get_subgraphs` / `save_group` (stub rdkit / h5py / Analyzer,
`get_graph` returning pre-built `PreprocessingGraph`s); the gib_preprocess_* C-ABI and its argument refusals."""
import ctypes
import importlib.util
import os
import sys
import types
from collections import namedtuple

import numpy as np
import pytest

from oracle.reference_install import REF
from tests import molecules_reference as MR
from tests import preprocess_reference as P
from tests.conftest import GOLDEN

NEW_SYMBOLS = ("gib_preprocess_apd_length", "gib_preprocess_ws_bytes", "gib_preprocess_chunk")
LAYOUTS = {"gdb13": (5, 3, 0, 0), "imp_H": (5, 3, 4, 0), "chirality": (5, 3, 0, 3), "imp_H+chirality": (4, 3, 4, 3)}


def test_symbols_and_abi():
    from graphinvent_b200 import _lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    assert ctypes.sizeof(_lib.PPDims) == 8 * 4


def _dims(**kw):
    from graphinvent_b200._lib import PPDims
    d = dict(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1000)
    d.update(kw)
    return PPDims(**d)


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_apd_length_of_every_layout(layout):
    from graphinvent_b200 import config
    from graphinvent_b200._lib import lib
    A, Fc, H, C = LAYOUTS[layout]
    L = config.layout_dims(A, Fc, use_explicit_H=False, ignore_H=not H, use_chirality=bool(C))
    d = _dims(N=38, F=L["n_node_features"], n_atom_types=A, n_formal_charge=Fc, n_imp_H=L["n_imp_H"],
              n_chirality=L["n_chirality"])
    want = 38 * (L["len_f_add_per_node"] + L["len_f_conn_per_node"]) + 1
    assert lib.gib_preprocess_apd_length(ctypes.byref(d)) == want == P.apd_length(38, 3, P.segments(A, Fc, H, C))


@pytest.mark.parametrize("kw,msg", [
    (dict(N=105, Ef=3), b"N*N*Ef <= 32768"),
    (dict(F=9), b"sum of the layout"),
    (dict(batch_size=0), b"batch_size"),
    (dict(n_formal_charge=0, F=5), b"n_formal_charge >= 1"),
    (dict(n_imp_H=-1), b"n_imp_H >= 0"),
])
def test_dims_refused(kw, msg):
    from graphinvent_b200._lib import lib
    d = _dims(**kw)
    assert lib.gib_preprocess_apd_length(ctypes.byref(d)) < 0
    assert msg in lib.gib_last_error()
    assert lib.gib_preprocess_ws_bytes(ctypes.byref(d), 100, 1000) == 0


def test_workspace_and_chunk_arguments_refused():
    from graphinvent_b200._lib import lib
    d = _dims(N=104, Ef=3)                             # 104 * 104 * 3 = 32448: inside the limit
    assert lib.gib_preprocess_ws_bytes(ctypes.byref(d), 100, 1000) > 0
    d = _dims()
    assert lib.gib_preprocess_ws_bytes(ctypes.byref(d), 100, 999) == 0 and b"max_rows" in lib.gib_last_error()
    assert lib.gib_preprocess_ws_bytes(ctypes.byref(d), 0, 1000) == 0
    assert lib.gib_preprocess_ws_bytes(ctypes.byref(d), 1 << 25, 1000) == 0 and b"states" in lib.gib_last_error()
    small, large = (lib.gib_preprocess_ws_bytes(ctypes.byref(d), m, 1000) for m in (10, 1000))
    assert 0 < small < large
    p = ctypes.c_void_p(64)
    assert lib.gib_preprocess_chunk(ctypes.byref(d), p, p, 0, 1, 10, 1000, p, p, p, p, p, p, None) < 0
    assert b"n_molecules" in lib.gib_last_error()
    assert lib.gib_preprocess_chunk(ctypes.byref(d), p, p, 11, 1, 10, 1000, p, p, p, p, p, p, None) < 0
    assert lib.gib_preprocess_chunk(ctypes.byref(d), None, p, 5, 1, 10, 1000, p, p, p, p, p, p, None) < 0
    assert b"null" in lib.gib_last_error()


# ---- the restatement against the shipped files ------------------------------------------------------------------
def test_golden_fixture_matches_the_restatement():
    """tests/golden/preprocess_gdb13.npz: the recovered full graphs rebuild the stored counters"""
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    for key in ("gdb13_1K_debug_train", "gdb13_1K_debug_valid", "gdb13_1K_train"):
        gs = list(P.groups(z[f"{key}/nodes"], z[f"{key}/edges"], int(z[f"{key}/batch_size"]), P.segments(5, 3)))
        got = np.array([[g["start"], g["stop"], g["init_idx"], g["nodes"].shape[0], g["resume_idx"],
                         g["dataset_size"]] for g in gs])
        assert np.array_equal(got, z[f"{key}/counters"])
    assert z["gdb13_1K_train/nodes"].shape[0] == 979


@pytest.mark.parametrize("name,B,dataset_size", [("gdb13_1K/train", 1000, 11044), ("gdb13_1K-debug/train", 50, 102),
                                                 ("gdb13_1K-debug/valid", 50, 100)])
def test_restatement_rebuilds_the_shipped_files(name, B, dataset_size):
    path = os.path.join(REF, "data", "pre-training", name + ".h5")
    if not os.path.exists(path):
        pytest.skip("the reference's shipped data is not present")
    from graphinvent_b200 import data
    nodes, edges, apds = data.read_hdf5_raw(path, 13, 8, 3, 625)
    full = apds[:, -1] > 0
    gs = list(P.groups(nodes[full], edges[full], B, P.segments(5, 3)))
    n, e, a = P.assemble(gs, len(gs) * B, 13, 8, 3, 625)
    assert np.array_equal(n, nodes) and np.array_equal(e, edges) and np.array_equal(a, apds)
    # the files hold groups * batch_size rows; the reference's dataset_size counter says otherwise
    assert gs[-1]["dataset_size"] == dataset_size and len(gs) * B == nodes.shape[0]


# ---- the live reference ---------------------------------------------------------------------------------------
def _constants(N, Ef, layout, B):
    A, Fc, H, C = layout
    fields = dict(max_n_nodes=N, n_edge_features=Ef, n_atom_types=A, n_formal_charge=Fc, n_imp_H=H, n_chirality=C,
                  use_explicit_H=False, ignore_H=not H, use_chirality=bool(C), batch_size=B,
                  dim_f_add=[N] + P.segments(*layout) + [Ef], dim_f_conn=[N, Ef], n_node_features=A + Fc + H + C,
                  atom_types=["X"] * A, formal_charge=[0] * Fc, imp_H=list(range(H)), chirality=["c"] * C,
                  device="cpu")
    return namedtuple("constants", sorted(fields))(**fields)


def live_groups(monkeypatch, nodes, edges, B, layout, on_group=None, max_groups=None):
    """the reference's own get_molecule_subset / get_subgraphs / save_group loop, as preprocess() runs it (the first
    max_groups groups; on_group() after each, tools/bench_preprocess.py times them)"""
    src = os.path.join(REF, "graphinvent", "DataProcesser.py")
    if not os.path.exists(src):
        pytest.skip("the reference's DataProcesser.py is not present")
    M, N, F = nodes.shape
    Ef = edges.shape[3]
    C = _constants(N, Ef, layout, B)
    ref = MR.load_reference(C, monkeypatch.setitem)
    if ref is None:
        pytest.skip("oracle/_ref holds no MolecularGraph.py (run __graft_entry__.build() with the reference)")
    for name, mod in (("h5py", types.ModuleType("h5py")), ("tqdm", types.ModuleType("tqdm")),
                      ("Analyzer", types.ModuleType("Analyzer")), ("parameters.load", types.ModuleType("parameters.load"))):
        monkeypatch.setitem(sys.modules, name, mod)
    sys.modules["tqdm"].tqdm = lambda x: x
    sys.modules["h5py"]._hl = types.SimpleNamespace(files=types.SimpleNamespace(File=object))
    sys.modules["Analyzer"].Analyzer = object
    sys.modules["parameters"].load = sys.modules["parameters.load"]
    spec = importlib.util.spec_from_file_location("DataProcesser", src)
    DP = importlib.util.module_from_spec(spec)
    monkeypatch.setitem(sys.modules, "DataProcesser", DP)
    spec.loader.exec_module(DP)
    DP.constants = C
    graphs = []
    for m in range(M):
        g = ref.MolecularGraph.PreprocessingGraph.__new__(ref.MolecularGraph.PreprocessingGraph)
        g.constants = C
        g.node_features, g.edge_features = nodes[m].astype(np.float64), edges[m].astype(np.float64)
        g.n_nodes = P.n_atoms(nodes[m])
        graphs.append(g)
    dp = DP.DataProcesser.__new__(DP.DataProcesser)
    dp.molecule_set, dp.n_molecules, dp.is_training_set = list(range(M)), M, False
    dp.resume_idx, dp.dataset_size = 0, 0
    dp.get_graph = lambda m: graphs[m]
    saved = []

    def save_group(data_subgraphs, data_apds, group_size, init_idx):
        saved.append(dict(init_idx=init_idx, nodes=np.array([s[0] for s in data_subgraphs]).astype(np.int8),
                          edges=np.array([s[1] for s in data_subgraphs]).astype(np.int8),
                          apds=np.array(data_apds).astype(np.int64), group_size=group_size))
    dp.save_group = save_group
    g = 0
    while dp.resume_idx < M and (max_groups is None or g < max_groups):
        start = dp.resume_idx
        dp.get_molecule_subset()
        dp.get_subgraphs(init_idx=g * B)
        if on_group:
            on_group()
        saved[-1].update(start=start, stop=dp.resume_idx, resume_idx=dp.resume_idx, dataset_size=dp.dataset_size)
        g += 1
    return saved


def assert_same_as_live(ours, live):
    assert len(ours) == len(live)
    for o, r in zip(ours, live):
        for k in ("init_idx", "start", "stop", "resume_idx", "dataset_size"):
            assert o[k] == r[k], k
        assert r["group_size"] == o["nodes"].shape[0]
        assert np.array_equal(o["nodes"], r["nodes"]) and np.array_equal(o["edges"], r["edges"])
        assert np.array_equal(o["apds"], r["apds"])


def _synthetic(M, N, layout, Ef=3, seed=0, repeat=None):
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
    nodes = np.concatenate([nodes] + extra, axis=2)
    if repeat is not None:
        nodes, edges = nodes[repeat], edges[repeat]
    return nodes, edges


@pytest.mark.parametrize("case", ["quirk", "cut_groups", "partial_middle", "B1", "identical", "rings_N13",
                                  "imp_H", "chirality", "imp_H+chirality", "Ef4"])
def test_restatement_matches_the_live_reference(monkeypatch, case):
    layout, N, Ef, B, M, repeat = LAYOUTS["gdb13"], 13, 3, 20, 30, None
    if case == "quirk":
        repeat = [0, 1, 2, 0, 1, 2, 2, 3, 4, 5, 5, 6]
        B = 200
    elif case == "cut_groups":
        B = 9
    elif case == "partial_middle":
        repeat, B = [0] * 8 + list(range(1, 10)), 6          # a group of repeats runs out of molecules mid-set
    elif case == "B1":
        B, M = 1, 6
    elif case == "identical":
        repeat, B = [3] * 40, 1000
    elif case == "rings_N13":
        B, M = 40, 40
    elif case in LAYOUTS:
        layout, N, B = LAYOUTS[case], 16, 25
    elif case == "Ef4":
        Ef, B = 4, 15
    nodes, edges = _synthetic(M, N, layout, Ef=Ef, seed=sum(map(ord, case)), repeat=repeat)
    ours = list(P.groups(nodes, edges, B, P.segments(*layout)))
    assert_same_as_live(ours, live_groups(monkeypatch, nodes, edges, B, layout))
    if case == "quirk":      # the rule fires: some row repeats the row before it
        assert any((g["nodes"][1:] == g["nodes"][:-1]).all((1, 2)).any() for g in ours)
    if case == "rings_N13":  # ring closures give connect APDs
        assert any(g["apds"][:, 13 * 45:13 * 48].any() for g in ours)
