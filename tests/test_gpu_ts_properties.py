"""GPU: the training-set properties of the device preprocessing pass -- gib_preprocess_group_statistics through
`preprocess.groups(..., statistics=True)` against the numpy restatement (tests/ts_properties_reference.py), on fresh and
on guarded, poisoned buffers; `run_data_processer(..., device_properties=True)` against the reference's
`get_ts_properties` loop with constants.device = "cuda": the same dict, type for type and bit for bit, the same CSV
bytes, and the values of the shipped gdb13_1K train.csv."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from tests import molecules_reference as MR
from tests import preprocess_reference as P
from tests import test_ts_properties_host as H
from tests import ts_properties_reference as TR
from tests.conftest import GOLDEN
from tests.guarded import Guarded

pytestmark = pytest.mark.gpu

LAYOUTS = TR.LAYOUTS


def assert_statistics(dev_groups, nodes, edges):
    assert dev_groups
    for g in dev_groups:
        want = TR.statistics(nodes[g.start:g.stop], edges[g.start:g.stop])
        for name, a, b in zip(g.statistics._fields, g.statistics, want):
            assert a.dtype == np.int64 and np.array_equal(a, b), (g.index, name, a, b)


@pytest.mark.parametrize("case", H.cases())
@pytest.mark.parametrize("chunk", [4096, 1])
def test_group_statistics_match_the_restatement(case, chunk):
    from graphinvent_b200 import preprocess as PP
    layout, nodes, edges, B, _ = H.make_case(case)
    gs = list(PP.groups(nodes, edges, B, *LAYOUTS[layout], chunk_molecules=chunk, statistics=True))
    ref = list(P.groups(nodes, edges, B, P.segments(*LAYOUTS[layout])))
    assert [(g.start, g.stop, g.nodes.shape[0]) for g in gs] == [(r["start"], r["stop"], r["nodes"].shape[0])
                                                                 for r in ref]
    assert_statistics(gs, nodes, edges)
    plain = list(PP.groups(nodes, edges, B, *LAYOUTS[layout], chunk_molecules=chunk))
    assert all(p.statistics is None and np.array_equal(p.apds, g.apds) for p, g in zip(plain, gs))


@pytest.mark.parametrize("N,M,B,chunk,layout", [
    (13, 600, 20, 4096, "gdb13"),      # many groups per chunk
    (13, 600, 20, 45, "gdb13"),        # chunk boundaries inside groups: the cut group re-runs in the next chunk
    (38, 300, 100, 130, "imp_H"),
    (38, 200, 60, 70, "chirality"),
    (38, 200, 30, 40, "imp_H+chirality"),
])
def test_many_groups_and_chunks(N, M, B, chunk, layout):
    from graphinvent_b200 import preprocess as PP
    nodes, edges = H.synthetic(M, N, LAYOUTS[layout], seed=N * 7 + B)
    gs = list(PP.groups(nodes, edges, B, *LAYOUTS[layout], chunk_molecules=chunk, statistics=True))
    assert len(gs) > 3
    assert_statistics(gs, nodes, edges)


def test_guarded_buffers():
    """poisoned workspace and output with guard bands: nothing written outside them, rows past the group count
    untouched, results as the restatement's"""
    from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, lib
    layout, nodes, edges, B, _ = H.make_case("single_atoms_and_hubs")
    M, N, F = nodes.shape
    Ef, max_rows = edges.shape[3], 4000
    d = PPDims(N=N, F=F, Ef=Ef, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=B)
    apd = lib.gib_preprocess_apd_length(ctypes.byref(d))
    ws = Guarded(lib.gib_preprocess_ws_bytes(ctypes.byref(d), M, max_rows))
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    on, oe = Guarded(max_rows * N * F), Guarded(max_rows * N * N * Ef)
    oa, og, st = Guarded(4 * max_rows * apd), Guarded(4 * 4 * M), Guarded(4 * PP_STATUS_INTS)
    sws = Guarded(lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(d), M))
    words = lib.gib_preprocess_group_statistics_bytes(ctypes.byref(d), 1) // 4
    so = Guarded(lib.gib_preprocess_group_statistics_bytes(ctypes.byref(d), M))
    ref = list(P.groups(nodes, edges, B, P.segments(*LAYOUTS[layout])))
    for _ in range(2):                            # the second call finds the first call's workspace
        assert lib.gib_preprocess_chunk(ctypes.byref(d), gn.ptr(), ge.ptr(), M, 1, M, max_rows, ws.ptr(), on.ptr(),
                                        oe.ptr(), oa.ptr(), og.ptr(), st.ptr(), None) == 0
        assert lib.gib_preprocess_group_statistics(ctypes.byref(d), gn.ptr(), ge.ptr(), M, M, og.ptr(), st.ptr(),
                                                   sws.ptr(), so.ptr(), None) == 0
        torch.cuda.synchronize()
        status = st.view(torch.int32).cpu().numpy()
        assert status[0] == len(ref) and status[3] == 0
        out = so.view(torch.int32).cpu().numpy().reshape(M, words)
        groups = og.view(torch.int32).cpu().numpy().reshape(M, 4)
        for g, r in enumerate(ref):
            assert np.array_equal(out[g, :4], groups[g])
            want = np.concatenate(TR.statistics(nodes[r["start"]:r["stop"]], edges[r["start"]:r["stop"]]))
            assert np.array_equal(out[g, 4:], want), g
        assert (out[len(ref):] == -1).all()      # 0xFF poison: rows past the group count are not written
        for gd in (ws, gn, ge, on, oe, oa, og, st, sws, so):
            assert gd.intact(), gd.damage()


# ---- run_data_processer ------------------------------------------------------------------------------------------
@pytest.fixture
def ref(monkeypatch):
    r = MR.load_reference(TR.constants("gdb13", device="cuda"), monkeypatch.setitem)
    if r is None:
        pytest.skip("oracle/_ref holds no Analyzer.py (run __graft_entry__.build() with the reference)")
    return r


def run_stand_in(ref, C, graphs, tmp_path, monkeypatch):
    """run_data_processer(device_properties=True) on a stand-in DataProcesser whose module carries the reference's
    Analyzer; returns its ts_properties and the CSV its util wrote"""
    from graphinvent_b200 import preprocess as PP
    mod = types.ModuleType("stub_ts_data_processer")
    csv_path = tmp_path / "device.csv"
    mod.constants, mod.Analyzer = C, ref.Analyzer.Analyzer
    mod.util = types.SimpleNamespace(
        write_last_molecule_idx=lambda **kw: None,
        write_ts_properties=lambda training_set_properties: TR.write_ts_properties(csv_path, training_set_properties))

    class File:
        def __init__(self, path, mode):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *exc):
            return False
    mod.h5py = types.SimpleNamespace(File=File)

    class DataProcesser:
        path, is_training_set, molecule_set = str(tmp_path / "train.smi"), True, list(range(len(graphs)))

        def get_graph(self, m):
            return graphs[m]

        def start_new_preprocessing_job(self):
            self.resume_idx, self.skip_collection = 0, False

        def save_group(self, **kw):
            pass

        def get_ts_properties(self, **kw):
            raise AssertionError("the device path computes the properties itself")

        def resize_datasets(self):
            pass

        def resave_datasets_unchunked(self):
            pass
    DataProcesser.__module__ = mod.__name__
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    dp = DataProcesser()
    PP.run_data_processer(dp, chunk_molecules=64, device_properties=True)
    return dp.ts_properties, csv_path


@pytest.mark.parametrize("case", ["single_atoms_and_hubs", "cut_groups", "one_group", "unique_smiles",
                                  "imp_H+chirality"])
def test_run_data_processer_matches_the_reference_loop(ref, monkeypatch, tmp_path, case):
    layout, nodes, edges, B, keys = H.make_case(case)
    C = TR.constants(layout, nodes.shape[1], edges.shape[3], B, device="cuda", dataset_dir=str(tmp_path) + "/")
    MR.set_constants(ref, C)
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges, keys)
    spans = [(g["start"], g["stop"]) for g in P.groups(nodes, edges, B, P.segments(*LAYOUTS[layout]))]
    want = TR.reference_ts_properties(ref, graphs, spans, B)
    TR.write_ts_properties(tmp_path / "reference.csv", want)
    got, csv_path = run_stand_in(ref, C, graphs, tmp_path, monkeypatch)
    TR.assert_identical(got, want)
    if case == "one_group":
        assert got[("Training set", "n_nodes_hist")].is_cuda
    assert csv_path.read_bytes() == (tmp_path / "reference.csv").read_bytes()


def test_gdb13_train_csv(ref, monkeypatch, tmp_path):
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges, B = z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"], int(z["gdb13_1K_train/batch_size"])
    C = TR.constants("gdb13", 13, 3, B, device="cuda", dataset_dir=str(tmp_path) + "/")
    MR.set_constants(ref, C)
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges)
    got, csv_path = run_stand_in(ref, C, graphs, tmp_path, monkeypatch)
    assert TR.parse_csv(csv_path) == TR.parse_csv(os.path.join(GOLDEN, "gdb13_1K_train.csv"))
