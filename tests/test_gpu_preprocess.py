"""GPU: the training-set construction of graphinvent_b200.preprocess (csrc/preprocess.cu) against the numpy
restatement of the reference (tests/preprocess_reference.py) and the reference's shipped gdb13 files
(tests/golden/preprocess_gdb13.npz): rows, APD counts, group molecule ranges and counters, bit for bit."""
import ctypes
import hashlib
import os
import types

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests.conftest import GOLDEN
from tests.guarded import Guarded

pytestmark = pytest.mark.gpu

LAYOUTS = {"gdb13": (5, 3, 0, 0), "imp_H": (5, 3, 4, 0), "chirality": (5, 3, 0, 3), "imp_H+chirality": (4, 3, 4, 3)}


def graphs(M, N, layout, Ef=3, seed=0, min_atoms=1):
    """seeded synthetic molecules (graphinvent_b200.synthetic) with the layout's implicit-H / chirality segments"""
    from graphinvent_b200 import synthetic as S
    A, Fc, H, C = layout
    nodes, edges = S.random_graphs(M, N, A, Fc, n_edge_features=Ef, seed=seed, min_atoms=min_atoms)
    rng = np.random.default_rng(seed + 1)
    extra = []
    for w in (H, C):
        if w:
            seg = np.zeros((M, N, w), np.int8)
            present = nodes.any(2)
            seg[present, rng.integers(0, w, int(present.sum()))] = 1
            extra.append(seg)
    return np.concatenate([nodes] + extra, axis=2), edges


def device_groups(nodes, edges, B, layout, **kw):
    from graphinvent_b200 import preprocess as PP
    return list(PP.groups(nodes, edges, B, *layout, **kw))


def assert_same(dev, ref):
    assert len(dev) == len(ref)
    for d, r in zip(dev, ref):
        assert (d.index, d.init_idx, d.start, d.stop, d.full, d.resume_idx, d.dataset_size) == \
            (r["index"], r["init_idx"], r["start"], r["stop"], r["full"], r["resume_idx"], r["dataset_size"]), d.index
        assert d.nodes.dtype == np.int8 and d.edges.dtype == np.int8 and d.apds.dtype == np.int32
        assert np.array_equal(d.nodes, r["nodes"]), d.index
        assert np.array_equal(d.edges, r["edges"]), d.index
        assert np.array_equal(d.apds, r["apds"]), d.index


def segs_of(layout):
    return P.segments(*layout)


@pytest.mark.parametrize("key", ["gdb13_1K_train", "gdb13_1K_debug_train", "gdb13_1K_debug_valid"])
@pytest.mark.parametrize("chunk", [4096, 1])
def test_gdb13_files_rebuilt_byte_for_byte(key, chunk):
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    X, E, B = z[f"{key}/nodes"], z[f"{key}/edges"], int(z[f"{key}/batch_size"])
    gs = device_groups(X, E, B, LAYOUTS["gdb13"], chunk_molecules=chunk)
    got = np.array([[g.start, g.stop, g.init_idx, g.nodes.shape[0], g.resume_idx, g.dataset_size] for g in gs])
    assert np.array_equal(got, z[f"{key}/counters"])
    ref = [dict(init_idx=g.init_idx, nodes=g.nodes, edges=g.edges, apds=g.apds.astype(np.int64)) for g in gs]
    nodes, edges, apds = P.assemble(ref, len(gs) * B, 13, 8, 3, 625)
    blob = z[f"{key}/header"].tobytes() + apds.tobytes() + edges.tobytes() + nodes.tobytes()
    assert hashlib.sha256(blob).hexdigest() == str(z[f"{key}/sha256"])


@pytest.mark.parametrize("N,M,B,chunk,Ef,layout", [
    (13, 300, 1000, 4096, 3, "gdb13"),
    (13, 300, 50, 64, 3, "gdb13"),            # chunk boundaries inside groups
    (13, 120, 7, 7, 4, "gdb13"),              # Ef = 4, smallest chunk
    (13, 40, 1, 16, 3, "gdb13"),              # B = 1
    (38, 200, 1000, 4096, 3, "gdb13"),
    (38, 150, 100, 128, 3, "imp_H"),
    (38, 120, 60, 70, 3, "chirality"),
    (38, 120, 30, 40, 4, "imp_H+chirality"),
    (90, 24, 200, 4096, 3, "gdb13"),
    (90, 24, 64, 64, 1, "gdb13"),
])
def test_matches_restatement(N, M, B, chunk, Ef, layout):
    L = LAYOUTS[layout]
    nodes, edges = graphs(M, N, L, Ef=Ef, seed=N * 1000 + B)
    ref = list(P.groups(nodes, edges, B, segs_of(L)))
    assert_same(device_groups(nodes, edges, B, L, chunk_molecules=chunk), ref)


@pytest.mark.parametrize("B,chunk", [(1000, 1000), (5, 8), (1, 1)])
def test_identical_molecules(B, chunk):
    """every molecule the same: a group of batch_size 1000 never fills before its molecules run out"""
    nodes, edges = graphs(1, 13, LAYOUTS["gdb13"], seed=3)
    nodes, edges = np.repeat(nodes, 1500, 0), np.repeat(edges, 1500, 0)
    ref = list(P.groups(nodes, edges, B, segs_of(LAYOUTS["gdb13"])))
    assert_same(device_groups(nodes, edges, B, LAYOUTS["gdb13"], chunk_molecules=chunk), ref)


def test_quirk_rows_and_single_atoms():
    """a state whose first match is the last row is appended again; single-atom molecules; repeats across groups"""
    nodes, edges = graphs(60, 13, LAYOUTS["gdb13"], seed=5, min_atoms=1)
    nodes = np.concatenate([nodes[:5], nodes[:5], nodes[2:3], nodes[5:]])
    edges = np.concatenate([edges[:5], edges[:5], edges[2:3], edges[5:]])
    for B in (3, 17, 40):
        ref = list(P.groups(nodes, edges, B, segs_of(LAYOUTS["gdb13"])))
        assert_same(device_groups(nodes, edges, B, LAYOUTS["gdb13"], chunk_molecules=B), ref)


def test_invalid_molecules_are_refused():
    nodes, edges = graphs(8, 13, LAYOUTS["gdb13"], seed=9, min_atoms=3)
    n2, e2 = nodes.copy(), edges.copy()
    k = P.n_atoms(n2[4])
    e2[4, :, k - 1] = 0                           # the last atom loses its bonds: the route disconnects
    e2[4, k - 1, :] = 0
    with pytest.raises(ValueError, match="disconnects"):
        device_groups(n2, e2, 10, LAYOUTS["gdb13"])
    n3 = nodes.copy()
    n3[2, 0, :5] = 1                              # two atom types
    with pytest.raises(ValueError, match="molecule 2"):
        device_groups(n3, edges, 10, LAYOUTS["gdb13"])
    e4 = edges.copy()
    e4[6, 0, 1, 2] = 1 - e4[6, 0, 1, 2]           # asymmetric
    with pytest.raises(ValueError, match="symmetric"):
        device_groups(nodes, e4, 10, LAYOUTS["gdb13"])


def test_guarded_buffers():
    """poisoned workspace and outputs with guard bands: nothing written outside them, results as with fresh buffers"""
    from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, lib
    N, F, Ef, B, M, max_rows = 13, 8, 3, 40, 90, 2000
    nodes, edges = graphs(M, N, LAYOUTS["gdb13"], seed=11)
    d = PPDims(N=N, F=F, Ef=Ef, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=B)
    apd = lib.gib_preprocess_apd_length(ctypes.byref(d))
    ws = Guarded(lib.gib_preprocess_ws_bytes(ctypes.byref(d), M, max_rows))
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    on, oe = Guarded(max_rows * N * F), Guarded(max_rows * N * N * Ef)
    oa, og, st = Guarded(4 * max_rows * apd), Guarded(4 * 4 * M), Guarded(4 * PP_STATUS_INTS)
    for _ in range(2):                            # the second call finds the first call's workspace
        rc = lib.gib_preprocess_chunk(ctypes.byref(d), gn.ptr(), ge.ptr(), M, 1, M, max_rows, ws.ptr(), on.ptr(),
                                      oe.ptr(), oa.ptr(), og.ptr(), st.ptr(), None)
        assert rc == 0
        torch.cuda.synchronize()
        status = st.view(torch.int32).cpu().numpy()
        ref = list(P.groups(nodes, edges, B, segs_of(LAYOUTS["gdb13"])))
        rows = sum(r["nodes"].shape[0] for r in ref)
        assert status[0] == len(ref) and status[1] == M and status[2] == rows and status[3] == 0
        assert np.array_equal(on.view(torch.int8)[:rows * N * F].cpu().numpy(),
                              np.concatenate([r["nodes"] for r in ref]).ravel())
        assert np.array_equal(oe.view(torch.int8)[:rows * N * N * Ef].cpu().numpy(),
                              np.concatenate([r["edges"] for r in ref]).ravel())
        assert np.array_equal(oa.view(torch.int32)[:rows * apd].cpu().numpy(),
                              np.concatenate([r["apds"] for r in ref]).ravel())
        for g in (ws, gn, ge, on, oe, oa, og, st):
            assert g.intact(), g.damage()


def test_run_data_processer_writes_the_reference_arrays(tmp_path):
    """the helper drives a stand-in DataProcesser exactly as preprocess() does: the same save_group calls, counters,
    ts-properties calls, restart-file writes and the final resize / resave"""
    from graphinvent_b200 import preprocess as PP
    N, B, M = 13, 25, 70
    nodes, edges = graphs(M, N, LAYOUTS["gdb13"], seed=21)
    ref = list(P.groups(nodes, edges, B, segs_of(LAYOUTS["gdb13"])))
    total = P.total_subgraphs(edges)
    C = types.SimpleNamespace(restart=False, dataset_dir=str(tmp_path) + "/", batch_size=B, n_atom_types=5,
                              n_formal_charge=3, n_imp_H=0, n_chirality=0, use_explicit_H=False, ignore_H=True,
                              use_chirality=False)
    calls = []
    util = types.SimpleNamespace(
        write_last_molecule_idx=lambda **kw: calls.append(("restart", kw["last_molecule_idx"], kw["dataset_size"])),
        write_ts_properties=lambda **kw: calls.append(("ts", None, None)))
    mod = types.ModuleType("stub_data_processer")
    mod.constants, mod.util = C, util

    class File:
        def __init__(self, path, mode):
            calls.append(("open", path[len(str(tmp_path)):], mode))

        def __enter__(self):
            return self

        def __exit__(self, *exc):
            return False
    mod.h5py = types.SimpleNamespace(File=File)

    class Graph:
        def __init__(self, m):
            self.node_features, self.edge_features = nodes[m].astype(np.float64), edges[m].astype(np.float64)

    class DataProcesser:
        def __init__(self):
            self.path, self.is_training_set, self.molecule_set = str(tmp_path / "train.smi"), True, list(range(M))
            self.file = dict(nodes=np.zeros((total, N, 8), np.int8), edges=np.zeros((total, N, N, 3), np.int8),
                             APDs=np.zeros((total, 625), np.int8))

        def get_graph(self, m):
            return Graph(m)

        def start_new_preprocessing_job(self):
            self.resume_idx, self.skip_collection = 0, False

        def save_group(self, data_subgraphs, data_apds, group_size, init_idx):
            a = np.array(data_apds)
            assert a.dtype == np.int64
            self.file["nodes"][init_idx:init_idx + group_size] = np.array([s[0] for s in data_subgraphs])
            self.file["edges"][init_idx:init_idx + group_size] = np.array([s[1] for s in data_subgraphs])
            self.file["APDs"][init_idx:init_idx + group_size] = a
            calls.append(("save", init_idx, group_size))

        def get_ts_properties(self, molecular_graphs, group_size):
            calls.append(("props", len(molecular_graphs), group_size))

        def resize_datasets(self):
            calls.append(("resize", self.resume_idx, self.dataset_size))

        def resave_datasets_unchunked(self):
            calls.append(("resave", None, None))

    DataProcesser.__module__ = mod.__name__
    import sys
    sys.modules[mod.__name__] = mod
    try:
        dp = DataProcesser()
        PP.run_data_processer(dp)
    finally:
        del sys.modules[mod.__name__]
    want = [("open", "/train.h5.chunked", "a")]
    for r in ref:
        want += [("save", r["init_idx"], r["nodes"].shape[0]), ("props", r["stop"] - r["start"], B),
                 ("restart", r["resume_idx"], r["dataset_size"])]
    want += [("resize", M, ref[-1]["dataset_size"]), ("ts", None, None), ("resave", None, None)]
    assert calls == want
    n, e, a = P.assemble(ref, total, N, 8, 3, 625)
    assert np.array_equal(dp.file["nodes"], n) and np.array_equal(dp.file["edges"], e)
    assert np.array_equal(dp.file["APDs"], a)
