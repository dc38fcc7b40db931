"""
Training sets built on the device: the decoding routes, target APDs and per-group deduplication of the reference's
`DataProcesser` (DataProcesser.py:60-117, 167-271, 340-361, 434-457; MolecularGraph.py:463-555, 635-732).

The reference expands every molecule into its `n_edges + 2` route states and deduplicates them per group of
`batch_size` rows with a Python scan of every row so far, quadratic per group.  `groups()` runs the same construction
as `gib_preprocess_chunk` (csrc/preprocess.cu) over chunks of molecules and yields the groups in order with the rows
the reference's `save_group` writes, byte for byte, and its `resume_idx` / `dataset_size` counters.

`run_data_processer(dp)` drives a reference `DataProcesser` through the device pass: the `PreprocessingGraph`s are
built once on the host with the caller's RDKit (the reference's own `get_graph`), and the HDF5 writing, the int64 ->
int8 conversion and the final resize / resave stay the reference's own methods.  The training-set properties are the
reference's `get_ts_properties` per group, or, with `device_properties=True`, each group's integer statistics from
`gib_preprocess_group_statistics` (`groups(..., statistics=True)`) turned into the dict `get_molecular_properties`
returns and merged by the reference's own `combine_ts_properties`.
"""
import ctypes
import sys
from collections import namedtuple

import numpy as np
import torch

from ._lib import (PP_BAD_EDGES, PP_BAD_NODES, PP_DISCONNECTED, PP_EMPTY, PP_STATUS_INTS, PPDims, check, lib)

Group = namedtuple("Group", "index init_idx start stop full nodes edges apds resume_idx dataset_size statistics",
                   defaults=(None,))
Group.__doc__ = """One group as `DataProcesser.get_subgraphs` saves it.
index, init_idx: the group's number and its first row in the chunked file (index * batch_size)
start, stop: the molecules [start, stop) it visited, the one whose route was cut included
full: it reached batch_size rows (the rest of molecule stop - 1's route was dropped)
nodes int8 [r, N, F], edges int8 [r, N, N, Ef], apds int32 [r, apd] (APD counts): its r rows
resume_idx, dataset_size: the reference's counters after the group
statistics: the group's `Statistics` (groups(..., statistics=True)), else None"""

Statistics = namedtuple("Statistics", "n_nodes_hist node_sums n_edges_hist bonds")
Statistics.__doc__ = """Integer (int64) sums over a group's molecules [start, stop), gib_preprocess_group_statistics:
n_nodes_hist [N+1]: molecules per atom count;  node_sums [F]: node-feature column sums;
n_edges_hist [10]: atoms per bond count as Analyzer bins them (above 10 -> bin 9, no bond -> bin 9);
bonds [Ef]: bonds per type"""

_REASONS = ((PP_BAD_NODES, "a node row that is not one-hot per segment with 0/1 entries, or a zero row between atoms"),
            (PP_BAD_EDGES, "edges that are not symmetric 0/1 single-type bonds between its atoms"),
            (PP_EMPTY, "no atoms"),
            (PP_DISCONNECTED, "a decoding route that disconnects (the reference's truncate_graph raises)"))


def refuse_bad(status, start, stop):
    """raises the ValueError naming the first bad molecule of the chunk [start, stop) whose status words (GIB_PP_*
    flags in [3], the molecule in [4]) are `status`"""
    if status[3]:
        why = "; ".join(r for bit, r in _REASONS if status[3] & bit)
        raise ValueError(f"molecule {start + int(status[4])} (or a later one in molecules [{start}, {stop})): {why}")


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def layout_of(constants):
    """(n_atom_types, n_formal_charge, n_imp_H, n_chirality) of the reference constants, 0 for an absent segment"""
    C = constants
    imp = not C.use_explicit_H and not C.ignore_H
    return C.n_atom_types, C.n_formal_charge, C.n_imp_H if imp else 0, C.n_chirality if C.use_chirality else 0


def stacks(graphs):
    """int8 (nodes [n, N, F], edges [n, N, N, Ef]) of the reference's padded `PreprocessingGraph`s"""
    nodes = np.stack([np.asarray(g.node_features) for g in graphs])
    edges = np.stack([np.asarray(g.edge_features) for g in graphs])
    out = nodes.astype(np.int8), edges.astype(np.int8)
    if not (np.array_equal(out[0], nodes) and np.array_equal(out[1], edges)):
        raise ValueError("graph features are not int8-exact")
    return out


def groups(nodes, edges, batch_size, n_atom_types, n_formal_charge, n_imp_H=0, n_chirality=0,
           chunk_molecules=4096, max_rows=None, device="cuda", statistics=False):
    """Yields the `Group`s of the molecules `nodes` [M, N, F] / `edges` [M, N, N, Ef] (int8, padded, decoding order).
    The layout is the node-feature segment widths (0: segment absent; `config.layout_dims` gives them).  Molecules go
    to the device `chunk_molecules` (at least batch_size) at a time; `max_rows` (at least batch_size, default
    16 * chunk) bounds the rows one chunk call writes.  statistics=True: each group also carries its `Statistics`,
    computed on the device after each chunk and copied back with the group table."""
    nodes = np.ascontiguousarray(nodes)
    edges = np.ascontiguousarray(edges)
    if nodes.dtype != np.int8 or edges.dtype != np.int8 or nodes.ndim != 3 or edges.ndim != 4:
        raise ValueError("nodes / edges must be int8 [M, N, F] / [M, N, N, Ef]")
    M, N, F = nodes.shape
    Ef = edges.shape[3]
    if edges.shape[:3] != (M, N, N):
        raise ValueError(f"edges {edges.shape} do not match nodes {nodes.shape}")
    d = PPDims(N=N, F=F, Ef=Ef, n_atom_types=n_atom_types, n_formal_charge=n_formal_charge, n_imp_H=n_imp_H,
               n_chirality=n_chirality, batch_size=batch_size)
    apd_len = lib.gib_preprocess_apd_length(ctypes.byref(d))
    if apd_len < 0:
        raise ValueError(lib.gib_last_error().decode())
    if M == 0:
        return
    B = batch_size
    chunk = min(max(int(chunk_molecules), B), M)
    max_rows = max(int(max_rows or 16 * chunk), B)
    ws_bytes = lib.gib_preprocess_ws_bytes(ctypes.byref(d), chunk, max_rows)
    if ws_bytes == 0:
        raise ValueError(lib.gib_last_error().decode())
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("graphinvent_b200.preprocess runs on a CUDA device (no CPU fallback)")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    in_nodes = torch.empty((chunk, N, F), dtype=torch.int8, device=dev)
    in_edges = torch.empty((chunk, N, N, Ef), dtype=torch.int8, device=dev)
    out_nodes = torch.empty((max_rows, N, F), dtype=torch.int8, device=dev)
    out_edges = torch.empty((max_rows, N, N, Ef), dtype=torch.int8, device=dev)
    out_apds = torch.empty((max_rows, apd_len), dtype=torch.int32, device=dev)
    out_groups = torch.empty((chunk, 4), dtype=torch.int32, device=dev)
    status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=dev)
    if statistics:
        words = lib.gib_preprocess_group_statistics_bytes(ctypes.byref(d), 1) // 4
        if words == 0:
            raise ValueError(lib.gib_last_error().decode())
        stats_ws = torch.empty(lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(d), chunk),
                               dtype=torch.uint8, device=dev)
        stats_out = torch.empty((chunk, words), dtype=torch.int32, device=dev)
        splits = np.cumsum([N + 1, F, 10])
    stream = torch.cuda.current_stream(dev)
    pos, g, size = 0, 0, 0
    while pos < M:
        stop = min(pos + chunk, M)
        n = stop - pos
        in_nodes[:n].copy_(torch.from_numpy(nodes[pos:stop]))
        in_edges[:n].copy_(torch.from_numpy(edges[pos:stop]))
        check(lib.gib_preprocess_chunk(ctypes.byref(d), _ptr(in_nodes), _ptr(in_edges), n, int(stop == M), chunk,
                                       max_rows, _ptr(ws), _ptr(out_nodes), _ptr(out_edges), _ptr(out_apds),
                                       _ptr(out_groups), _ptr(status), ctypes.c_void_p(stream.cuda_stream)),
              "gib_preprocess_chunk")
        if statistics:
            check(lib.gib_preprocess_group_statistics(ctypes.byref(d), _ptr(in_nodes), _ptr(in_edges), n, chunk,
                                                      _ptr(out_groups), _ptr(status), _ptr(stats_ws), _ptr(stats_out),
                                                      ctypes.c_void_p(stream.cuda_stream)),
                  "gib_preprocess_group_statistics")
        st = status.cpu().numpy()
        refuse_bad(st, pos, stop)
        ng, nxt, rows = int(st[0]), int(st[1]), int(st[2])
        if ng == 0:
            raise RuntimeError("gib_preprocess_chunk completed no group")
        gr = (stats_out if statistics else out_groups)[:ng].cpu().numpy()
        on, oe, oa = out_nodes[:rows].cpu().numpy(), out_edges[:rows].cpu().numpy(), out_apds[:rows].cpu().numpy()
        for row in gr:
            s, e, r0, r = row[:4].tolist()
            full = r == B
            size += B if full else e - s
            stats = Statistics(*np.split(row[4:].astype(np.int64), splits)) if statistics else None
            yield Group(g, g * B, pos + s, pos + e, full, on[r0:r0 + r], oe[r0:r0 + r], oa[r0:r0 + r], pos + e,
                        size, stats)
            g += 1
        pos += nxt


def ts_properties(stats, smiles, constants):
    """The dict `Analyzer.get_molecular_properties(graphs, "Training set")` returns for a group's `PreprocessingGraph`s
    (Analyzer.py:311-599), from the group's `Statistics` and the graphs' `get_smiles()`: the same keys in the same
    order, value types, dtypes and devices.  The histograms hold integer counts, exact in float32; the averages are
    the reference's own float32 tensor divisions, of sums that are exact below 2**24."""
    C = constants
    dev = C.device
    key = "Training set"
    n_graphs = len(smiles)
    n_nodes_hist = torch.tensor(stats.n_nodes_hist, dtype=torch.float32, device=dev)
    sum_n_nodes = int(np.dot(np.arange(stats.n_nodes_hist.size), stats.n_nodes_hist))
    avg_n_nodes = torch.tensor(sum_n_nodes, dtype=torch.float32, device=dev) / n_graphs
    nodes_hist = stats.node_sums.astype(np.float64)                # np.sum of the float64 node features
    ends = np.cumsum([w for w in layout_of(C) if w]).tolist()      # util.get_feature_vector_indices
    imp = not C.use_explicit_H and not C.ignore_H
    numh_hist = nodes_hist[ends[1]:ends[2]] if imp else [0] * C.n_imp_H
    chirality_hist = nodes_hist[ends[1 + imp]:ends[2 + imp]] if C.use_chirality else [0] * C.n_chirality
    n_edges_hist = torch.tensor(stats.n_edges_hist, dtype=torch.float32, device=dev)
    sum_n_edges = int(np.dot(np.arange(1, 11), stats.n_edges_hist))
    avg_n_edges = torch.tensor(sum_n_edges, dtype=torch.float32, device=dev) / torch.sum(n_edges_hist, dim=0)
    edge_feature_hist = torch.tensor(stats.bonds, dtype=torch.float32, device=dev)
    unique = set(smiles)
    unique.discard(None)
    fraction_unique = len(unique) / n_graphs if n_graphs else 0
    return {(key, "n_nodes_hist"): n_nodes_hist,
            (key, "avg_n_nodes"): avg_n_nodes,
            (key, "atom_type_hist"): nodes_hist[:ends[0]],
            (key, "formal_charge_hist"): nodes_hist[ends[0]:ends[1]],
            (key, "n_edges_hist"): n_edges_hist,
            (key, "avg_n_edges"): avg_n_edges,
            (key, "edge_feature_hist"): edge_feature_hist,
            (key, "fraction_unique"): fraction_unique,
            (key, "fraction_valid"): 1.0,
            (key, "fraction_valid_properly_terminated"): 1.0,
            (key, "fraction_properly_terminated"): 1.0,
            (key, "numh_hist"): numh_hist,
            (key, "chirality_hist"): chirality_hist}


def merge_ts_properties(analyzer, prev, props, batch_size):
    """DataProcesser.get_ts_properties' merge of a group's properties into the running ones (`prev`, None before the
    first group): the first as it is, a later one through `analyzer.combine_ts_properties` with weight batch_size"""
    if not prev:
        return props
    return analyzer.combine_ts_properties(prev_properties=prev, next_properties=props, weight_next=batch_size)


def run_data_processer(dp, chunk_molecules=4096, device="cuda", device_properties=False):
    """`dp.preprocess()` of a reference `DataProcesser` with `get_subgraphs` replaced by the device pass.  The
    reference module's `constants`, `util` and `h5py` are the ones `dp`'s class was defined with.  Restarting a preprocessing
    job (`constants.restart`) is not supported.

    device_properties=False: the training-set properties are `dp.get_ts_properties` over each group's graphs.
    device_properties=True: they come from the device statistics of each group (`ts_properties`), merged as
    `get_ts_properties` merges them -- the first group's dict as it is, each later one through the module's
    `Analyzer.combine_ts_properties` with weight batch_size -- on one Analyzer made without `__init__` (no TensorBoard
    writer per group).  Only the training set gets properties, as in the reference."""
    mod = sys.modules[type(dp).__module__]
    C, util, h5py = mod.constants, mod.util, mod.h5py
    if C.restart:
        raise NotImplementedError("run_data_processer starts a new preprocessing job; constants.restart is set")
    graphs = [dp.get_graph(mol) for mol in dp.molecule_set]
    nodes, edges = stacks(graphs)
    on_device = device_properties and dp.is_training_set
    if on_device:
        smiles = [g.get_smiles() for g in graphs]
        analyzer = mod.Analyzer.__new__(mod.Analyzer)
    with h5py.File(f"{dp.path[:-3]}h5.chunked", "a") as dp.hdf_file:
        dp.restart_index_file = C.dataset_dir + "index.restart"
        dp.start_new_preprocessing_job()
        dp.dataset_size = 0
        dp.ts_properties = None
        for grp in groups(nodes, edges, C.batch_size, *layout_of(C), chunk_molecules=chunk_molecules, device=device,
                          statistics=on_device):
            dp.save_group(data_subgraphs=list(zip(grp.nodes, grp.edges)), data_apds=list(grp.apds.astype(np.int64)),
                          group_size=grp.nodes.shape[0], init_idx=grp.init_idx)
            if on_device:
                props = ts_properties(grp.statistics, smiles[grp.start:grp.stop], C)
                dp.ts_properties = merge_ts_properties(analyzer, dp.ts_properties, props, C.batch_size)
            else:
                dp.get_ts_properties(molecular_graphs=graphs[grp.start:grp.stop], group_size=C.batch_size)
            dp.resume_idx, dp.dataset_size = grp.resume_idx, grp.dataset_size
            util.write_last_molecule_idx(last_molecule_idx=dp.resume_idx, dataset_size=dp.dataset_size,
                                         restart_file_path=C.dataset_dir)
        dp.resize_datasets()
        if dp.is_training_set:
            util.write_ts_properties(training_set_properties=dp.ts_properties)
    dp.resave_datasets_unchunked()
