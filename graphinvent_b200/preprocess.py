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

`reorder()` is the reference's choice of decoding route, `PreprocessingGraph.node_remap`, on the device
(`gib_reorder`): a BFS or DFS from a node ranking -- given, or drawn per (seed, epoch, molecule) -- and the reordered
stacks.  `file_rows()` runs the construction of `groups()` with the rows left on the device, laid out as the file
`run_data_processer` writes; `loader.RandomRouteLoader` builds every training pass from fresh routes with the two.

`scaffold_first()` finds each molecule's scaffold (`gib_scaffold_first`) and puts it first in decoding order, the
order the conditional route scorer and the scaffold decorators need.

`murcko_scaffolds()` extracts each molecule's Bemis-Murcko scaffold (`gib_murcko`) and deduplicates them into the
scaffold table, with counts and observed attachment points, that `scaffold_first` and the decorators take.
"""
import ctypes
import sys
from collections import namedtuple

import numpy as np
import torch

from ._lib import (PP_BAD_EDGES, PP_BAD_NODES, PP_BAD_RANKING, PP_DISCONNECTED, PP_EMPTY, PP_MATCH_BUDGET,
                   PP_STATUS_INTS, ROUTE_BFS, ROUTE_DFS, PPDims, check, lib)

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


def refuse_bad(status, start, stop, reasons=_REASONS):
    """raises the ValueError naming the first bad molecule of the chunk [start, stop) whose status words (GIB_PP_*
    flags in [3], the molecule in [4]) are `status`"""
    if status[3]:
        why = "; ".join(r for bit, r in reasons if status[3] & bit)
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
    M, N, F, Ef = _check_stacks(nodes, edges)
    d = _pp_dims(N, F, Ef, (n_atom_types, n_formal_charge, n_imp_H, n_chirality), batch_size)
    if M == 0:
        return
    B = batch_size
    chunk, max_rows = _chunk_sizes(d, M, chunk_molecules, max_rows)
    dev = _cuda(torch.device(device))
    in_nodes = torch.empty((chunk, N, F), dtype=torch.int8, device=dev)
    in_edges = torch.empty((chunk, N, N, Ef), dtype=torch.int8, device=dev)

    def inputs(pos, stop):
        in_nodes[:stop - pos].copy_(torch.from_numpy(nodes[pos:stop]))
        in_edges[:stop - pos].copy_(torch.from_numpy(edges[pos:stop]))
        return in_nodes, in_edges

    if statistics:
        splits = np.cumsum([N + 1, F, 10])
    g, size = 0, 0
    for pos, table, (out_nodes, out_edges, out_apds), rows in _chunks(d, M, chunk, max_rows, dev, inputs,
                                                                      statistics):
        on, oe, oa = out_nodes[:rows].cpu().numpy(), out_edges[:rows].cpu().numpy(), out_apds[:rows].cpu().numpy()
        for row in table:
            s, e, r0, r = row[:4].tolist()
            full = r == B
            size += B if full else e - s
            stats = Statistics(*np.split(row[4:].astype(np.int64), splits)) if statistics else None
            yield Group(g, g * B, pos + s, pos + e, full, on[r0:r0 + r], oe[r0:r0 + r], oa[r0:r0 + r], pos + e,
                        size, stats)
            g += 1


def _cuda(dev):
    if dev.type != "cuda":
        raise RuntimeError("graphinvent_b200.preprocess runs on a CUDA device (no CPU fallback)")
    return dev


def _chunks(d, M, chunk, max_rows, dev, inputs, statistics=False):
    """gib_preprocess_chunk over molecules [0, M) in chunks of at most `chunk`; inputs(pos, stop) gives the chunk's
    molecules as int8 device tensors whose first stop - pos rows are molecules [pos, stop).  Yields per chunk the
    first molecule, the host group table (int32 [groups, 4], or with statistics [groups, 4 + statistics words]) and the
    device output buffers (out_nodes, out_edges, out_apds), valid until the next chunk runs, and the rows written."""
    apd_len = lib.gib_preprocess_apd_length(ctypes.byref(d))
    ws = torch.empty(lib.gib_preprocess_ws_bytes(ctypes.byref(d), chunk, max_rows), dtype=torch.uint8, device=dev)
    N, F, Ef = d.N, d.F, d.Ef
    out = (torch.empty((max_rows, N, F), dtype=torch.int8, device=dev),
           torch.empty((max_rows, N, N, Ef), dtype=torch.int8, device=dev),
           torch.empty((max_rows, apd_len), dtype=torch.int32, device=dev))
    out_groups = torch.empty((chunk, 4), dtype=torch.int32, device=dev)
    status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=dev)
    if statistics:
        words = lib.gib_preprocess_group_statistics_bytes(ctypes.byref(d), 1) // 4
        if words == 0:
            raise ValueError(lib.gib_last_error().decode())
        stats_ws = torch.empty(lib.gib_preprocess_group_statistics_ws_bytes(ctypes.byref(d), chunk),
                               dtype=torch.uint8, device=dev)
        stats_out = torch.empty((chunk, words), dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev)
    pos = 0
    while pos < M:
        stop = min(pos + chunk, M)
        n = stop - pos
        in_nodes, in_edges = inputs(pos, stop)
        check(lib.gib_preprocess_chunk(ctypes.byref(d), _ptr(in_nodes), _ptr(in_edges), n, int(stop == M), chunk,
                                       max_rows, _ptr(ws), *map(_ptr, out), _ptr(out_groups), _ptr(status),
                                       ctypes.c_void_p(stream.cuda_stream)),
              "gib_preprocess_chunk")
        if statistics:
            check(lib.gib_preprocess_group_statistics(ctypes.byref(d), _ptr(in_nodes), _ptr(in_edges), n, chunk,
                                                      _ptr(out_groups), _ptr(status), _ptr(stats_ws), _ptr(stats_out),
                                                      ctypes.c_void_p(stream.cuda_stream)),
                  "gib_preprocess_group_statistics")
        st = status.cpu().numpy()
        refuse_bad(st, pos, stop)
        ng, nxt = int(st[0]), int(st[1])
        if ng == 0:
            raise RuntimeError("gib_preprocess_chunk completed no group")
        yield pos, (stats_out if statistics else out_groups)[:ng].cpu().numpy(), out, int(st[2])
        pos += nxt


def _check_stacks(nodes, edges):
    """(M, N, F, Ef) of int8 stacks nodes [M, N, F] / edges [M, N, N, Ef]"""
    if nodes.dtype not in (np.int8, torch.int8) or edges.dtype not in (np.int8, torch.int8) or nodes.ndim != 3 \
            or edges.ndim != 4:
        raise ValueError("nodes / edges must be int8 [M, N, F] / [M, N, N, Ef]")
    M, N, F = nodes.shape
    if tuple(edges.shape[:3]) != (M, N, N):
        raise ValueError(f"edges {tuple(edges.shape)} do not match nodes {tuple(nodes.shape)}")
    return M, N, F, edges.shape[3]


def _on_device(x, device):
    t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
    return t.to(_cuda(torch.device(device))).contiguous()


def _pp_dims(N, F, Ef, layout, batch_size=1):
    d = PPDims(N=N, F=F, Ef=Ef, n_atom_types=layout[0], n_formal_charge=layout[1], n_imp_H=layout[2],
               n_chirality=layout[3], batch_size=batch_size)
    if lib.gib_preprocess_apd_length(ctypes.byref(d)) < 0:
        raise ValueError(lib.gib_last_error().decode())
    return d


def _chunk_sizes(d, M, chunk_molecules, max_rows):
    """(chunk, max_rows) of the training-set construction over M >= 1 molecules: chunks of at least batch_size
    molecules, max_rows at least batch_size (default 16 * chunk), checked by gib_preprocess_ws_bytes"""
    B = d.batch_size
    chunk = min(max(int(chunk_molecules), B), M)
    max_rows = max(int(max_rows or 16 * chunk), B)
    if lib.gib_preprocess_ws_bytes(ctypes.byref(d), chunk, max_rows) == 0:
        raise ValueError(lib.gib_last_error().decode())
    return chunk, max_rows


def file_rows(nodes, edges, batch_size, n_atom_types, n_formal_charge, n_imp_H=0, n_chirality=0,
              chunk_molecules=4096, max_rows=None, keep=True, device="cuda"):
    """The training-set construction of `groups` with its rows left on the device: (nodes, edges, apds), int8 device
    tensors laid out as the file `run_data_processer` writes after its final resize -- each group's rows at
    group * batch_size, APD counts clipped to int8 as h5py stores them, zero rows where no group wrote, and
    `dataset_size` rows in all (the last group adds its molecule count, not its row count, so the file may cut rows
    or end in zero rows).  `nodes` / `edges`: int8 [M, N, F] / [M, N, N, Ef] in decoding order, M >= 1 (device
    tensors are used in place).
    Returns (rows or None with keep=False, dataset_size).  The rows are views of buffers of the file's initial
    length, sum over molecules of (bonds + 2) rows: at N*F + N*N*Ef + apd bytes a row."""
    M, N, F, Ef = _check_stacks(nodes, edges)
    if M == 0:
        raise ValueError("no molecules")
    layout = (n_atom_types, n_formal_charge, n_imp_H, n_chirality)
    d = _pp_dims(N, F, Ef, layout, batch_size)
    nodes, edges = _on_device(nodes, device), _on_device(edges, device)
    B = batch_size
    chunk, max_rows = _chunk_sizes(d, M, chunk_molecules, max_rows)
    dev = nodes.device
    rows = None
    if keep:
        total = int((torch.count_nonzero(edges.view(M, -1), dim=1) // 2 + 2).sum())
        apd_len = lib.gib_preprocess_apd_length(ctypes.byref(d))
        rows = (torch.zeros((total, N, F), dtype=torch.int8, device=dev),
                torch.zeros((total, N, N, Ef), dtype=torch.int8, device=dev),
                torch.zeros((total, apd_len), dtype=torch.int8, device=dev))
    g, size = 0, 0
    for _, table, out, _ in _chunks(d, M, chunk, max_rows, dev,
                                    lambda pos, stop: (nodes[pos:stop], edges[pos:stop])):
        if keep:
            # one copy per run of groups whose rows follow each other both in `out` and in the file: [src, dst, rows]
            runs = []
            for i, (s, e, r0, r) in enumerate(table[:, :4].tolist()):
                if runs and runs[-1][0] + runs[-1][2] == r0 and runs[-1][1] + runs[-1][2] == (g + i) * B:
                    runs[-1][2] += r
                else:
                    runs.append([r0, (g + i) * B, r])
            for src, dst, r in runs:
                r = min(r, total - dst)        # past the file's initial length: cut by the final resize anyway
                if r > 0:
                    rows[0][dst:dst + r].copy_(out[0][src:src + r])
                    rows[1][dst:dst + r].copy_(out[1][src:src + r])
                    rows[2][dst:dst + r].copy_(out[2][src:src + r].clamp(-128, 127))
        for s, e, r0, r in table[:, :4].tolist():
            size += B if r == B else e - s
        g += table.shape[0]
    return (tuple(t[:size] for t in rows) if keep else None), size


def rankings(n_atoms, N, seed=0, epoch=0, first=0, device="cuda"):
    """int32 [M, N] device tensor: the node rankings `reorder` draws for molecules of n_atoms[m] atoms (-1 past
    n_atoms[m]), uniform permutations that depend on (seed, epoch, first + m) only.  `first`: the index of molecule 0
    in the whole set, so that a set drawn in pieces gets the rankings it gets drawn at once.  Draws nothing from
    torch's generators."""
    n = _on_device(torch.as_tensor(np.asarray(n_atoms, np.int32)), device)
    M = n.numel()
    out = torch.empty((M, N), dtype=torch.int32, device=n.device)
    if M:
        check(lib.gib_draw_rankings(M, N, _ptr(n), ctypes.c_ulonglong(seed % 2**64), epoch, first, _ptr(out),
                                    ctypes.c_void_p(torch.cuda.current_stream(n.device).cuda_stream)),
              "gib_draw_rankings")
    return out


_REORDER_REASONS = ((PP_BAD_NODES, "a node row that is not one-hot per segment with 0/1 entries, or a zero row "
                     "between atoms"),
                    (PP_BAD_EDGES, "edges that are not symmetric 0/1 single-type bonds between its atoms"),
                    (PP_EMPTY, "no atoms"),
                    (PP_DISCONNECTED, "a disconnected graph (the reference's searches do not terminate on it)"),
                    (PP_BAD_RANKING, "a ranking that is not a permutation of 0..n-1 over its n atoms"))


def reorder(nodes, edges, route="bfs", rankings=None, seed=0, epoch=0, *, layout, first=0, device="cuda"):
    """`PreprocessingGraph.node_remap` (MolecularGraph.py:435-461) of every molecule of the int8 stacks `nodes`
    [M, N, F] / `edges` [M, N, N, Ef] (numpy or torch, any atom order): `breadth_first_search` (route="bfs") or
    `depth_first_search` ("dfs") from atom ranking[0], then `reorder_nodes`, atom for atom as the reference on
    CPython 3.12.  `rankings`: int32 [M, N] (row m's first n entries a permutation of 0..n-1), or None to draw them on
    the device from (seed, epoch, first + m) as `rankings()` does.  `layout`: the node-feature segment widths
    (n_atom_types, n_formal_charge, n_imp_H, n_chirality), as `groups` takes them (`layout_of(constants)`).
    Returns device tensors (nodes, edges, order): the reordered stacks and int32 [M, N] old atom indices in the new
    order, -1 past the atom count.  Raises ValueError naming the first molecule that `groups` would refuse, that is
    disconnected or empty, or whose ranking is not a permutation."""
    if route not in ("bfs", "dfs"):
        raise ValueError(f"route must be 'bfs' or 'dfs', got {route!r}")
    M, N, F, Ef = _check_stacks(nodes, edges)
    d = _pp_dims(N, F, Ef, tuple(layout))
    nodes, edges = _on_device(nodes, device), _on_device(edges, device)
    dev = nodes.device
    if rankings is None:
        rk = torch.empty((M, N), dtype=torch.int32, device=dev)
    else:
        rk = _on_device(torch.as_tensor(rankings), dev).to(torch.int32)
        if tuple(rk.shape) != (M, N):
            raise ValueError(f"rankings must be [M, N] = {(M, N)}, got {tuple(rk.shape)}")
    out_nodes, out_edges = torch.empty_like(nodes), torch.empty_like(edges)
    order = torch.empty((M, N), dtype=torch.int32, device=dev)
    if M == 0:
        return out_nodes, out_edges, order
    ws = torch.empty(lib.gib_reorder_ws_bytes(M), dtype=torch.uint8, device=dev)
    status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=dev)
    check(lib.gib_reorder(ctypes.byref(d), _ptr(nodes), _ptr(edges), M, ROUTE_BFS if route == "bfs" else ROUTE_DFS,
                          int(rankings is None), ctypes.c_ulonglong(seed % 2**64), epoch, first, _ptr(rk), _ptr(order),
                          _ptr(out_nodes), _ptr(out_edges), _ptr(ws), _ptr(status),
                          ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "gib_reorder")
    refuse_bad(status.cpu().numpy(), 0, M, _REORDER_REASONS)
    return out_nodes, out_edges, order


_MATCH_REASONS = _REORDER_REASONS + ((PP_MATCH_BUDGET, "the scaffold search ran out of its budget of search-tree nodes "
                                      "(raise `budget`)"),)


def scaffold_first(nodes, edges, scaffolds, attachment=None, scaffold_ids=None, rankings=None, seed=0, epoch=0, *,
                   layout, first=0, budget=1 << 20, chunk_molecules=65536, device="cuda"):
    """Scaffold-first decoding order (`gib_scaffold_first`, csrc/preprocess.cu): find each molecule's scaffold and
    renumber its atoms so that its first k_s atoms, with every bond among them, are byte for byte scaffold s -- the
    order `RouteScorer.score(..., scaffold_ids=)` and the scaffold decorators need.

    nodes [M, N, F] / edges [M, N, N, Ef]: int8 stacks (numpy or torch, any atom order), validated and refused as
    `reorder` refuses them.  scaffolds: a `generation.ScaffoldTable` (its attachment points are used), or a pair of
    int8 stacks (nodes [S, N', F], edges [S, N', N', Ef]) checked once by `ScaffoldTable` with `attachment`.
    An embedding of scaffold s maps its atom i to a molecule atom phi(i) whose node row equals scaffold row i (all F
    bytes), with edge cell (phi(i), phi(j)) equal to scaffold cell (i, j) for every pair (an induced match of the same
    bond types) and, with attachment points, no bond from a protected scaffold atom to an atom outside the image.  The
    chosen one is the lexicographically smallest (phi(0), ..., phi(k-1)).
    scaffold_ids: int [M] (-1: do not match), or None: the first scaffold in table order that embeds (order the table
    by priority, larger scaffolds first for example).
    The order: phi(0..k-1), then breadth-first layers out of the image, each layer highest-ranked atom first, rankings
    as `reorder` takes or draws them (seed, epoch, first + m): a fresh epoch redraws the decoration order.
    Returns device tensors (nodes, edges, order int32 [M, N] (old index per new position, -1 past the atom count),
    ids int32 [M] (the scaffold used)).  A molecule without an embedding keeps its bytes, the identity order and id -1,
    so `score(nodes, edges, scaffold_ids=ids)` scores it whole.
    budget: search-tree nodes per (molecule, scaffold); a search that needs more raises ValueError naming the molecule,
    as do the refusals of `reorder`.  Molecules go to the device chunk_molecules at a time."""
    from .generation import ScaffoldTable
    M, N, F, Ef = _check_stacks(nodes, edges)
    d = _pp_dims(N, F, Ef, tuple(layout))
    if isinstance(scaffolds, ScaffoldTable):
        if attachment is not None:
            raise ValueError("attachment is given with the ScaffoldTable, not here")
        table = scaffolds
        if table.N != N or tuple(table.nodes.shape[1:]) != (N, F) or table.edges.shape[3] != Ef:
            raise ValueError(f"the scaffold table holds [S, {table.N}, {table.nodes.shape[2]}] graphs, the molecules "
                             f"[M, {N}, {F}] with Ef = {Ef}")
    else:
        table = ScaffoldTable(scaffolds[0], scaffolds[1], attachment, N, F, Ef, tuple(layout), device)
    if int(budget) < 1:
        raise ValueError(f"budget must be >= 1, got {budget}")
    dev = _cuda(torch.device(device))
    if scaffold_ids is not None:
        ids_in = torch.as_tensor(np.asarray(torch.as_tensor(scaffold_ids).cpu(), np.int64))
        if tuple(ids_in.shape) != (M,):
            raise ValueError(f"scaffold_ids must be [M] = [{M}], got {tuple(ids_in.shape)}")
        bad = (ids_in < -1) | (ids_in >= table.S)
        if bool(bad.any()):
            m = int(torch.nonzero(bad)[0])
            raise ValueError(f"molecule {m}: scaffold id {int(ids_in[m])} outside [-1, {table.S})")
        ids_in = ids_in.to(torch.int32).to(dev)
    if rankings is not None:
        rk_in = torch.as_tensor(rankings)
        if tuple(rk_in.shape) != (M, N):
            raise ValueError(f"rankings must be [M, N] = {(M, N)}, got {tuple(rk_in.shape)}")
    out_nodes = torch.empty((M, N, F), dtype=torch.int8, device=dev)
    out_edges = torch.empty((M, N, N, Ef), dtype=torch.int8, device=dev)
    order = torch.empty((M, N), dtype=torch.int32, device=dev)
    ids = torch.empty(M, dtype=torch.int32, device=dev)
    if M == 0:
        return out_nodes, out_edges, order, ids
    chunk = min(max(int(chunk_molecules), 1), M)
    ws = torch.empty(lib.gib_scaffold_first_ws_bytes(ctypes.byref(d), chunk, table.S), dtype=torch.uint8, device=dev)
    status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=dev)
    rk = torch.empty((chunk, N), dtype=torch.int32, device=dev)
    sc = table.struct()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for pos in range(0, M, chunk):
        stop = min(pos + chunk, M)
        n = stop - pos
        x, e = _on_device(nodes[pos:stop], dev), _on_device(edges[pos:stop], dev)
        if rankings is not None:
            rk[:n].copy_(_on_device(rk_in[pos:stop], dev))
        check(lib.gib_scaffold_first(ctypes.byref(d), _ptr(x), _ptr(e), n, ctypes.byref(sc),
                                     _ptr(ids_in[pos:stop]) if scaffold_ids is not None else None,
                                     int(rankings is None), ctypes.c_ulonglong(seed % 2**64), epoch, first + pos,
                                     _ptr(rk), int(budget), _ptr(order[pos:stop]), _ptr(ids[pos:stop]),
                                     _ptr(out_nodes[pos:stop]), _ptr(out_edges[pos:stop]), _ptr(ws), _ptr(status),
                                     stream), "gib_scaffold_first")
        refuse_bad(status.cpu().numpy(), pos, stop, _MATCH_REASONS)
    return out_nodes, out_edges, order, ids


Murcko = namedtuple("Murcko", "nodes edges ids counts attachment keep")
Murcko.__doc__ = """The Murcko scaffolds of a set (`murcko_scaffolds`), all device tensors:
nodes int8 [S, N, F] / edges int8 [S, N, N, Ef]: the distinct scaffolds, in order of first occurrence
ids int32 [M]: each molecule's entry, -1 without a ring;  counts int64 [S]: molecules per entry
attachment bool [S, N]: entry atoms where some molecule of the entry carries a substituent
keep bool [M, N]: the kept atoms, in each molecule's own numbering"""

_MURCKO_REASONS = _REORDER_REASONS[:3] + ((PP_DISCONNECTED, "a disconnected graph"),
                                         (PP_MATCH_BUDGET, "the scaffold isomorphism search ran out of its budget of "
                                          "search-tree nodes (raise `budget`)"))


def murcko_scaffolds(nodes, edges, *, layout, known=None, budget=1 << 20, chunk_molecules=65536, device="cuda"):
    """Each molecule's Bemis-Murcko scaffold and the distinct scaffolds of the set (`gib_murcko`, csrc/preprocess.cu).

    nodes [M, N, F] / edges [M, N, N, Ef]: int8 stacks (numpy or torch, any atom order), validated and refused as
    `reorder` refuses them (ValueError naming the first bad molecule).  `layout` as `reorder` takes it.
    The rule is RDKit's `MurckoScaffold.GetScaffoldForMol`: an atom is kept when it lies on a ring or on the shortest
    path between two rings, or when it has a double bond (edge feature 1) to such an atom.  The scaffold keeps every
    bond among its atoms and copies their node rows byte for byte, implicit-H and chirality bytes included -- unlike
    RDKit's standalone scaffold molecule, whose hydrogens are recomputed -- so that `scaffold_first` finds each
    molecule's own scaffold in it.  Its atoms are in breadth-first order from the lowest kept index, each layer in
    increasing index.  A molecule without a ring has no scaffold (id -1).
    Two molecules share an entry when their scaffolds are isomorphic (checked by an exact search, never by a hash
    alone); entries come in order of first occurrence, each as its first molecule's scaffold.  An entry atom is an
    attachment point when, in some molecule of the entry, the atom it maps to (the smallest isomorphism) carries a
    bond out of the scaffold.
    known: an earlier result whose entries come first and keep their ids; new scaffolds follow, counts and attachment
    accumulate (ids >= known.nodes.shape[0] are novel scaffolds).  Calls chained over the pieces of a set give what
    one call over the whole set gives.  budget: search-tree nodes per isomorphism test (ValueError naming the molecule
    beyond it).  Molecules go to the device chunk_molecules at a time.  Returns a `Murcko`."""
    M, N, F, Ef = _check_stacks(nodes, edges)
    d = _pp_dims(N, F, Ef, tuple(layout))
    if int(budget) < 1:
        raise ValueError(f"budget must be >= 1, got {budget}")
    dev = _cuda(torch.device(device))
    if known is None:
        S = 0
        t_nodes = torch.zeros((0, N, F), dtype=torch.int8, device=dev)
        t_edges = torch.zeros((0, N, N, Ef), dtype=torch.int8, device=dev)
        counts = torch.zeros(0, dtype=torch.int64, device=dev)
        attach = torch.zeros((0, N), dtype=torch.uint8, device=dev)
    else:
        S = known.nodes.shape[0]
        if tuple(known.nodes.shape) != (S, N, F) or tuple(known.edges.shape) != (S, N, N, Ef) \
                or tuple(known.counts.shape) != (S,) or tuple(known.attachment.shape) != (S, N):
            raise ValueError(f"known holds [S, {N}, {F}] / Ef = {Ef} scaffolds with counts [S] and attachment "
                             f"[S, {N}], got {tuple(known.nodes.shape)} / {tuple(known.edges.shape)}")
        t_nodes, t_edges = _on_device(known.nodes, dev).to(torch.int8), _on_device(known.edges, dev).to(torch.int8)
        counts = _on_device(known.counts, dev).to(torch.int64)
        attach = _on_device(known.attachment, dev).to(torch.uint8)
    ids = torch.empty(M, dtype=torch.int32, device=dev)
    keep = torch.zeros((M, N), dtype=torch.uint8, device=dev)
    status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    chunk = min(max(int(chunk_molecules), 1), max(M, 1))
    for pos in range(0, M, chunk):
        stop = min(pos + chunk, M)
        n = stop - pos
        x, e = _on_device(nodes[pos:stop], dev), _on_device(edges[pos:stop], dev)
        # room for n new entries after the S known ones; the call appends status[5] of them
        t_nodes = torch.cat([t_nodes, t_nodes.new_zeros((n, N, F))])
        t_edges = torch.cat([t_edges, t_edges.new_zeros((n, N, N, Ef))])
        counts = torch.cat([counts, counts.new_zeros(n)])
        attach = torch.cat([attach, attach.new_zeros((n, N))])
        ws_bytes = lib.gib_murcko_ws_bytes(ctypes.byref(d), n, S)
        if ws_bytes == 0:
            raise ValueError(lib.gib_last_error().decode())
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        check(lib.gib_murcko(ctypes.byref(d), _ptr(x), _ptr(e), n, S, _ptr(t_nodes), _ptr(t_edges), _ptr(counts),
                             _ptr(attach), int(budget), _ptr(keep[pos:stop]), _ptr(ids[pos:stop]), _ptr(ws),
                             _ptr(status), stream), "gib_murcko")
        st = status.cpu().numpy()
        refuse_bad(st, pos, stop, _MURCKO_REASONS)
        S += int(st[5])
        t_nodes, t_edges, counts, attach = t_nodes[:S], t_edges[:S], counts[:S], attach[:S]
    return Murcko(t_nodes, t_edges, ids, counts, attach.bool(), keep.bool())


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
