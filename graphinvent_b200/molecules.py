"""
Generated batches as the reference's molecules and Analyzer statistics, from one device pass.

The reference turns a generated batch into `GenerationGraph`s one atom at a time (`graph_to_graph`,
GraphGenerator.py:659-804; GraphGeneratorRL.py:725): per atom a `torch.nonzero` and 3-5 tensor reads, per bond three
`.item()` calls.  `Analyzer.get_molecular_properties` (Analyzer.py:311-599) then reads the same tensors again per atom
and bond type.  On CUDA tensors each read is a blocking device->host copy, about 10^5 per batch of 1000 molecules.

`MoleculeBatch` runs `gib_molecule_table` and `gib_graph_statistics` (csrc/molecules.cu) once, copies the table back in
two copies (its header, then the used records) and keeps the statistics on the device:

  * `generation_graphs()` replays, from the host table, the RDKit calls `graph_to_graph` makes, with the same arguments
    in the same order and the same exceptions (`mol = None` on IndexError; KeyError and RDKit's errors propagate);
  * `properties(epoch_key, termination, graphs)` returns `get_molecular_properties`' dict, every value of the same type,
    dtype, device and bits: the histograms are views of the device statistics and the 0-d quotients are formed with the
    reference's own torch ops.  Only the RDKit parts (uniqueness, validity) run on the host, by the reference's rules.

`rdkit` and `MolecularGraph` are the modules of the caller's environment (the reference's Workflow imports them by
these names); this package does not depend on them.

`MoleculeSet` is a persistent device set of distinct molecules (`gib_molset_identify`, csrc/preprocess.cu) for
uniqueness across a whole sample and novelty against a training set; `uniqueness` is the reference's per-batch
uniqueness tensor from one call on a transient set.
"""
import ctypes
from collections import namedtuple

import numpy as np
import torch

from ._lib import (MOL_ATOM_WORDS, MOL_DECODES, MOL_ERR_INDEX, MOL_ERR_OVERFLOW, MOL_ERR_VALUE, MOL_HDR_WORDS,
                   MOL_WORDS, PP_BAD_EDGES, PP_BAD_NODES, PP_CAPACITY, PP_DISCONNECTED, PP_MATCH_BUDGET, PP_STATUS_INTS,
                   MolLayout, MolSet, check, lib)

N_EDGES_TO_BIN = 10      # Analyzer.py:557-560

_SET_REASONS = ((PP_BAD_NODES, "a node row that is not one-hot per segment with 0/1 entries, or a zero row between "
                 "atoms"),
                (PP_BAD_EDGES, "edges that are not symmetric 0/1 single-type bonds between its atoms"),
                (PP_DISCONNECTED, "a disconnected graph"),
                (PP_MATCH_BUDGET, "the isomorphism search ran out of its budget of search-tree nodes (raise `budget`)"))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _imp_h_segment(C):
    return not C.use_explicit_H and not C.ignore_H


def mol_layout(C):
    """the gib_mol_layout of the reference constants `C`"""
    return MolLayout(n_atom_types=C.n_atom_types, n_formal_charge=C.n_formal_charge, n_imp_H=C.n_imp_H,
                     use_imp_H=int(_imp_h_segment(C)), use_chirality=int(bool(C.use_chirality)),
                     len_atom_types=len(C.atom_types), len_formal_charge=len(C.formal_charge), len_imp_H=len(C.imp_H),
                     len_chirality=len(C.chirality))


def feature_vector_indices(C):
    """the ends of the node-feature segments (util.get_feature_vector_indices): atom type, formal charge, then the
    implicit-H and chirality segments when the layout has them"""
    ends = [C.n_atom_types, C.n_formal_charge]
    if _imp_h_segment(C):
        ends.append(C.n_imp_H)
    if C.use_chirality:
        ends.append(C.n_chirality)
    return np.cumsum(ends).tolist()


def split_table(header, body):
    """(per-molecule rows [B, MOL_WORDS], atom records int16 [atoms, 6], bonds uint8 [bonds, 4]) of a host table"""
    B = (len(header) - MOL_HDR_WORDS) // MOL_WORDS
    n_atoms, n_bonds = int(header[0]), int(header[1])
    mols = header[MOL_HDR_WORDS:MOL_HDR_WORDS + B * MOL_WORDS].reshape(B, MOL_WORDS)
    atoms = body[:MOL_ATOM_WORDS * n_atoms].view(np.int16).reshape(n_atoms, 2 * MOL_ATOM_WORDS)
    bonds = body[MOL_ATOM_WORDS * n_atoms:MOL_ATOM_WORDS * n_atoms + n_bonds].view(np.uint8).reshape(n_bonds, 4)
    return mols, atoms, bonds


def _features_to_atom(rec, C):
    """GraphGenerator.py:672-730 on one atom record (nnz, first, second, third, last): `nonzero_idc[k]` raises
    IndexError where the row has too few non-zeros, list indices wrap as Python's do"""
    import rdkit

    nnz, first = rec[0], rec[1:4]

    def nonzero_idc(k):
        if k >= nnz or nnz == 0:
            raise IndexError(f"index {k} is out of bounds for dimension 0 with size {nnz}")
        return rec[4] if k == -1 else first[k]

    new_atom = rdkit.Chem.Atom(C.atom_types[nonzero_idc(0)])
    new_atom.SetFormalCharge(C.formal_charge[nonzero_idc(1) - C.n_atom_types])
    imp_h = _imp_h_segment(C)
    if imp_h:
        total_num_h = C.imp_H[nonzero_idc(2) - C.n_atom_types - C.n_formal_charge]
        new_atom.SetUnsignedProp("_TotalNumHs", total_num_h)
    if C.use_chirality:
        cip_code = C.chirality[nonzero_idc(-1) - C.n_atom_types - C.n_formal_charge - imp_h * C.n_imp_H]
        new_atom.SetProp("_CIPCode", cip_code)
    return new_atom


def _graph_to_mol(n_nodes, atoms, bonds, N, C):
    """GraphGenerator.py:732-788 on one molecule's records"""
    import rdkit

    molecule = rdkit.Chem.RWMol()
    node_to_idx = {}
    for node_idx in range(n_nodes):
        if node_idx >= N:
            raise IndexError(f"index {node_idx} is out of bounds for dimension 0 with size {N}")
        node_to_idx[node_idx] = molecule.AddAtom(_features_to_atom(atoms[node_idx], C))
    for node_idx1, node_idx2, bond_idx, _ in bonds:
        molecule.AddBond(node_to_idx[node_idx1], node_to_idx[node_idx2], C.int_to_bondtype[bond_idx])
    try:
        molecule.GetMol()
    except AttributeError:
        pass
    if C.ignore_H and molecule:
        try:
            rdkit.Chem.SanitizeMol(molecule)
        except ValueError:
            pass
    return molecule


def graphs_from_table(header, body, nodes, edges, constants):
    """the `GenerationGraph` list `[graph_to_graph(idx) for idx in range(B)]` of the reference, from a host table
    (header / body: int32 arrays laid out as include/gib200.h describes) and the batch's node / edge tensors"""
    from MolecularGraph import GenerationGraph

    mols, atoms, bonds = split_table(header, body)
    N = nodes.shape[1]
    graphs = []
    for idx, (n_nodes, n_atoms, n_bonds, atom_off, bond_off, _) in enumerate(mols.tolist()):
        try:
            mol = _graph_to_mol(n_nodes, atoms[atom_off:atom_off + n_atoms].tolist(),
                                bonds[bond_off:bond_off + n_bonds].tolist(), N, constants)
        except (IndexError, AttributeError):
            mol = None
        graphs.append(GenerationGraph(constants=constants, molecule=mol, node_features=nodes[idx],
                                      edge_features=edges[idx]))
    return graphs


class MoleculeBatch:
    """One generated batch: nodes [B,N,F] f32, edges [B,N,N,Ef] f32, n_nodes [B] int8 on one CUDA device (what
    `sample()` of the generators returns), and the reference constants `constants`.  The constructor launches both
    kernels and brings the table to the host in two blocking copies; nothing else is read back."""

    def __init__(self, nodes, edges, n_nodes, constants):
        if not (nodes.is_cuda and edges.is_cuda and n_nodes.is_cuda):
            raise ValueError("MoleculeBatch: nodes, edges and n_nodes must be CUDA tensors")
        if nodes.dtype != torch.float32 or edges.dtype != torch.float32 or n_nodes.dtype != torch.int8:
            raise TypeError("MoleculeBatch: nodes / edges must be float32 and n_nodes int8 (the generators' dtypes)")
        B, N, F = nodes.shape
        Ef = edges.shape[-1]
        if tuple(edges.shape) != (B, N, N, Ef) or tuple(n_nodes.shape) != (B,):
            raise ValueError(f"MoleculeBatch: shapes nodes {tuple(nodes.shape)}, edges {tuple(edges.shape)}, "
                             f"n_nodes {tuple(n_nodes.shape)} do not describe one batch")
        if constants.dim_nodes[0] != N or constants.n_node_features != F or constants.n_edge_features != Ef:
            raise ValueError("MoleculeBatch: the tensors' dims differ from the constants' dim_nodes / n_node_features "
                             "/ n_edge_features")
        self.constants = constants
        self.nodes, self.edges, self.n_nodes = nodes, edges, n_nodes
        self.B, self.N, self.F, self.Ef = B, N, F, Ef
        dev = nodes.device
        table_bytes = lib.gib_molecule_table_bytes(B, N, F, Ef)
        stat_bytes = lib.gib_graph_statistics_bytes(N, F, Ef)
        ws_bytes = lib.gib_graph_statistics_ws_bytes(B, N, F, Ef)
        if not (table_bytes and stat_bytes and ws_bytes):
            check(-1, "MoleculeBatch")
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            st = ctypes.c_void_p(stream.cuda_stream)
            c_nodes, c_edges, c_n = nodes.contiguous(), edges.contiguous(), n_nodes.contiguous()
            table = torch.empty(table_bytes // 4, dtype=torch.int32, device=dev)
            self.stats = torch.empty(stat_bytes // 4, dtype=torch.float32, device=dev)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            layout = mol_layout(constants)
            check(lib.gib_molecule_table(B, N, F, Ef, ctypes.byref(layout), _ptr(c_nodes), _ptr(c_edges), _ptr(c_n),
                                         _ptr(table), st), "gib_molecule_table")
            check(lib.gib_graph_statistics(B, N, F, Ef, _ptr(c_nodes), _ptr(c_edges), _ptr(table), _ptr(self.stats),
                                           _ptr(ws), st), "gib_graph_statistics")
            n_hdr = MOL_HDR_WORDS + MOL_WORDS * B
            header = torch.empty(n_hdr, dtype=torch.int32, pin_memory=True)
            header.copy_(table[:n_hdr], non_blocking=True)
            stream.synchronize()
            self.header = header.numpy()
            n_body = MOL_ATOM_WORDS * int(self.header[0]) + int(self.header[1])
            body = torch.empty(n_body, dtype=torch.int32, pin_memory=True)
            if n_body:
                body.copy_(table[n_hdr:n_hdr + n_body], non_blocking=True)
                stream.synchronize()
            self.body = body.numpy()

    @property
    def decodes(self):
        """per molecule: does graph_to_graph build a molecule (True) or return mol = None (False)"""
        return (split_table(self.header, self.body)[0][:, 5] & MOL_DECODES) != 0

    def generation_graphs(self):
        """the reference's `[graph_to_graph(idx) for idx in range(B)]`, with node_features / edge_features the
        batch's device views"""
        return graphs_from_table(self.header, self.body, self.nodes, self.edges, self.constants)

    def properties(self, epoch_key, termination, graphs):
        """`Analyzer.get_molecular_properties(graphs, epoch_key, termination)` for `graphs` = generation_graphs() of
        this batch.  `termination` (the properly-terminated flags) is read to the host once; it is not used for the
        "Training set" key, as in the reference."""
        C, N, F, Ef = self.constants, self.N, self.F, self.Ef
        if len(graphs) != self.B:
            raise ValueError(f"properties: {len(graphs)} graphs for a batch of {self.B}")
        err_mol, err_kind, err_atom = (int(v) for v in self.header[2:5])
        if err_mol >= 0:        # _get_n_edges_distribution raises in the reference (Analyzer.py:352-368)
            where = f"(molecule {err_mol}, atom {err_atom})"
            if err_kind == MOL_ERR_VALUE:
                raise ValueError(f"cannot convert float NaN to integer {where}")
            if err_kind == MOL_ERR_OVERFLOW:
                raise OverflowError(f"cannot convert float infinity to integer {where}")
            assert err_kind == MOL_ERR_INDEX
            raise IndexError(f"n_edges_histogram index out of bounds for dimension 0 with size {N_EDGES_TO_BIN} {where}")
        s = self.stats
        o_nf = N + 1
        o_ne = o_nf + F
        o_ef = o_ne + N_EDGES_TO_BIN
        o_sum = o_ef + Ef
        n_nodes_hist = s[:o_nf]
        avg_n_nodes = s[o_sum] / len(graphs)                                           # Analyzer.py:403-408
        nodes_hist = s[o_nf:o_ne]
        idc = feature_vector_indices(C)
        atom_type_hist = nodes_hist[:idc[0]]
        formal_charge_hist = nodes_hist[idc[0]:idc[1]]
        numh_hist = nodes_hist[idc[1]:idc[2]] if _imp_h_segment(C) else [0] * C.n_imp_H
        if C.use_chirality:
            correction = int(_imp_h_segment(C))
            chirality_hist = nodes_hist[idc[1 + correction]:idc[2 + correction]]
        else:
            chirality_hist = [0] * C.n_chirality
        n_edges_hist = s[o_ne:o_ef]
        avg_n_edges = s[o_sum + 1] / torch.sum(n_edges_hist, dim=0)                   # Analyzer.py:371-378
        edge_feature_hist = s[o_ef:o_sum]
        fraction_unique = _fraction_unique(graphs)
        if epoch_key == "Training set":
            fraction_valid, fraction_valid_pt, fraction_pt = 1.0, 1.0, 1.0
        else:
            fraction_valid, fraction_valid_pt, fraction_pt = _fraction_valid(graphs, termination)
        return {
            (epoch_key, "n_nodes_hist"): n_nodes_hist,
            (epoch_key, "avg_n_nodes"): avg_n_nodes,
            (epoch_key, "atom_type_hist"): atom_type_hist,
            (epoch_key, "formal_charge_hist"): formal_charge_hist,
            (epoch_key, "n_edges_hist"): n_edges_hist,
            (epoch_key, "avg_n_edges"): avg_n_edges,
            (epoch_key, "edge_feature_hist"): edge_feature_hist,
            (epoch_key, "fraction_unique"): fraction_unique,
            (epoch_key, "fraction_valid"): fraction_valid,
            (epoch_key, "fraction_valid_properly_terminated"): fraction_valid_pt,
            (epoch_key, "fraction_properly_terminated"): fraction_pt,
            (epoch_key, "numh_hist"): numh_hist,
            (epoch_key, "chirality_hist"): chirality_hist,
        }


def _fraction_unique(graphs):
    """Analyzer.py:480-499"""
    smiles_set = set(g.get_smiles() for g in graphs)
    smiles_set.discard(None)
    try:
        return len(smiles_set) / len(graphs)
    except ZeroDivisionError:
        return 0


def _fraction_valid(graphs, termination):
    """Analyzer.py:501-544 with `termination` read to the host once; the tensor-valued quotients use the device
    tensor, as the reference's do"""
    import rdkit

    term_host = termination.cpu()
    n_invalid = n_valid_and_properly_terminated = 0
    n_graphs = len(graphs)
    for idx, graph in enumerate(graphs):
        mol = graph.get_molecule()
        try:
            rdkit.Chem.SanitizeMol(mol)
            n_valid_and_properly_terminated += int(term_host[idx])
        except:  # noqa: E722  -- the reference's rule: whatever RDKit raises marks the molecule invalid
            n_invalid += 1
    fraction_valid = (n_graphs - n_invalid) / n_graphs
    if 1 in term_host:
        fraction_valid_pt = n_valid_and_properly_terminated / torch.sum(termination)
    else:
        fraction_valid_pt = 0.0
    fraction_pt = torch.sum(termination) / len(termination)
    return fraction_valid, fraction_valid_pt, fraction_pt


# ---- the molecule set ------------------------------------------------------------------------------------------------
Identity = namedtuple("Identity", "ids new first")
Identity.__doc__ = """What a `MoleculeSet` call says about each molecule of a batch, all device tensors [B]:
ids int32: its entry (-1: not in the set after a `find`, or skipped by `valid`)
new bool: its class was not in the set before the call;  first bool: the first molecule of its class in the call"""


class MoleculeSet:
    """A persistent set of distinct molecules on the device (`gib_molset_identify`, csrc/preprocess.cu): uniqueness
    across batches, novelty against a training set, a run-long memory of what was generated.

    Two molecules are the same when their graphs are isomorphic: every node row (atom type, charge and the implicit-H
    and chirality bytes of the layout) and every edge cell equal under some renumbering of the atoms.  This is graph
    identity, not RDKit's canonical-SMILES identity: two Kekule structures of one aromatic ring, or a group RDKit's
    sanitisation rewrites, are two entries, so the number of distinct graphs bounds the number of distinct SMILES from
    above (DESIGN.md).  All empty graphs are one entry.

    max_n_nodes, n_node_features, n_edge_features: the graphs' N, F, Ef; capacity: entries the set can hold, fixed at
    creation (its buffers take `nbytes`); layout: the node-feature segment widths (n_atom_types, n_formal_charge,
    n_imp_H, n_chirality) as `preprocess.reorder` takes them; budget: search-tree nodes per isomorphism test.
    Each entry holds its first molecule in canonical order (breadth-first from atom 0, each layer in increasing index)
    and the number of molecules `add` gave it.

    `add` and `find` take int8 stacks nodes [B, N, F] / edges [B, N, N, Ef] (numpy or torch, any atom order) or the
    generators' float32 nodes / edges (0 / 1 entries, converted on the device), and valid (bool / uint8 [B], optional:
    molecules with 0 are skipped).  A call's work does not depend on the set's size.  A refused call -- a bad node row,
    a zero row between atoms, bad edges, a disconnected graph, a search beyond `budget`, or more new classes than the
    set has room for -- raises ValueError naming the first such molecule and leaves the set exactly as it was."""

    def __init__(self, max_n_nodes, n_node_features, n_edge_features, capacity, *, layout, budget=1 << 20,
                 device="cuda"):
        from . import preprocess as PP
        N, F, Ef = int(max_n_nodes), int(n_node_features), int(n_edge_features)
        self.d = PP._pp_dims(N, F, Ef, tuple(layout))
        self.N, self.F, self.Ef = N, F, Ef
        self.layout = tuple(layout)
        if int(budget) < 1:
            raise ValueError(f"budget must be >= 1, got {budget}")
        self.budget = int(budget)
        self.capacity = int(capacity)
        self.nbytes = lib.gib_molset_bytes(ctypes.byref(self.d), self.capacity)
        if self.nbytes == 0:
            raise ValueError(lib.gib_last_error().decode())
        slots = lib.gib_molset_slots(self.capacity)
        dev = PP._cuda(torch.device(device))
        C = self.capacity
        self._nodes = torch.empty((C, N, F), dtype=torch.int8, device=dev)
        self._edges = torch.empty((C, N, N, Ef), dtype=torch.int8, device=dev)
        self._hash = torch.empty(C, dtype=torch.int64, device=dev)
        self._n_atoms = torch.empty(C, dtype=torch.int32, device=dev)
        self._n_bonds = torch.empty(C, dtype=torch.int32, device=dev)
        self._counts = torch.empty(C, dtype=torch.int64, device=dev)
        self._next = torch.empty(C, dtype=torch.int32, device=dev)
        self._index_keys = torch.empty(slots, dtype=torch.int64, device=dev)
        self._index_first = torch.empty(slots, dtype=torch.int32, device=dev)
        self._size = torch.empty(1, dtype=torch.int32, device=dev)
        self.device = self._nodes.device
        self._status = torch.empty(PP_STATUS_INTS, dtype=torch.int32, device=self.device)
        self._struct = MolSet(*(_ptr(t) for t in self.buffers()), C, slots)
        check(lib.gib_molset_init(ctypes.byref(self._struct), self._stream()), "gib_molset_init")

    def buffers(self):
        """every device buffer of the set, in `gib_molset` order"""
        return (self._nodes, self._edges, self._hash, self._n_atoms, self._n_bonds, self._counts, self._next,
                self._index_keys, self._index_first, self._size)

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _int8(self, x, shape, what):
        from . import preprocess as PP
        t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
        if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int8, torch.float32) or tuple(t.shape[1:]) != shape:
            raise ValueError(f"{what} must be int8 or float32 [B, {', '.join(map(str, shape))}], got "
                             f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
        t = PP._on_device(t, self.device)
        if t.dtype == torch.int8:
            return t
        out = torch.empty(t.shape, dtype=torch.int8, device=self.device)
        check(lib.gib_molset_from_float(_ptr(t), _ptr(out), t.numel(), self._stream()), "gib_molset_from_float")
        return out

    def _call(self, nodes, edges, valid, insert):
        from . import preprocess as PP
        N, F, Ef = self.N, self.F, self.Ef
        x = self._int8(nodes, (N, F), "nodes")
        e = self._int8(edges, (N, N, Ef), "edges")
        B = x.shape[0]
        if e.shape[0] != B:
            raise ValueError(f"{B} node graphs but {e.shape[0]} edge graphs")
        v = None
        if valid is not None:
            v = torch.as_tensor(valid)
            if tuple(v.shape) != (B,):
                raise ValueError(f"valid must be [B] = [{B}], got {tuple(v.shape)}")
            v = v.to(self.device).ne(0).to(torch.uint8).contiguous()
        ids = torch.full((B,), -1, dtype=torch.int32, device=self.device)
        new = torch.zeros(B, dtype=torch.uint8, device=self.device)
        first = torch.zeros(B, dtype=torch.uint8, device=self.device)
        if B:
            ws = torch.empty(lib.gib_molset_ws_bytes(ctypes.byref(self.d), B), dtype=torch.uint8, device=self.device)
            check(lib.gib_molset_identify(ctypes.byref(self.d), ctypes.byref(self._struct), _ptr(x), _ptr(e),
                                          None if v is None else _ptr(v), B, int(insert), self.budget, _ptr(ids),
                                          _ptr(new), _ptr(first), _ptr(ws), _ptr(self._status), self._stream()),
                  "gib_molset_identify")
            PP.refuse_bad(self._status.cpu().numpy(), 0, B, _SET_REASONS + (
                (PP_CAPACITY, f"the set is full: its {self.capacity} entries cannot take this molecule's new class"),))
        return Identity(ids, new.view(torch.bool), first.view(torch.bool))

    def add(self, nodes, edges, valid=None):
        """inserts the batch: new classes become entries in order of first occurrence, every molecule counts once for
        its entry.  Returns an `Identity`."""
        return self._call(nodes, edges, valid, True)

    def find(self, nodes, edges, valid=None):
        """looks the batch up without changing the set (ids -1 for molecules not in it).  Returns an `Identity`."""
        return self._call(nodes, edges, valid, False)

    def __len__(self):
        return int(self._size.item())

    @property
    def counts(self):
        """int64 [len(self)] device tensor: molecules added per entry"""
        return self._counts[:len(self)]

    def entries(self):
        """(nodes int8 [S, N, F], edges int8 [S, N, N, Ef]): views of the entries, each its first molecule in
        canonical order"""
        S = len(self)
        return self._nodes[:S], self._edges[:S]


def uniqueness(nodes, edges, valid=None, *, layout):
    """float32 [B] on the device: the reference's per-batch `uniqueness_tensor` (util.write_molecules, util.py:549-585)
    with graph identity in place of SMILES equality: 1 for the first occurrence of a molecule or a molecule with
    valid 0 (the reference's invalid molecules), 0 for a later duplicate of a valid one.  nodes / edges as
    `MoleculeSet.add` takes them; one call on a transient set."""
    t = nodes if isinstance(nodes, torch.Tensor) else torch.from_numpy(np.asarray(nodes))
    B, N, F = t.shape
    dev = t.device if t.is_cuda else torch.device("cuda")
    s = MoleculeSet(N, F, edges.shape[-1], max(B, 1), layout=layout, device=dev)
    ident = s.add(nodes, edges, valid)
    keep = ident.first if valid is None else ident.first | ~torch.as_tensor(valid).to(dev).bool()
    return keep.float()
