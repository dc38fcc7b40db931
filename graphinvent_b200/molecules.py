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
"""
import ctypes

import numpy as np
import torch

from ._lib import (MOL_ATOM_WORDS, MOL_DECODES, MOL_ERR_INDEX, MOL_ERR_OVERFLOW, MOL_ERR_VALUE, MOL_HDR_WORDS,
                   MOL_WORDS, MolLayout, check, lib)

N_EDGES_TO_BIN = 10      # Analyzer.py:557-560


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
