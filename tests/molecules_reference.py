"""What the molecule tests compare against:

  * the reference's own `graph_to_graph` (GraphGenerator.py:659-804) and `get_molecular_properties`
    (Analyzer.py:311-599), loaded unmodified from oracle/_ref with stub modules for what is not installed here:
    a recording `rdkit` (every call and its arguments, with their Python types, go to one log), `matplotlib`,
    `torch.utils.tensorboard`, `util` and `parameters.constants`;
  * a numpy restatement of the table of `gib_molecule_table` and of the statistics of `gib_graph_statistics`
    (include/gib200.h), written from the reference's rules, not from the kernels.
"""
import importlib.util
import os
import sys
import types
from collections import namedtuple

import numpy as np

from tests import refimpl

HDR, MOL, ATOM = 8, 6, 3          # GIB_MOL_HDR_WORDS, GIB_MOL_WORDS, GIB_MOL_ATOM_WORDS
DECODES, KEY_ERROR, DUPLICATE = 1, 2, 4
A, CH, H, CHI = 5, 3, 4, 3
LAYOUTS = {"L0": (0, 0), "L1": (H, 0), "L2": (0, CHI), "L3": (H, CHI)}     # gdb13, implicit H, chirality, both
BONDS = ("SINGLE", "DOUBLE", "TRIPLE", "AROMATIC")


def constants(layout="L0", N=13, Ef=3, device="cpu"):
    """reference-style constants of one of the four action layouts (parameters/constants.py:23-95); bond types are
    named by strings, which the rdkit stub records"""
    h, c = LAYOUTS[layout]
    F = A + CH + h + c
    fields = dict(dim_nodes=[N, F], dim_edges=[N, N, Ef], max_n_nodes=N, n_node_features=F, n_edge_features=Ef,
                  n_atom_types=A, n_formal_charge=CH, n_imp_H=h, n_chirality=c, use_explicit_H=False,
                  ignore_H=not h, use_chirality=bool(c), atom_types=["C", "N", "O", "S", "Cl"],
                  formal_charge=[-1, 0, 1], imp_H=[0, 1, 2, 3], chirality=["None", "R", "S"],
                  int_to_bondtype={t: BONDS[t % 4] + ("" if t < 4 else str(t)) for t in range(Ef)}, device=device,
                  tensorboard_dir="/nonexistent")
    return namedtuple("constants", sorted(fields))(**fields)


# ---- the recording rdkit stub -------------------------------------------------------------------------------------
LOG = []


def _rec(*call):
    LOG.append(tuple(call) + (tuple(type(a).__name__ for a in call[1:]),))


class Atom:
    def __init__(self, symbol):
        _rec("Atom", symbol)
        self.symbol, self.charge = symbol, 0

    def SetFormalCharge(self, charge):
        _rec("SetFormalCharge", charge)
        self.charge = charge

    def SetUnsignedProp(self, key, value):
        _rec("SetUnsignedProp", key, value)

    def SetProp(self, key, value):
        _rec("SetProp", key, value)


class RWMol:
    def __init__(self):
        _rec("RWMol")
        self.atoms, self.bonds = [], []

    def AddAtom(self, atom):
        _rec("AddAtom", atom.symbol)
        self.atoms.append((atom.symbol, atom.charge))
        return len(self.atoms) - 1

    def AddBond(self, i, j, bond_type):
        _rec("AddBond", i, j, bond_type)
        if i == j or any({i, j} == {a, b} for a, b, _ in self.bonds):     # RDKit: "bond already exists"
            raise RuntimeError(f"Pre-condition Violation: bond already exists ({i}, {j})")
        self.bonds.append((i, j, bond_type))
        return len(self.bonds)

    def GetMol(self):
        _rec("GetMol")
        return self

    def GetNumAtoms(self):
        return len(self.atoms)

    def key(self):
        return tuple(self.atoms), tuple(self.bonds)


def SanitizeMol(mol):
    _rec("SanitizeMol", None if mol is None else len(mol.atoms))
    if not isinstance(mol, RWMol):
        raise TypeError("SanitizeMol: not a molecule")
    if any(charge != 0 for _, charge in mol.atoms):          # a deterministic stand-in for RDKit's valence checks
        raise ValueError("Sanitization error: charged atom")


def MolToSmiles(mol, kekuleSmiles=False):
    _rec("MolToSmiles", None if mol is None else len(mol.atoms))
    if mol is None:
        raise TypeError("MolToSmiles: None")
    return repr(mol.key())


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    return m


def load_reference(C, setitem=None):
    """installs the stubs (through `setitem(sys.modules, name, module)`, e.g. pytest's monkeypatch.setitem) and loads
    the reference's MolecularGraph, GraphGenerator, GraphGeneratorRL and Analyzer from oracle/_ref under their module
    names; returns them as a namespace, or None when oracle/_ref does not hold them"""
    setitem = setitem or (lambda d, k, v: d.__setitem__(k, v))
    paths = {k: os.path.join(refimpl.REF_ROOT, k + ".py") for k in
             ("MolecularGraph", "GraphGenerator", "GraphGeneratorRL", "Analyzer")}
    if not all(os.path.exists(p) for p in paths.values()):
        return None
    rdmolfiles = _module("rdkit.Chem.rdmolfiles", MolToSmiles=MolToSmiles)
    chem = _module("rdkit.Chem", Atom=Atom, RWMol=RWMol, Mol=RWMol, SanitizeMol=SanitizeMol, MolToSmiles=MolToSmiles,
                   rdmolfiles=rdmolfiles)
    rdkit = _module("rdkit", Chem=chem)
    pc = _module("parameters.constants", constants=C)
    pkg = _module("parameters", constants=pc)
    pkg.__path__ = []
    util = _module("util", get_feature_vector_indices=lambda: feature_vector_ends(sys.modules["parameters.constants"]
                                                                                  .constants))
    mpl = _module("matplotlib", use=lambda *a, **k: None)
    mpl.pyplot = _module("matplotlib.pyplot")
    tb = _module("torch.utils.tensorboard", SummaryWriter=lambda *a, **k: None)
    for name, mod in (("rdkit", rdkit), ("rdkit.Chem", chem), ("rdkit.Chem.rdmolfiles", rdmolfiles),
                      ("parameters", pkg), ("parameters.constants", pc), ("util", util), ("matplotlib", mpl),
                      ("matplotlib.pyplot", mpl.pyplot), ("torch.utils.tensorboard", tb)):
        setitem(sys.modules, name, mod)
    ns = types.SimpleNamespace(constants_module=pc)
    for name, path in paths.items():
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        setitem(sys.modules, name, mod)
        spec.loader.exec_module(mod)
        setattr(ns, name, mod)
    return ns


def set_constants(ref, C):
    """the reference modules bound `constants` at import: point them (and the stubs) at C"""
    ref.constants_module.constants = C
    for m in (ref.GraphGenerator, ref.GraphGeneratorRL, ref.Analyzer):
        m.constants = C


def feature_vector_ends(C):
    ends = [C.n_atom_types, C.n_formal_charge]
    if not C.use_explicit_H and not C.ignore_H:
        ends.append(C.n_imp_H)
    if C.use_chirality:
        ends.append(C.n_chirality)
    return list(np.cumsum(ends))


def reference_graphs(ref, nodes, edges, n_nodes, rl=False):
    """[graph_to_graph(idx) for idx in range(B)] of the unmodified reference on these tensors, and the stub's call
    log; an exception the reference raises is returned in place of the list"""
    gen = types.SimpleNamespace(generated_nodes=nodes, generated_edges=edges, generated_n_nodes=n_nodes)
    cls = ref.GraphGeneratorRL.GraphGeneratorRL if rl else ref.GraphGenerator.GraphGenerator
    LOG.clear()
    try:
        out = [cls.graph_to_graph(gen, idx) for idx in range(nodes.shape[0])]
    except Exception as ex:                # noqa: BLE001 -- the outcome is compared, exceptions included
        out = ex
    return out, list(LOG)


def reference_properties(ref, graphs, epoch_key, termination):
    LOG.clear()
    try:
        out = ref.Analyzer.Analyzer.get_molecular_properties(None, graphs, epoch_key, termination)
    except Exception as ex:                # noqa: BLE001
        out = ex
    return out, list(LOG)


def describe(graphs):
    """what a GenerationGraph list holds: n_nodes, the molecule's atoms and bonds (None for mol = None), and which
    tensors node_features / edge_features are"""
    if isinstance(graphs, Exception):
        return type(graphs).__name__
    return [(g.n_nodes, None if g.molecule is None else g.molecule.key(), g.node_features.data_ptr(),
             tuple(g.node_features.shape), g.edge_features.data_ptr(), tuple(g.edge_features.shape)) for g in graphs]


# ---- numpy restatement of the table and the statistics ------------------------------------------------------------
def _nonzero(x):
    return ~(x == 0)                                     # torch.nonzero: NaN counts


def _index_ok(i, n):
    return -n <= i < n


def atom_decodes(rec, C):
    nnz, i0, i1, i2, last = rec
    imp_h = not C.use_explicit_H and not C.ignore_H
    if nnz < 1 or not _index_ok(i0, len(C.atom_types)):
        return False
    if nnz < 2 or not _index_ok(i1 - C.n_atom_types, len(C.formal_charge)):
        return False
    if imp_h and (nnz < 3 or not _index_ok(i2 - C.n_atom_types - C.n_formal_charge, len(C.imp_H))):
        return False
    if C.use_chirality and not _index_ok(last - C.n_atom_types - C.n_formal_charge - imp_h * C.n_imp_H,
                                         len(C.chirality)):
        return False
    return True


def table(nodes, edges, n_nodes, C):
    """(header int32 [HDR + MOL * B], body int32 [used words]) as gib_molecule_table + gib_graph_statistics leave
    them (header words 2..4 from `statistics`)"""
    nodes, edges, n_nodes = np.asarray(nodes, np.float32), np.asarray(edges, np.float32), np.asarray(n_nodes)
    B, N, F = nodes.shape
    Ef = edges.shape[-1]
    mols, atom_recs, bond_recs = [], [], []
    upper = np.triu(np.ones((N, N), np.float32), 1)[:, :, None]
    flags_or = 0
    for b in range(B):
        n = int(n_nodes[b])
        na = min(max(n, 0), N)
        decodes = n <= N
        for a in range(na):
            idx = np.flatnonzero(_nonzero(nodes[b, a]))
            rec = [len(idx)] + [int(idx[k]) if k < len(idx) else -1 for k in range(3)] + \
                  [int(idx[-1]) if len(idx) else -1]
            decodes &= atom_decodes(rec, C)
            atom_recs.append(rec + [0])
        with np.errstate(invalid="ignore"):
            listed = np.argwhere(_nonzero(edges[b] * upper))          # row-major (i, j, t)
        flags = DECODES if decodes else 0
        pairs = {}
        for i, j, t in listed:
            if i >= n or j >= n:
                flags |= KEY_ERROR
            key = (min(i, j), max(i, j))
            pairs[key] = pairs.get(key, 0) + 1
            bond_recs.append((int(i), int(j), int(t), 0))
        if any(v > 1 or i == j for (i, j), v in pairs.items()):
            flags |= DUPLICATE
        flags_or |= flags & (KEY_ERROR | DUPLICATE)
        mols.append([n, na, len(listed), 0, 0, flags])
    mols = np.array(mols, np.int64).reshape(B, MOL)
    mols[:, 3] = np.concatenate([[0], np.cumsum(mols[:, 1])[:-1]])
    mols[:, 4] = np.concatenate([[0], np.cumsum(mols[:, 2])[:-1]])
    header = np.zeros(HDR + MOL * B, np.int32)
    header[0], header[1], header[2], header[5] = len(atom_recs), len(bond_recs), -1, flags_or
    header[HDR:] = mols.reshape(-1)
    atoms = np.array(atom_recs, np.int16).reshape(-1, 2 * ATOM)
    bonds = np.array(bond_recs, np.uint8).reshape(-1, 4)
    body = np.concatenate([atoms.reshape(-1).view(np.int32), bonds.reshape(-1).view(np.int32)])
    n_eff = np.where(mols[:, 5] & DECODES, np.maximum(mols[:, 0], 0), 0)
    stats, err = statistics(nodes, edges, n_eff)
    if err is not None:
        header[2:5] = err
    return header, body, stats


def statistics(nodes, edges, n_eff):
    """gib_graph_statistics' output vector (float32) and the first (molecule, error kind, atom) whose
    _get_n_edges_distribution raises, from the effective atom counts (GenerationGraph.n_nodes)"""
    nodes, edges = np.asarray(nodes, np.float32), np.asarray(edges, np.float32)
    B, N, F = nodes.shape
    Ef = edges.shape[-1]
    n_nodes_hist = np.zeros(N + 1, np.float32)
    nodes_hist = np.zeros(F, np.float32)
    n_edges_hist = np.zeros(10, np.float32)
    edge_hist = np.zeros(Ef, np.float32)
    err = None
    with np.errstate(invalid="ignore", over="ignore"):
        for b in range(B):
            n_nodes_hist[n_eff[b]] += 1
            nodes_hist += nodes[b].sum(0, dtype=np.float32)
            rows = edges[b].sum(1, dtype=np.float32)                 # [N, Ef]
            for i in range(n_eff[b]):
                ne, kind = 0, 0
                for t in range(Ef):
                    s = rows[i, t]
                    if np.isnan(s):
                        kind = 1
                    elif np.isinf(s):
                        kind = 2
                    else:
                        ne += int(s)
                        continue
                    break
                if not kind:
                    idx = min(ne, 10) - 1
                    if idx < -10:
                        kind = 3
                    else:
                        n_edges_hist[idx] += 1
                if kind and err is None:
                    err = (b, kind, i)
            edge_hist += (edges[b].sum((0, 1), dtype=np.float32) * np.float32(0.5)).astype(np.float32)
        sum_n = np.float32(sum(np.float32(k) * c for k, c in enumerate(n_nodes_hist)))
        sum_e = np.float32(sum(np.float32(k + 1) * c for k, c in enumerate(n_edges_hist)))
    out = np.concatenate([n_nodes_hist, nodes_hist, n_edges_hist, edge_hist, [sum_n, sum_e]]).astype(np.float32)
    return out, err
