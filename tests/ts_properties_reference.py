"""What the training-set property tests compare against:

  * a numpy restatement of the integer statistics `gib_preprocess_group_statistics` returns per group
    (include/gib200.h), written from the rules of `Analyzer.get_molecular_properties` (Analyzer.py:337-478), not from
    the kernels;
  * the reference's per-group loop, `DataProcesser.get_ts_properties` (DataProcesser.py:389-417), around the live
    `Analyzer` from oracle/_ref (tests/molecules_reference.py loads it with its stubs);
  * the CSV rule of the reference's `util.write_ts_properties` (util.py:715-742), for the machines where the
    reference's util.py is not installed (checked against it where it is).
"""
import csv
import types
from collections import namedtuple

import numpy as np
import torch

from tests import molecules_reference as MR
from tests import preprocess_reference as P

LAYOUTS = {"gdb13": (5, 3, 0, 0), "imp_H": (5, 3, 4, 0), "chirality": (5, 3, 0, 3), "imp_H+chirality": (4, 3, 4, 3)}


def statistics(nodes, edges):
    """int64 (n_nodes_hist [N+1], node_sums [F], n_edges_hist [10], bonds [Ef]) of molecules nodes [M, N, F] /
    edges [M, N, N, Ef]: the counts the reference's histograms accumulate, in integers"""
    M, N, F = nodes.shape
    Ef = edges.shape[3]
    n_nodes_hist = np.zeros(N + 1, np.int64)
    node_sums = np.zeros(F, np.int64)
    n_edges_hist = np.zeros(10, np.int64)
    bonds = np.zeros(Ef, np.int64)
    for m in range(M):
        n = P.n_atoms(nodes[m])                          # GetNumAtoms(): rows up to the last atom
        n_nodes_hist[n] += 1
        node_sums += nodes[m].astype(np.int64).sum(0)
        for i in range(n):
            ne = min(int(edges[m, i].astype(np.int64).sum()), 10)
            n_edges_hist[ne - 1] += 1                    # an atom without bonds lands in bin -1, the last one
        bonds += edges[m].astype(np.int64).sum((0, 1)) // 2
    return n_nodes_hist, node_sums, n_edges_hist, bonds


def constants(layout, N=13, Ef=3, B=20, device="cpu", training_set="/nonexistent/train.smi",
              dataset_dir="/nonexistent/"):
    """reference-style constants of one of the four layouts, with what the preprocessing phase reads"""
    A, Fc, H, C = LAYOUTS[layout]
    fields = dict(dim_nodes=[N, A + Fc + H + C], dim_edges=[N, N, Ef], max_n_nodes=N,
                  n_node_features=A + Fc + H + C, n_edge_features=Ef, n_atom_types=A, n_formal_charge=Fc, n_imp_H=H,
                  n_chirality=C, use_explicit_H=False, ignore_H=not H, use_chirality=bool(C),
                  atom_types=["C", "N", "O", "S", "Cl", "Br"][:A], formal_charge=[-1, 0, 1][:Fc],
                  imp_H=list(range(H)), chirality=["None", "R", "S"][:C], int_to_bondtype={}, device=device,
                  tensorboard_dir="/nonexistent", batch_size=B, restart=False, training_set=training_set,
                  dataset_dir=dataset_dir)
    return namedtuple("constants", sorted(fields))(**fields)


def preprocessing_graphs(ref, C, nodes, edges, smiles_keys=None):
    """the reference's PreprocessingGraph (float64 padded features, n_nodes) for each molecule; `molecule` is a stub
    RWMol whose SMILES is smiles_keys[m] (None: molecule=False as PreprocessingGraph leaves it, get_smiles -> None)"""
    graphs = []
    for m in range(nodes.shape[0]):
        g = ref.MolecularGraph.PreprocessingGraph.__new__(ref.MolecularGraph.PreprocessingGraph)
        g.constants = C
        g.node_features, g.edge_features = nodes[m].astype(np.float64), edges[m].astype(np.float64)
        g.n_nodes = P.n_atoms(nodes[m])
        g.molecule = False
        if smiles_keys is not None and smiles_keys[m] is not None:
            mol = MR.RWMol()
            mol.atoms, mol.bonds = [(smiles_keys[m], 0)], []
            g.molecule = mol
        graphs.append(g)
    return graphs


def reference_ts_properties(ref, graphs, spans, batch_size, is_training_set=True):
    """DataProcesser.get_ts_properties over the groups' graph slices [start, stop), in order"""
    dp = types.SimpleNamespace(is_training_set=is_training_set, ts_properties=None)
    for start, stop in spans:
        if dp.is_training_set:
            analyzer = ref.Analyzer.Analyzer()
            props = analyzer.evaluate_training_set(preprocessing_graphs=graphs[start:stop])
            if dp.ts_properties:
                dp.ts_properties = analyzer.combine_ts_properties(prev_properties=dp.ts_properties,
                                                                  next_properties=props, weight_next=batch_size)
            else:
                dp.ts_properties = props
        else:
            dp.ts_properties = None
    return dp.ts_properties


def write_ts_properties(path, training_set_properties):
    """the CSV util.write_ts_properties writes: one `key;value` row per property, numpy arrays as a list of their
    elements, one-element tensors as a float, other tensors as a list of floats, anything else as it is"""
    with open(path, "w") as f:
        w = csv.writer(f, delimiter=";")
        for key, value in training_set_properties.items():
            if isinstance(value, np.ndarray):
                value = list(value)
            elif isinstance(value, torch.Tensor):
                value = float(value) if value.numel() == 1 else [float(v) for v in value]
            w.writerow([key, value])


def assert_identical(got, want):
    """same keys in the same order; each value of the same type, dtype, device and shape, and the same bits"""
    assert list(got) == list(want)
    for k in want:
        a, b = got[k], want[k]
        assert type(a) is type(b), (k, type(a), type(b))
        if isinstance(b, torch.Tensor):
            assert (a.dtype, a.device, a.shape) == (b.dtype, b.device, b.shape), k
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), (k, a, b)
        elif isinstance(b, np.ndarray):
            assert (a.dtype, a.shape) == (b.dtype, b.shape), k
            assert a.tobytes() == b.tobytes(), (k, a, b)
        elif isinstance(b, list):
            assert a == b and all(type(x) is type(y) for x, y in zip(a, b)), k
        else:
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), (k, a, b)


def parse_csv(path):
    """{key: list of floats} of a train.csv, whatever numpy's repr of its values"""
    out = {}
    with open(path) as f:
        for key, value in csv.reader(f, delimiter=";"):
            cleaned = value.replace("np.float64(", "").replace("np.float32(", "").replace(")", "")
            out[key] = [float(v) for v in cleaned.strip("[]").split(",") if v.strip()]
    return out
