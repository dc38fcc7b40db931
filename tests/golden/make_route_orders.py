"""Writes tests/golden/route_orders.npz: the reference's decoding-route orders for given node rankings.

    python tests/golden/make_route_orders.py /path/to/reference

For every molecule of two sets -- the gdb13_1K training molecules (the graphs of preprocess_gdb13.npz) and a seeded
synthetic N = 38 set (graphinvent_b200.synthetic) -- and for each of R rankings -- the identity, the reversed one and
RANDOM seeded `random.shuffle(list(range(n)))` draws, as `PreprocessingGraph.node_remap` draws them with
use_canon=False -- it runs the unmodified reference's `PreprocessingGraph.breadth_first_search`,
`depth_first_search` (node_init = ranking[0], as node_remap passes it) and `reorder_nodes` on a stand-in object that
holds `n_nodes`, the unpadded `node_features` / `edge_features` and `constants.n_edge_features`.  RDKit and the
reference's `util` are stubbed at import: none of these methods touches them.

Stored per set S: S/nodes, S/edges (int8 padded inputs), S/rankings int32 [M, R, N] (-1 past the atom count),
S/orders int32 [M, R, 2, N] (route 0 = bfs, 1 = dfs; -1 past the atom count) and S/sha256_{bfs,dfs}: the SHA-256 of
the reordered int8 stacks padded back to N, all nodes of [M, R] then all edges.  `python_version` records the
interpreter the set iteration order came from.
"""
import hashlib
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

RANDOM = 3


def _annotation(name):
    if name.startswith("__"):
        raise AttributeError(name)
    return object


def load_reference(ref):
    import torch  # noqa: F401  (the reference imports it; loaded before the stubs exist)
    for name in ("rdkit", "rdkit.Chem", "rdkit.Chem.rdmolfiles"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["rdkit"].Chem = sys.modules["rdkit.Chem"]
    sys.modules["rdkit.Chem"].__getattr__ = _annotation                  # rdkit.Chem.Atom etc. in type annotations
    sys.modules["rdkit.Chem.rdmolfiles"].MolToSmiles = None
    sys.modules["util"] = types.ModuleType("util")
    sys.path.insert(0, os.path.join(ref, "graphinvent"))
    import MolecularGraph
    return MolecularGraph.PreprocessingGraph


def stand_in(nodes, edges, n):
    g = types.SimpleNamespace(n_nodes=n, node_features=nodes[:n].astype(np.int32),
                              edge_features=edges[:n, :n].astype(np.int32),
                              constants=types.SimpleNamespace(n_edge_features=edges.shape[2]))
    return g


def rankings_of(n, rng):
    out = [list(range(n)), list(range(n))[::-1]]
    for _ in range(RANDOM):
        r = list(range(n))
        rng.shuffle(r)
        out.append(r)
    return out


def run(PG, nodes, edges, seed):
    from tests.route_order_reference import n_atoms
    M, N, _ = nodes.shape
    R = RANDOM + 2
    rng = random.Random(seed)
    rankings = np.full((M, R, N), -1, np.int32)
    orders = np.full((M, R, 2, N), -1, np.int32)
    out_n = np.zeros((2, M, R) + nodes.shape[1:], np.int8)
    out_e = np.zeros((2, M, R) + edges.shape[1:], np.int8)
    for m in range(M):
        n = n_atoms(nodes[m])
        for k, ranking in enumerate(rankings_of(n, rng)):
            rankings[m, k, :n] = ranking
            for r, search in enumerate((PG.breadth_first_search, PG.depth_first_search)):
                g = stand_in(nodes[m], edges[m], n)
                g.node_ordering = search(g, node_ranking=ranking, node_init=ranking[0])
                PG.reorder_nodes(g)
                orders[m, k, r, :n] = [int(a) for a in g.node_ordering]
                out_n[r, m, k, :n] = g.node_features
                out_e[r, m, k, :n, :n] = g.edge_features
    digests = [hashlib.sha256(out_n[r].tobytes() + out_e[r].tobytes()).hexdigest() for r in (0, 1)]
    return rankings, orders, digests


def main(ref):
    from graphinvent_b200 import synthetic as S
    PG = load_reference(ref)
    z = np.load(os.path.join(HERE, "preprocess_gdb13.npz"))
    sets = {"gdb13": (z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]),
            "synthetic38": S.random_graphs(200, 38, 5, 3, n_edge_features=3, seed=38, min_atoms=1)}
    out = {"python_version": np.array(sys.version.split()[0])}
    for seed, (name, (nodes, edges)) in enumerate(sets.items()):
        rankings, orders, digests = run(PG, nodes, edges, seed)
        out.update({f"{name}/nodes": nodes, f"{name}/edges": edges, f"{name}/rankings": rankings,
                    f"{name}/orders": orders, f"{name}/sha256_bfs": np.array(digests[0]),
                    f"{name}/sha256_dfs": np.array(digests[1])})
        print(name, nodes.shape, "orders", orders.shape)
    np.savez_compressed(os.path.join(HERE, "route_orders.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/reference")
