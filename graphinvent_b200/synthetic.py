"""
Synthetic molecular-graph batches in the `BlockDatasetLoader` tensor layout.

Layout contract (reference `BlockDatasetLoader.py:135-143`): `nodes` float32
`[B, max_n_nodes, n_node_features]`, `edges` float32 `[B, N, N, n_edge_features]`
(dense, zero padded, symmetric one-hot bond types), `apds` float32 `[B, APD]`.

Generator recipe = SURVEY.md §8(d): per graph `n` atoms; atom type uniform over the
atom list, formal charge fixed to the neutral slot (node rows sum to 2, as in the
real gdb13 data); a random recursive tree (atom i bonds to a uniformly chosen
earlier atom of degree < 4) plus floor(n/6) ring closures between non-adjacent
atoms of degree < 4; bond type ~ Categorical(0.84, 0.14, 0.02) on tree bonds,
single on closures.  With n_edge_features = 4 (the reference's `use_aromatic_bonds`)
the fourth, aromatic type has weight 0.10 and the four are renormalised; fewer types
take the leading weights, renormalised.  Targets are uniform-random positive APD rows.
"""
import numpy as np

BOND_P = (0.84, 0.14, 0.02, 0.10)


def random_graphs(batch, max_n_nodes, n_atom_types, n_charges, n_edge_features=3,
                  n_atoms=None, seed=0, min_atoms=None):
    """Returns (nodes int8 [B,N,F], edges int8 [B,N,N,Ef]) with F = types + charges.

    n_atoms=None -> every graph has max_n_nodes atoms; min_atoms set -> sizes drawn
    uniformly from [min_atoms, max_n_nodes] (0 gives empty graphs)."""
    rng = np.random.default_rng(seed)
    N, F, Ef = max_n_nodes, n_atom_types + n_charges, n_edge_features
    nodes = np.zeros((batch, N, F), np.int8)
    edges = np.zeros((batch, N, N, Ef), np.int8)
    neutral = n_atom_types + n_charges // 2
    p = np.asarray(BOND_P[:Ef], np.float64)
    p /= p.sum()
    for b in range(batch):
        if n_atoms is not None:
            n = n_atoms
        elif min_atoms is not None:
            n = int(rng.integers(min_atoms, N + 1))
        else:
            n = N
        if n == 0:
            continue
        nodes[b, np.arange(n), rng.integers(0, n_atom_types, n)] = 1
        nodes[b, :n, neutral] = 1
        deg = np.zeros(n, np.int64)
        adj = np.zeros((n, n), bool)
        for i in range(1, n):
            cand = np.flatnonzero(deg[:i] < 4)
            if cand.size == 0:
                break
            j = int(cand[rng.integers(cand.size)])
            t = int(rng.choice(Ef, p=p))
            edges[b, i, j, t] = edges[b, j, i, t] = 1
            adj[i, j] = adj[j, i] = True
            deg[i] += 1
            deg[j] += 1
        for _ in range(n // 6):
            ok = np.flatnonzero(deg < 4)
            if ok.size < 2:
                break
            i, j = (int(v) for v in rng.choice(ok, 2, replace=False))
            if adj[i, j]:
                continue
            edges[b, i, j, 0] = edges[b, j, i, 0] = 1
            adj[i, j] = adj[j, i] = True
            deg[i] += 1
            deg[j] += 1
    return nodes, edges


def random_targets(batch, apd_len, seed=0):
    """Uniform-random positive APD rows, renormalised (SURVEY §8d)."""
    rng = np.random.default_rng(seed + 7919)
    t = rng.random((batch, apd_len), np.float32) + 1e-3
    return (t / t.sum(1, keepdims=True)).astype(np.float32)


def corner_case_graphs(max_n_nodes, n_node_features, n_edge_features=3):
    """The degenerate inputs every generation run produces (SURVEY Appendix B):
    slot 0 = the dummy graph (all-ones node row 0 and a self-loop edges[0,0,0,0]=1,
    `GraphGenerator.py:418-423`), slot 1 = empty graph, slot 2 = one isolated atom,
    slot 3 = a node of degree 5 (valence is not enforced while sampling),
    slot 4 = a two-atom molecule with a triple bond."""
    N, F, Ef = max_n_nodes, n_node_features, n_edge_features
    nodes = np.zeros((5, N, F), np.int8)
    edges = np.zeros((5, N, N, Ef), np.int8)
    nodes[0, 0, :] = 1
    edges[0, 0, 0, 0] = 1
    nodes[2, 0, 0] = nodes[2, 0, F - 2] = 1
    k = min(6, N)
    for i in range(k):
        nodes[3, i, i % max(1, F - 3)] = nodes[3, i, F - 2] = 1
    for i in range(1, k):
        edges[3, 0, i, 0] = edges[3, i, 0, 0] = 1
    nodes[4, 0, 0] = nodes[4, 1, 1] = 1
    nodes[4, :2, F - 2] = 1
    edges[4, 0, 1, Ef - 1] = edges[4, 1, 0, Ef - 1] = 1
    return nodes, edges
