"""Python restatement of the Murcko scaffolds (graphinvent_b200.preprocess.murcko_scaffolds, `gib_murcko` in
csrc/preprocess.cu), the oracle of its tests.  Written from the rule in include/gib200.h:

  * kept atoms, twice: RDKit's form (`keep_rdkit`: the ring atoms, by cycle membership, plus one shortest path between
    every pair of ring atoms, plus the atoms with a double bond -- edge feature 1 -- to those) and the 2-core form
    (`keep_core`: atoms of degree <= 1 peeled until none is left, plus the same double-bond clause);
  * the scaffold: the induced subgraph on the kept atoms, breadth-first from the lowest kept index, each layer in
    increasing index;
  * the 64-bit colour-refinement hash, bit for bit as the kernel computes it;
  * the deduplication: a molecule's scaffold joins the first table entry of equal hash, atom count and bond count in
    which `scaffold_match_reference.search` embeds the entry (the smallest embedding: the isomorphism the attachment
    points are read through), else it is appended.
"""
from collections import deque

import numpy as np

from tests import scaffold_match_reference as SM

MASK = (1 << 64) - 1
EMPTY = MASK
PP_MATCH_BUDGET = 32


def n_atoms(nodes):
    return SM.n_atoms(nodes)


def _bonded(edges, n):
    return np.asarray(edges)[:n, :n].any(-1)


def _double(edges, n, keep_set):
    """atoms outside keep_set with a double bond (edge feature 1) to an atom of it"""
    E = np.asarray(edges)
    if E.shape[2] < 2:
        return set()
    return {a for a in range(n) if a not in keep_set and any(E[a, b, 1] for b in keep_set)}


def _mask(n, N, atoms):
    keep = np.zeros(N, bool)
    keep[sorted(atoms)] = True
    return keep


def keep_core(nodes, edges):
    """bool [N]: the 2-core, peeled one atom at a time, plus the double-bond clause"""
    n, N = n_atoms(nodes), nodes.shape[0]
    adj = _bonded(edges, n)
    alive = set(range(n))
    changed = True
    while changed:
        changed = False
        for a in sorted(alive):
            if sum(adj[a, b] for b in alive) <= 1:
                alive.discard(a)
                changed = True
    return _mask(n, N, alive | _double(edges, n, alive))


def _path(adj, n, u, v, banned=None):
    """a shortest path u .. v (None: none) avoiding the edge `banned`"""
    prev = {u: None}
    q = deque([u])
    while q:
        a = q.popleft()
        if a == v:
            out = [v]
            while prev[out[-1]] is not None:
                out.append(prev[out[-1]])
            return out
        for b in np.flatnonzero(adj[a, :n]):
            b = int(b)
            if b not in prev and (a, b) != banned and (b, a) != banned:
                prev[b] = a
                q.append(b)
    return None


def keep_rdkit(nodes, edges):
    """bool [N]: ring atoms (an atom is on a cycle when one of its bonds lies on a cycle: its ends stay connected
    without it), one shortest path between every pair of ring atoms, plus the double-bond clause"""
    n, N = n_atoms(nodes), nodes.shape[0]
    adj = _bonded(edges, n)
    ring = set()
    for a in range(n):
        for b in range(a + 1, n):
            if adj[a, b] and _path(adj, n, a, b, banned=(a, b)) is not None:
                ring |= {a, b}
    kept = set(ring)
    ring = sorted(ring)
    for i, u in enumerate(ring):
        for v in ring[i + 1:]:
            kept |= set(_path(adj, n, u, v))
    return _mask(n, N, kept | _double(edges, n, kept))


def canonical_order(edges, keep):
    """kept atoms breadth-first from the lowest kept index, each layer in increasing index"""
    atoms = np.flatnonzero(keep)
    if atoms.size == 0:
        return []
    n = int(atoms[-1]) + 1
    adj = _bonded(edges, n)
    order, seen, layer = [int(atoms[0])], {int(atoms[0])}, [int(atoms[0])]
    while layer:
        nxt = sorted({int(b) for a in layer for b in np.flatnonzero(adj[a] & keep[:n])} - seen)
        seen |= set(nxt)
        order += nxt
        layer = nxt
    return order


def scaffold(nodes, edges, keep=None):
    """(scaffold nodes, scaffold edges, order, keep) of one molecule; order[i] = the molecule atom at scaffold
    position i"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    if keep is None:
        keep = keep_core(nodes, edges)
    order = canonical_order(edges, keep)
    X, E = SM.reorder(nodes, edges, order)
    return X, E, order, keep


# ---- the hash ---------------------------------------------------------------------------------------------------------
def mix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def wl_hash(nodes, edges):
    """the kernel's colour-refinement hash of a scaffold (k rounds over its k atoms)"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    k = n_atoms(nodes)
    nbrs = [[(int(b), int(np.flatnonzero(edges[a, b])[0])) for b in range(k) if edges[a, b].any()]
            for a in range(k)]
    bonds = sum(len(x) for x in nbrs) // 2
    col = []
    for a in range(k):
        h = 0
        for f in np.flatnonzero(nodes[a]):
            h += mix64((int(f) << 8) | (int(nodes[a, f]) & 0xFF))
        col.append(mix64(h & MASK))
    for _ in range(k):
        col = [mix64((col[a] + sum(mix64(col[b] ^ ((t + 1) << 56)) for b, t in nbrs[a])) & MASK) for a in range(k)]
    total = sum(mix64(c) for c in col) & MASK
    h = mix64(total ^ ((k << 32) | bonds))
    return EMPTY - 1 if h == EMPTY else h


def n_bonds(edges, k):
    return int(_bonded(edges, k).sum()) // 2


# ---- the deduplication -----------------------------------------------------------------------------------------------
class Table:
    """the scaffold table: entries (nodes, edges) in order, their hashes, counts and attachment points"""

    def __init__(self, N, F, Ef, known=None):
        self.N = N
        self.nodes, self.edges, self.hash, self.counts, self.attach = [], [], [], [], []
        if known is not None:
            kn, ke, kc, ka = (np.asarray(t) for t in known)
            for s in range(kn.shape[0]):
                self.nodes.append(kn[s])
                self.edges.append(ke[s])
                self.hash.append(wl_hash(kn[s], ke[s]))
                self.counts.append(int(kc[s]))
                self.attach.append(ka[s].astype(bool).copy())

    def find(self, X, E, h, budget):
        """(entry, phi) of the scaffold (X, E), (None, None) when new, ("budget", None) when a search runs out"""
        k = n_atoms(X)
        for s, hs in enumerate(self.hash):
            if hs != h or n_atoms(self.nodes[s]) != k or n_bonds(self.edges[s], k) != n_bonds(E, k):
                continue
            res, phi = SM.search(X, E, self.nodes[s], self.edges[s], None, budget)
            if res == "budget":
                return "budget", None
            if res == "found":
                return s, phi
        return None, None

    def arrays(self):
        S, N = len(self.nodes), self.N
        if S == 0:
            return None
        return (np.stack(self.nodes), np.stack(self.edges), np.array(self.counts, np.int64),
                np.stack(self.attach))


def murcko(nodes, edges, known=None, budget=1 << 20, keep_fn=keep_core):
    """(table (nodes, edges, counts, attachment) or None when empty, ids, keep, status (flags, first flagged)) of a
    valid, connected stack; known: an earlier (nodes, edges, counts, attachment)"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    M, N, F = nodes.shape
    T = Table(N, F, edges.shape[3], known)
    ids = np.full(M, -1, np.int32)
    keeps = np.zeros((M, N), bool)
    flags, first = 0, SM.NO_MOLECULE
    for m in range(M):
        X, E, order, keep = scaffold(nodes[m], edges[m], keep_fn(nodes[m], edges[m]))
        keeps[m] = keep
        k = len(order)
        if k == 0:
            continue
        h = wl_hash(X, E)
        s, phi = T.find(X, E, h, budget)
        if s == "budget":
            flags |= PP_MATCH_BUDGET
            first = min(first, m)
            continue
        if s is None:
            s, phi = len(T.nodes), list(range(k))
            T.nodes.append(X)
            T.edges.append(E)
            T.hash.append(h)
            T.counts.append(0)
            T.attach.append(np.zeros(N, bool))
        ids[m] = s
        T.counts[s] += 1
        n = n_atoms(nodes[m])
        bonded = _bonded(edges[m], n)
        for i in range(k):
            a = order[phi[i]]
            if (bonded[a] & ~keep[:n]).any():
                T.attach[s][i] = True
    return T.arrays(), ids, keeps, (flags, first)
