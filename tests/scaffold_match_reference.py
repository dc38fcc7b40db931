"""Python restatement of the scaffold-first decoding order (graphinvent_b200.preprocess.scaffold_first,
`gib_scaffold_first` in csrc/preprocess.cu), the oracle of its tests.  Written from the rule in include/gib200.h:

  * an embedding of scaffold s (k atoms) in a molecule (n atoms) is an injective phi with node row phi(i) == scaffold
    row i (all F bytes), edge cell (phi(i), phi(j)) == scaffold cell (i, j) for all i != j (all Ef bytes: an induced
    match of the same bond types) and, with attachment points, no bond from a protected scaffold atom out of the image;
  * the chosen one is the lexicographically smallest (phi(0), ..., phi(k-1)), found by a depth-first search whose
    nodes (one per assignment) are counted against a budget exactly as the kernel counts them;
  * the order is phi(0..k-1), then breadth-first layers out of the image, each layer highest-ranked atom first.

`brute_force` states the embedding rule alone, over every injective map (itertools.permutations): the search's
pruning must never change its answer.
"""
import itertools

import numpy as np

from tests import preprocess_reference as P

PP_EMPTY, PP_DISCONNECTED, PP_BAD_RANKING, PP_MATCH_BUDGET = 4, 8, 16, 32      # GIB_PP_* (include/gib200.h)
NO_MOLECULE = 2**31 - 1


def n_atoms(nodes):
    return P.n_atoms(np.asarray(nodes))


def _any(edges, n):
    """bool [n, n]: a bond of any type"""
    return np.asarray(edges)[:n, :n].any(-1)


def is_embedding(nodes, edges, sc_nodes, sc_edges, phi, protect=None):
    """rules 1-3 for the map phi (a sequence of k molecule atoms), stated directly"""
    k, n = len(phi), n_atoms(nodes)
    if len(set(phi)) != k or any(a < 0 or a >= n for a in phi):
        return False
    o = np.asarray(phi, np.int64)
    if not np.array_equal(nodes[o], sc_nodes[:k]) or not np.array_equal(edges[o][:, o], sc_edges[:k, :k]):
        return False
    if protect is not None:
        outside = np.setdiff1d(np.arange(n), o)
        bonded = _any(edges, n)
        for i in range(k):
            if protect[i] and bonded[o[i], outside].any():
                return False
    return True


def brute_force(nodes, edges, sc_nodes, sc_edges, protect=None):
    """the smallest embedding over every injective map in lexicographic order (None: no embedding)"""
    k, n = n_atoms(sc_nodes), n_atoms(nodes)
    for phi in itertools.permutations(range(n), k):
        if is_embedding(nodes, edges, sc_nodes, sc_edges, phi, protect):
            return list(phi)
    return None


def _bits(mask):
    return sum(1 << int(a) for a in np.flatnonzero(mask))


def search(nodes, edges, sc_nodes, sc_edges, protect=None, budget=1 << 20):
    """("found", phi) / ("none", None) / ("budget", None): the kernel's depth-first search.  Depth i's candidates are
    the atoms whose row is scaffold row i and whose degree fits (>=, == for a protected atom), unused, bonded to every
    assigned phi(j) by the type of the scaffold's (i, j) bond (its first non-zero byte) or not bonded to phi(j) at all
    where the scaffold has no (i, j) bond; ascending index; a leaf is confirmed by `is_embedding`'s byte comparison."""
    nodes, edges, sc_nodes, sc_edges = map(np.asarray, (nodes, edges, sc_nodes, sc_edges))
    k, n = n_atoms(sc_nodes), n_atoms(nodes)
    Ef = edges.shape[2]
    bonded = _any(edges, n)
    mdeg = bonded.sum(1)
    sdeg = _any(sc_edges, k).sum(1)
    typed = [[_bits(edges[a, :n, t] != 0) for t in range(Ef)] for a in range(n)]
    anyb = [_bits(bonded[a]) for a in range(n)]
    full = (1 << n) - 1
    label = []
    for i in range(k):
        prot = protect is not None and protect[i]
        ok = [(mdeg[a] == sdeg[i] or (mdeg[a] > sdeg[i] and not prot)) and np.array_equal(nodes[a], sc_nodes[i])
              for a in range(n)]
        label.append(_bits(np.array(ok, bool)))
    stype = [[next((t for t in range(Ef) if sc_edges[i, j, t]), -1) for j in range(k)] for i in range(k)]
    phi, used, count = [], 0, 0

    def candidates(i):
        c = label[i] & ~used & full
        for j in range(i):
            t = stype[i][j]
            c &= typed[phi[j]][t] if t >= 0 else ~anyb[phi[j]] & full
        return c

    stack = [candidates(0)]
    while True:
        d = len(stack) - 1
        c = stack[d]
        if not c:
            stack.pop()
            if d == 0:
                return "none", None
            used &= ~(1 << phi.pop())
            continue
        count += 1
        if count > budget:
            return "budget", None
        a = (c & -c).bit_length() - 1
        stack[d] = c & ~(1 << a)
        phi.append(a)
        used |= 1 << a
        if d + 1 < k:
            stack.append(candidates(d + 1))
            continue
        if is_embedding(nodes, edges, sc_nodes, sc_edges, phi, None):
            return "found", list(phi)
        used &= ~(1 << phi.pop())


def layers(edges, n, seed_atoms, ranking):
    """seed_atoms, then breadth-first layers out of them, each layer highest-ranked atom first (fewer than n atoms:
    the molecule is disconnected)"""
    bonded = _any(edges, n)
    order, seen, layer = list(seed_atoms), set(seed_atoms), list(seed_atoms)
    while layer:
        nxt = sorted({int(b) for a in layer for b in np.flatnonzero(bonded[a])} - seen, key=lambda v: -ranking[v])
        seen |= set(nxt)
        order += nxt
        layer = nxt
    return order


def choose(nodes, edges, sc_nodes, sc_edges, protect=None, sid=None, budget=1 << 20):
    """("found", s, phi) / ("none", -1, None) / ("budget", s, None): scaffold sid only (-1: none), or sid=None the first
    scaffold in table order that embeds, after the cheap rejects (more atoms or more bonds than the molecule)"""
    n = n_atoms(nodes)
    mbonds = int(_any(edges, n).sum()) // 2
    S = sc_nodes.shape[0]
    cands = range(S) if sid is None else ([sid] if 0 <= sid < S else [])
    for s in cands:
        k = n_atoms(sc_nodes[s])
        if k < 1 or k > n or int(_any(sc_edges[s], k).sum()) // 2 > mbonds:
            continue
        res, phi = search(nodes, edges, sc_nodes[s], sc_edges[s], None if protect is None else protect[s], budget)
        if res == "budget":
            return res, s, None
        if res == "found":
            return res, s, phi
    return "none", -1, None


def scaffold_first(nodes, edges, sc_nodes, sc_edges, rankings, protect=None, ids=None, budget=1 << 20):
    """(out_nodes, out_edges, order, ids, status [flags, first flagged molecule]) of a valid stack (the count stage's
    checks are not restated); rankings int [M, N] (row m's first n entries a permutation)"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    M, N = nodes.shape[:2]
    out_n, out_e = np.zeros_like(nodes), np.zeros_like(edges)
    order = np.full((M, N), -1, np.int32)
    out_ids = np.full(M, -1, np.int32)
    flags, first = 0, NO_MOLECULE

    def flag(bit, m):
        nonlocal flags, first
        flags |= bit
        first = min(first, m)

    for m in range(M):
        n = n_atoms(nodes[m])
        if n == 0:
            flag(PP_EMPTY, m)
            continue
        rk = [int(r) for r in rankings[m, :n]]
        if sorted(rk) != list(range(n)):
            flag(PP_BAD_RANKING, m)
            continue
        if len(layers(edges[m], n, [0], rk)) != n:
            flag(PP_DISCONNECTED, m)
            continue
        res, s, phi = choose(nodes[m], edges[m], sc_nodes, sc_edges, protect,
                             None if ids is None else int(ids[m]), budget)
        if res == "budget":
            flag(PP_MATCH_BUDGET, m)
            continue
        o = layers(edges[m], n, phi, rk) if res == "found" else list(range(n))
        order[m, :n] = o
        out_ids[m] = s
        out_n[m], out_e[m] = reorder(nodes[m], edges[m], o)
    return out_n, out_e, order, out_ids, (flags, first)


def reorder(nodes, edges, order):
    """node rows and edge rows / columns in `order`, zero past len(order)"""
    X, E = np.zeros_like(nodes), np.zeros_like(edges)
    o = np.asarray(order, np.int64)
    X[:o.size] = nodes[o]
    E[:o.size, :o.size] = edges[o][:, o]
    return X, E


# ---- inputs ----------------------------------------------------------------------------------------------------------
def one_hot_rows(rng, n, layout, n_types=2):
    """int8 [n, F] node rows, one-hot per segment of the layout, each segment's index drawn from its first n_types
    entries (a small alphabet: many equal rows, many candidate embeddings)"""
    rows = []
    for _ in range(n):
        parts = []
        for w in P.segments(*layout):
            v = np.zeros(w, np.int8)
            v[rng.integers(0, min(w, n_types))] = 1
            parts.append(v)
        rows.append(np.concatenate(parts))
    return np.stack(rows)


def random_molecule(rng, n, N, layout, Ef, n_types=2, extra_bonds=0.25):
    """a connected molecule of n atoms padded to N: a random tree plus extra bonds, bond types drawn from Ef"""
    F = sum(P.segments(*layout))
    X = np.zeros((N, F), np.int8)
    E = np.zeros((N, N, Ef), np.int8)
    X[:n] = one_hot_rows(rng, n, layout, n_types)
    for a in range(1, n):
        b = int(rng.integers(0, a))
        t = int(rng.integers(0, Ef))
        E[a, b, t] = E[b, a, t] = 1
    for a in range(n):
        for b in range(a + 1, n):
            if not E[a, b].any() and rng.random() < extra_bonds / max(n, 1):
                t = int(rng.integers(0, Ef))
                E[a, b, t] = E[b, a, t] = 1
    return X, E


def shuffle(nodes, edges, rng):
    """the molecule with its atoms in a random order"""
    n = n_atoms(nodes)
    perm = rng.permutation(n)
    return reorder(nodes, edges, perm)


def cut_scaffold(nodes, edges, k, rng):
    """a connected k-atom induced subgraph of the molecule, its atoms in an order where each bonds to an earlier one
    (the order a scaffold table accepts)"""
    n = n_atoms(nodes)
    bonded = _any(edges, n)
    start = int(rng.integers(0, n))
    picked = [start]
    while len(picked) < k:
        front = sorted({int(b) for a in picked for b in np.flatnonzero(bonded[a])} - set(picked))
        if not front:
            break
        picked.append(int(rng.choice(front)))
    # an order the route plan accepts: every atom after the first bonds to an earlier one
    order, inside = [picked[0]], set(picked)
    for a in order:
        order += [int(b) for b in np.flatnonzero(bonded[a]) if int(b) in inside and int(b) not in order]
    return reorder(nodes, edges, order)
