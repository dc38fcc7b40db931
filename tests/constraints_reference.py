"""
numpy restatement of the constraint rule (graphinvent_b200/csrc/constraints.cuh), for the constraint tests.

A constraint set here is a dict with the table's fields (`table_dict`): min_atoms, max_atoms, min_rings, max_rings,
min_ring_size, min_type [A], max_type [A], max_charge [CH], max_bond [Ef]; 0 is off for a minimum and for
min_ring_size, -1 for a maximum.  `mask(...)` gives, for one state, a bool per flat APD index: True where
`gib_action_mask_logits_constrained` writes -inf, the action rule (action_mask_reference) and the attachment points
(scaffold_route_reference) included, with the dead-end rule on terminate.  `check(...)` gives the flags of
`gib_constraints_check` for one finished molecule.
"""
from collections import deque

import numpy as np

try:
    from . import action_mask_reference as AM
    from . import scaffold_route_reference as SR
except ImportError:             # run as a plain module
    import action_mask_reference as AM
    import scaffold_route_reference as SR

OVER_MAX, SMALL_RING, UNDER_MIN, DEAD_END = 1, 2, 4, 8
HDR = 8


def table_dict(values, A, CH, Ef):
    """the fields of a table's words (GIB_CONS_* order)"""
    v = np.asarray(values, np.int64)
    return dict(min_atoms=int(v[0]), max_atoms=int(v[1]), min_rings=int(v[2]), max_rings=int(v[3]),
                min_ring_size=int(v[4]), min_type=v[HDR:HDR + A], max_type=v[HDR + A:HDR + 2 * A],
                max_charge=v[HDR + 2 * A:HDR + 2 * A + CH], max_bond=v[HDR + 2 * A + CH:HDR + 2 * A + CH + Ef])


def off_values(A, CH, Ef):
    """the words of a table with every field off"""
    v = np.full(HDR + 2 * A + CH + Ef, -1, np.int32)
    v[:HDR] = 0
    v[1] = v[3] = -1
    v[HDR:HDR + A] = 0
    return v


def adjacency(edges, n):
    """bool [n, n]: atoms i and j are bonded (any bond type)"""
    return (np.asarray(edges)[:n, :n] != 0).any(-1)


def summary(nodes, edges, n, A, CH, Ef):
    """(count per type [A], count per charge index [CH], bonds per type [Ef], cycle rank) of a state of n atoms"""
    nd, ed = np.asarray(nodes), np.asarray(edges)
    first = lambda row: int(np.flatnonzero(row)[0]) if row.any() else 0
    tc = np.zeros(A, np.int64)
    cc = np.zeros(CH, np.int64)
    for i in range(n):
        tc[first(nd[i, :A])] += 1
        cc[first(nd[i, A:A + CH])] += 1
    iu = np.triu_indices(n, 1)
    bc = (ed[:n, :n][iu] != 0).sum(0).astype(np.int64) if n > 1 else np.zeros(Ef, np.int64)
    rank = int(bc.sum()) - n + 1 if n >= 1 else 0
    return tc, cc, bc, rank


def bfs(adj, src, skip=-1):
    """shortest-path distances from src over the bool adjacency adj (None: unreached); skip: the bond (src, skip) is
    left out"""
    n = adj.shape[0]
    dist = [None] * n
    dist[src] = 0
    q = deque([src])
    while q:
        u = q.popleft()
        for v in np.flatnonzero(adj[u]):
            if dist[v] is None and not (u == src and v == skip):
                dist[v] = dist[u] + 1
                q.append(v)
    return dist


def girth(adj):
    """the length of the shortest cycle (None: a forest), from every bond (u, v): dist(u, v) without it, plus one"""
    n = adj.shape[0]
    g = None
    for u in range(n):
        for v in range(u + 1, n):
            if adj[u, v]:
                d = bfs(adj, u, skip=v)[v]
                if d is not None and (g is None or d + 1 < g):
                    g = d + 1
    return g


def below(t, tc, n, rank):
    return n < t["min_atoms"] or rank < t["min_rings"] or bool((tc < t["min_type"]).any())


def cons_forbidden(t, nodes, edges, n, N, A, CH, H, C, Ef):
    """bool [apd - 1]: the maxima and the ring-size bound on every non-terminate action"""
    apd = N * (A * CH * max(H, 1) * max(C, 1) * Ef + Ef) + 1
    kind, to, at, q, _, _, bt = (x[:-1] for x in AM.decode(apd, N, A, CH, H, C, Ef))
    tc, cc, bc, rank = summary(nodes, edges, n, A, CH, Ef)
    f = np.zeros(apd - 1, bool)
    off = lambda m: m < 0
    ma = t["max_atoms"]
    mt, mc, mb = t["max_type"][at], t["max_charge"][q], t["max_bond"][bt]
    add = (~off(mt) & (tc[at] >= mt)) | (~off(mc) & (cc[q] >= mc)) | ((n > 0) & ~off(mb) & (bc[bt] >= mb))
    if ma >= 0 and n >= ma:
        add[:] = True
    conn = ~off(mb) & (bc[bt] >= mb)
    if t["max_rings"] >= 0 and rank >= t["max_rings"]:
        conn[:] = True
    m = t["min_ring_size"]
    if m > 0 and n >= 1:
        dist = bfs(adjacency(edges, n), n - 1)
        small = np.array([to_ < n and dist[to_] is not None and dist[to_] + 1 < m for to_ in to])
        conn |= small
    f[kind == 0] = add[kind == 0]
    f[kind == 1] = conn[kind == 1]
    return f


def mask(t, nodes, edges, n, N, A, CH, H, C, Ef, V=None, order=None, imp_h=None, scaffold=None):
    """bool [apd]: every entry the constrained launch writes -inf into.  scaffold = (k, protect bool [>= k]) of the
    slot's scaffold with attachment points, or None"""
    f = AM.forbidden(nodes, edges, n, N, A, CH, H, C, Ef, V, order, imp_h).copy()
    if scaffold is not None:
        k, protect = scaffold
        per_node = A * CH * max(H, 1) * max(C, 1) * Ef
        f |= SR.mask_row(n, k, protect, N, Ef, per_node)
    f[:-1] |= cons_forbidden(t, nodes, edges, n, N, A, CH, H, C, Ef)
    tc, _, _, rank = summary(nodes, edges, n, A, CH, Ef)
    f[-1] = below(t, tc, n, rank) and not f[:-1].all()
    return f


def check(t, nodes, edges, n, N, A, CH, H, C, Ef, V=None, order=None, imp_h=None, scaffold=None):
    """the GIB_CONS_* flags of one finished molecule"""
    tc, cc, bc, rank = summary(nodes, edges, n, A, CH, Ef)
    over = lambda cnt, mx: bool(((mx >= 0) & (cnt > mx)).any())
    f = 0
    if ((t["max_atoms"] >= 0 and n > t["max_atoms"]) or (t["max_rings"] >= 0 and rank > t["max_rings"])
            or over(tc, t["max_type"]) or over(cc, t["max_charge"]) or over(bc, t["max_bond"])):
        f |= OVER_MAX
    if below(t, tc, n, rank):
        f |= DEAD_END if mask(t, nodes, edges, n, N, A, CH, H, C, Ef, V, order, imp_h, scaffold)[:-1].all() \
            else UNDER_MIN
    m = t["min_ring_size"]
    if m > 0 and n:
        g = girth(adjacency(edges, n))
        if g is not None and g < m:
            f |= SMALL_RING
    return f
