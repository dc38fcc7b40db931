"""
numpy restatement of the generator's action rule (graphinvent_b200/csrc/action_mask.cuh), for the action-mask tests.

`forbidden(...)` gives, for one state, a bool per flat APD index: True where `gib_action_mask_logits` writes -inf.
Its structural part is the reference's `GraphGenerator.get_invalid_actions` (GraphGenerator.py:573-657), quirks
included, on every index of the action space.  One deliberate deviation, which the reference cannot show: outside
the gdb13 layout L0 the reference has no verdict for an add into a graph that already holds max_n_nodes atoms (it
raises IndexError one step later, indexing nodes[b, N]); here, as in the round kernel, such an add is forbidden in
every layout, which is the reference's own L0 verdict.
"""
import numpy as np

BOND_HALF_ORDERS = (2, 4, 6, 3)     # single, double, triple, aromatic


def decode(apd_len, N, A, CH, H, C, Ef):
    """kind (0 add, 1 connect, 2 terminate), bond_to, atom, charge, imp_h, chirality, bond type of every index"""
    a = np.arange(apd_len - 1)
    per = A * CH * max(H, 1) * max(C, 1) * Ef
    len_add = N * per
    kind = np.where(a < len_add, 0, 1)
    r = np.where(kind == 0, a, 0)
    bt = r % Ef
    r = r // Ef
    ch = np.zeros_like(a)
    ih = np.zeros_like(a)
    if C:
        ch = r % C
        r = r // C
    if H:
        ih = r % H
        r = r // H
    q = r % CH
    r = r // CH
    t = r % A
    to = r // A
    c = a - len_add
    to = np.where(kind == 1, c // Ef, to)
    bt = np.where(kind == 1, c % Ef, bt)
    kind = np.append(kind, 2)
    pad = lambda x: np.append(x, 0)
    return kind, pad(to), pad(t), pad(q), pad(ih), pad(ch), pad(bt)


def structure(n, edges, N, A, CH, H, C, Ef):
    """bool [apd]: the structural rule for a state of n atoms with edges [N, N, Ef]"""
    apd_len = N * (A * CH * max(H, 1) * max(C, 1) * Ef + Ef) + 1
    kind, to, t, q, ih, ch, bt = decode(apd_len, N, A, CH, H, C, Ef)
    e5 = n if (H == 0 and C == 0) else (ch if (H and C) else bt)
    e5 = np.broadcast_to(e5, kind.shape)
    add = (n >= N) | ((n > 0) & (to >= n)) | ((n == 0) & (to != 0)) | (e5 >= N)
    bf = n - 1 if n > 0 else N - 1
    psum = edges.astype(np.float64)[np.minimum(to, N - 1), bf].sum(-1)
    conn = (n == 0) | (to >= n) | (to == n - 1) | (psum == 1)
    return np.where(kind == 0, add, np.where(kind == 1, conn, False))


def atom_usage(nodes, edges, n, A, CH, H, V, order, imp_h):
    """used and limit (half-bond units) of atoms 0..n-1 of one state"""
    nd = np.asarray(nodes)
    t = np.array([np.flatnonzero(nd[i, :A])[0] if nd[i, :A].any() else 0 for i in range(n)], np.int64)
    q = np.array([np.flatnonzero(nd[i, A:A + CH])[0] if nd[i, A:A + CH].any() else 0 for i in range(n)], np.int64)
    used = (np.asarray(edges, np.int64)[:n] * np.asarray(order, np.int64)).sum((1, 2))
    if H:
        seg = nd[:n, A + CH:A + CH + H]
        h = np.array([np.flatnonzero(seg[i])[0] if seg[i].any() else 0 for i in range(n)], np.int64)
        used = used + 2 * np.asarray(imp_h, np.int64)[h]
    limit = 2 * np.asarray(V, np.int64)[t, q] if n else np.zeros(0, np.int64)
    return used, limit


def forbidden(nodes, edges, n, N, A, CH, H, C, Ef, V=None, order=None, imp_h=None):
    """bool [apd]: the whole rule (structure, and valence when the table V [A, CH] is given)"""
    s = structure(n, edges, N, A, CH, H, C, Ef)
    if V is None:
        return s
    order = np.asarray(order if order is not None else BOND_HALF_ORDERS[:Ef], np.int64)
    imp_h = np.asarray(imp_h if imp_h is not None else np.arange(H), np.int64)
    apd_len = s.size
    kind, to, t, q, ih, ch, bt = decode(apd_len, N, A, CH, H, C, Ef)
    used, limit = atom_usage(nodes, edges, n, A, CH, H, V, order, imp_h)
    used = np.append(used, 0)[np.minimum(to, n)] if n else np.zeros_like(to)
    lim_to = np.append(limit, 0)[np.minimum(to, n)] if n else np.zeros_like(to)
    o = order[bt]
    own = 2 * imp_h[ih] if H else np.zeros_like(to)
    lim_new = 2 * np.asarray(V, np.int64)[t, q]
    if n == 0:
        add_v = own > lim_new
    else:
        add_v = (o + own > lim_new) | (used + o > lim_to)
    if n > 0:
        u_last, l_last = atom_usage(nodes, edges, n, A, CH, H, V, order, imp_h)
        conn_v = (used + o > lim_to) | (u_last[n - 1] + o > l_last[n - 1])
    else:
        conn_v = np.zeros_like(s)
    v = np.where(kind == 0, add_v, np.where(kind == 1, conn_v, False))
    return s | (v & ~s)


def valence_ok(nodes, edges, n, A, CH, H, V, order, imp_h):
    """True when every atom of a finished molecule is within its limit"""
    if n == 0:
        return True
    used, limit = atom_usage(nodes, edges, n, A, CH, H, V, np.asarray(order), np.asarray(imp_h))
    return bool((used <= limit).all())
