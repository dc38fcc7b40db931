"""numpy / fp64 restatement of the conditional route likelihood p(molecule | scaffold)
(graphinvent_b200.graphed.RouteScorer.score(..., scaffold_ids=)), the oracle of its tests.

A molecule in decoding order whose first k atoms, with every bond among them, are scaffold s has the prefix state S_k
on its canonical route, as state 1 + m_k in build order (m_k: the bonds among those atoms).  The conditional route is
the route's last n_bonds - m_k + 1 states (tests/route_nll_reference.build_order_states), from S_k to terminate.  With
attachment points each state's logits are masked by the generator's rule (tests/scaffold_oracle.forbidden) before the
softmax."""
import numpy as np
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R


def n_bonds(edges):
    return int(np.asarray(edges).astype(np.int64).sum()) // 2


def prefix(nodes, edges, k):
    """the k-atom prefix state of one molecule: rows 0..k-1 and the bonds among them, padded like the molecule"""
    X, E = np.zeros_like(nodes), np.zeros_like(edges)
    X[:k], E[:k, :k] = nodes[:k], edges[:k, :k]
    return X, E


def prefix_scaffolds(nodes, edges, ks):
    """scaffold m = molecule m's ks[m]-atom prefix: int8 stacks [M, N, F] / [M, N, N, Ef]"""
    pairs = [prefix(nodes[m], edges[m], int(k)) for m, k in enumerate(ks)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def decoration_points(nodes, edges, k):
    """the scaffold atoms (< k) bonded to an atom >= k: the attachment points a decoration of this molecule uses"""
    return sorted({int(i) for i in range(k) if edges[i, k:].any()})


def forbidden(a, n, k, protect, N, Ef, per_node):
    """the generator's attachment-point rule for action a in a state of n atoms decorating a k-atom scaffold whose
    protected atoms are `protect` (bool [>= k]); terminate is never forbidden"""
    len_add = N * per_node
    if a < len_add:
        i = a // per_node
        return bool(i < k and protect[i])
    if a < len_add + N * Ef:
        i = (a - len_add) // Ef
        return bool(n - 1 < k or (i < k and protect[i]))
    return False


def mask_row(n, k, protect, N, Ef, per_node):
    """bool [apd]: every action `forbidden` forbids in that state"""
    apd = N * (per_node + Ef) + 1
    return np.array([forbidden(a, n, k, protect, N, Ef, per_node) for a in range(apd)], bool)


def conditional_states(nodes, edges, ids, sc_nodes, segs):
    """(X [S, N, F], E [S, N, N, Ef], actions [S], offsets [M + 1], state scaffold ids [S], state atom counts [S]) of
    every molecule's conditional route in build order (ids[m] = -1: the whole route)"""
    X, E, acts, off = R.build_order_states(nodes, edges, segs)
    keep, offsets, sid, n_at = [], [0], [], []
    for m in range(nodes.shape[0]):
        a, b = int(off[m]), int(off[m + 1])
        s = int(ids[m])
        first = a if s < 0 else a + 1 + n_bonds(prefix(nodes[m], edges[m], P.n_atoms(sc_nodes[s]))[1])
        keep += range(first, b)
        offsets.append(offsets[-1] + b - first)
        sid += [s] * (b - first)
        n_at += [P.n_atoms(X[i]) for i in range(first, b)]
    keep = np.array(keep, np.int64)
    return X[keep], E[keep], acts[keep], np.array(offsets, np.int64), np.array(sid, np.int64), np.array(n_at, np.int64)


def state_masks(sid, n_at, sc_nodes, protect, N, Ef, per_node):
    """bool [S, apd] masks of the conditional states (all False without attachment points or for id -1)"""
    apd = N * (per_node + Ef) + 1
    out = np.zeros((sid.shape[0], apd), bool)
    if protect is None:
        return out
    for i, (s, n) in enumerate(zip(sid, n_at)):
        if s >= 0:
            out[i] = mask_row(int(n), P.n_atoms(sc_nodes[s]), protect[s], N, Ef, per_node)
    return out


def protect_of(sc_nodes, attachment):
    """bool [S, N]: the scaffold atoms that are not attachment points (one index list per scaffold)"""
    k = [P.n_atoms(x) for x in sc_nodes]
    p = np.arange(sc_nodes.shape[1])[None] < np.asarray(k)[:, None]
    for s, idx in enumerate(attachment):
        p[s, list(idx)] = False
    return p


def probabilities(sd, C, X, E, actions, masks, batch=512, dtype=torch.float64):
    """softmax(forward(state) with -inf at the masked entries)[action] in `dtype`, and the unmasked logits"""
    _, logits = R.probabilities(sd, C, X, E, actions, batch=batch, dtype=dtype)
    masked = logits.masked_fill(torch.from_numpy(masks), float("-inf"))
    p = torch.softmax(masked, dim=1).gather(1, torch.from_numpy(actions).view(-1, 1)).view(-1)
    return p, logits


def score(sd, C, nodes, edges, ids, sc_nodes, segs, protect=None):
    """(likelihoods, offsets, nll, final, log_p_bound) of the conditional routes in fp64, in the form
    route_nll_reference.assert_within takes (masking a row only removes terms: the unmasked logits' bound holds)"""
    X, E, acts, offsets, sid, n_at = conditional_states(nodes, edges, ids, sc_nodes, segs)
    N, Ef = X.shape[1], E.shape[3]
    masks = state_masks(sid, n_at, sc_nodes, protect, N, Ef, C.len_f_add_per_node)
    assert not masks[np.arange(acts.shape[0]), acts].any(), "a conditional action is masked"
    p, logits = probabilities(sd, C, X, E, acts, masks)
    nll, final = R.reduce(p, offsets)
    return p, offsets, nll, final, R.log_p_bound(sd, C, X, E, acts, logits)
