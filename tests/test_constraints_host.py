"""CPU: the constraint rule restated in tests/constraints_reference.py -- hand-worked states for every field and the
dead end, the route independence of the maxima and of the ring-size bound (girth) by brute force over random build
orders -- and the refusals and name resolution of `generation.Constraints` and `gib_constraints_set`."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest

from tests import action_mask_reference as AM
from tests import constraints_reference as R

GDB13 = namedtuple("C", "atom_types formal_charge n_edge_features")(["C", "N", "O", "S", "Cl"], [-1, 0, 1], 3)
N, A, CH, Ef = 13, 5, 3, 3
APD = N * (A * CH * Ef + Ef) + 1


def _table(**fields):
    v = R.off_values(A, CH, Ef)
    t = R.table_dict(v, A, CH, Ef)
    for k, x in fields.items():
        if isinstance(t[k], np.ndarray):
            t[k] = np.array(x, np.int64)
        else:
            t[k] = x
    return t


def _state(atoms, bonds):
    """nodes / edges of a gdb13 state: atoms = [(type, charge index)], bonds = [(i, j, type)]"""
    nodes = np.zeros((N, A + CH), np.int8)
    edges = np.zeros((N, N, Ef), np.int8)
    for i, (t, c) in enumerate(atoms):
        nodes[i, t] = nodes[i, A + c] = 1
    for i, j, e in bonds:
        edges[i, j, e] = edges[j, i, e] = 1
    return nodes, edges, len(atoms)


def _idx(kind, bond_to=0, atom=0, charge=1, btype=0):
    if kind == "add":
        return ((bond_to * A + atom) * CH + charge) * Ef + btype
    if kind == "conn":
        return N * A * CH * Ef + bond_to * Ef + btype
    return APD - 1


CHAIN = _state([(0, 1)] * 5, [(0, 1, 0), (1, 2, 0), (2, 3, 0), (3, 4, 0)])


def test_off_masks_only_what_the_structure_masks():
    nodes, edges, n = CHAIN
    assert (R.mask(_table(), nodes, edges, n, N, A, CH, 0, 0, Ef) == AM.structure(n, edges, N, A, CH, 0, 0, Ef)).all()


def test_max_atoms_type_charge_and_bond():
    nodes, edges, n = CHAIN
    f = R.mask(_table(max_atoms=5), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[:N * A * CH * Ef].all() and not f[_idx("conn", 0)]
    f = R.mask(_table(max_type=[5, -1, -1, -1, -1]), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[_idx("add", 2, atom=0)] and not f[_idx("add", 2, atom=1)]
    f = R.mask(_table(max_charge=[-1, -1, 0]), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[_idx("add", 2, charge=2)] and not f[_idx("add", 2, charge=1)]
    f = R.mask(_table(max_bond=[4, -1, -1]), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[_idx("add", 2, btype=0)] and f[_idx("conn", 0, btype=0)] and not f[_idx("conn", 0, btype=1)]
    empty = _state([], [])
    f = R.mask(_table(max_bond=[0, 0, 0]), *empty, N, A, CH, 0, 0, Ef)
    assert not f[_idx("add", 0, btype=0)]                            # the first add has no bond


def test_rings_and_min_ring_size():
    nodes, edges, n = CHAIN                                          # a path 0-1-2-3-4, the newest atom is 4
    f = R.mask(_table(max_rings=0), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[_idx("conn", 0)] and not f[_idx("add", 4)]
    f = R.mask(_table(min_ring_size=5), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert not f[_idx("conn", 0)]                                    # closes a 5-ring
    assert f[_idx("conn", 1)] and f[_idx("conn", 2)]                 # a 4-ring, a 3-ring
    f = R.mask(_table(min_ring_size=6), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[_idx("conn", 0)]


def test_minima_mask_terminate_unless_nothing_else_survives():
    nodes, edges, n = CHAIN
    assert R.mask(_table(min_atoms=6), nodes, edges, n, N, A, CH, 0, 0, Ef)[-1]
    assert R.mask(_table(min_type=[0, 1, 0, 0, 0]), nodes, edges, n, N, A, CH, 0, 0, Ef)[-1]
    assert R.mask(_table(min_rings=1), nodes, edges, n, N, A, CH, 0, 0, Ef)[-1]
    assert not R.mask(_table(min_atoms=5), nodes, edges, n, N, A, CH, 0, 0, Ef)[-1]
    # the dead end: a saturated carbon 3-ring (double bonds) under min_atoms with the valence rule
    V = np.full((A, CH), 4)
    ring = _state([(0, 1)] * 3, [(0, 1, 1), (1, 2, 1), (0, 2, 1)])
    f = R.mask(_table(min_atoms=6), *ring, N, A, CH, 0, 0, Ef, V, (2, 4, 6), ())
    assert f[:-1].all() and not f[-1]
    assert R.check(_table(min_atoms=6), *ring, N, A, CH, 0, 0, Ef, V, (2, 4, 6), ()) == R.DEAD_END
    assert R.check(_table(min_atoms=6), *ring, N, A, CH, 0, 0, Ef) == R.UNDER_MIN   # structure alone: adds survive
    # maxima make dead ends too: max_atoms = 5 and every connect closing a ring under 6 atoms
    f = R.mask(_table(min_rings=1, max_atoms=5, min_ring_size=6), nodes, edges, n, N, A, CH, 0, 0, Ef)
    assert f[:-1].all() and not f[-1]


def _random_molecule(rng, n, p_ring):
    """a connected graph of n atoms: a random tree plus extra bonds"""
    adj = np.zeros((n, n), bool)
    for i in range(1, n):
        j = rng.integers(0, i)
        adj[i, j] = adj[j, i] = True
    for i in range(n):
        for j in range(i + 1, n):
            if not adj[i, j] and rng.random() < p_ring:
                adj[i, j] = adj[j, i] = True
    return adj


def _route(adj, rng):
    """a random build order of a connected graph the generator could follow: each new atom bonded to an existing one,
    then any subset of the remaining bonds to it as connects (as a list of ('add' | 'conn', i, j) in order)"""
    n = adj.shape[0]
    order = [int(rng.integers(0, n))]
    while len(order) < n:
        cand = [v for v in range(n) if v not in order and adj[v, order].any()]
        order.append(int(rng.choice(cand)))
    pos = {v: k for k, v in enumerate(order)}
    steps = []
    for k, v in enumerate(order[1:], 1):
        back = [u for u in order[:k] if adj[v, u]]
        rng.shuffle(back)
        steps.append(("add", back[0], v))
        steps += [("conn", u, v) for u in back[1:]]
    return steps, pos


def test_ring_size_bound_is_the_girth_whatever_the_route():
    """brute force over random small graphs and random build orders: the smallest ring any connect of the route
    closes (BFS in the graph so far) equals the girth of the finished graph"""
    rng = np.random.default_rng(11)
    seen = 0
    for _ in range(300):
        n = int(rng.integers(3, 10))
        adj = _random_molecule(rng, n, 0.25)
        g = R.girth(adj)
        for _ in range(4):
            steps, _ = _route(adj, rng)
            cur = np.zeros_like(adj)
            smallest = None
            for kind, u, v in steps:
                if kind == "conn":
                    d = R.bfs(cur, v)[u]
                    assert d is not None
                    smallest = d + 1 if smallest is None else min(smallest, d + 1)
                cur[u, v] = cur[v, u] = True
            assert smallest == g
            seen += g is not None
    assert seen > 100


def test_maxima_are_route_independent():
    """over random build orders: a route takes a forbidden add / connect exactly when the finished molecule is over
    the maximum (counts, bond types and the cycle rank grow by one per action)"""
    rng = np.random.default_rng(12)
    for _ in range(200):
        n = int(rng.integers(1, 9))
        adj = _random_molecule(rng, n, 0.2)
        types = rng.integers(0, A, n)
        btype = {(min(i, j), max(i, j)): int(rng.integers(0, Ef)) for i in range(n) for j in range(i) if adj[i, j]}
        mx_t, mx_b, mx_r = int(rng.integers(0, 4)), int(rng.integers(0, 5)), int(rng.integers(0, 3))
        steps, _ = _route(adj, rng)
        first = steps[0][1] if steps else 0
        cnt_t = {int(types[first]): 1}                               # the first add, into the empty graph
        cnt_b, rank, refused = {}, 0, mx_t == 0
        for kind, u, v in steps:
            e = btype[(min(u, v), max(u, v))]
            if kind == "add":
                refused |= cnt_t.get(int(types[v]), 0) >= mx_t or cnt_b.get(e, 0) >= mx_b
                cnt_t[int(types[v])] = cnt_t.get(int(types[v]), 0) + 1
            else:
                refused |= cnt_b.get(e, 0) >= mx_b or rank >= mx_r
                rank += 1
            cnt_b[e] = cnt_b.get(e, 0) + 1
        over = (max(cnt_t.values()) > mx_t or (cnt_b and max(cnt_b.values()) > mx_b)
                or int(adj.sum()) // 2 - n + 1 > mx_r)
        assert refused == bool(over)


# ---- the value object -------------------------------------------------------------------------------------------
def test_names_resolve_through_the_constants_and_indices_without():
    from graphinvent_b200.generation import Constraints
    c = Constraints(atoms=(3, 12), atom_types={"N": (1, None), "S": (0, 0)}, charges={1: 0}, bonds={"triple": 0},
                    rings=(0, 2), min_ring_size=5, constants=GDB13)
    v = c.values((A, CH, 0, 0), N, Ef)
    t = R.table_dict(v, A, CH, Ef)
    assert (t["min_atoms"], t["max_atoms"], t["min_rings"], t["max_rings"], t["min_ring_size"]) == (3, 12, 0, 2, 5)
    assert t["min_type"].tolist() == [0, 1, 0, 0, 0] and t["max_type"].tolist() == [-1, -1, -1, 0, -1]
    assert t["max_charge"].tolist() == [-1, -1, 0] and t["max_bond"].tolist() == [-1, -1, 0]
    by_index = Constraints(atoms=(3, 12), atom_types={1: (1, None), 3: (0, 0)}, charges={2: 0}, bonds={2: 0},
                           rings=(0, 2), min_ring_size=5)
    assert (by_index.values((A, CH, 0, 0), N, Ef) == v).all()
    assert Constraints().off and not c.off
    assert Constraints(atoms=(None, None), atom_types={"C": (None, None)}).off


@pytest.mark.parametrize("kw,match", [
    (dict(atoms=(5, 4)), "over the maximum"), (dict(atoms=(-1, 4)), "non-negative"), (dict(atoms=5), "pair"),
    (dict(rings=(2, 1)), "over the maximum"), (dict(min_ring_size=2), "min_ring_size"),
    (dict(min_ring_size=1), "min_ring_size"), (dict(min_ring_size=-3), "min_ring_size"),
    (dict(charges={0: (1, 2)}), "maximum only"), (dict(bonds={0: -1}), "non-negative"),
    (dict(atom_types={"C": (3, 1)}), "over the maximum"), (dict(atom_types={"C": 2.5}), "pair")])
def test_value_object_refusals(kw, match):
    from graphinvent_b200.generation import Constraints
    with pytest.raises(ValueError, match=match):
        Constraints(**kw)


@pytest.mark.parametrize("kw,match", [
    (dict(atoms=(0, 14)), "over max_n_nodes"), (dict(atoms=(14, None)), "over max_n_nodes"),
    (dict(atoms=(None, 3), atom_types={"C": (2, None), "N": (2, None)}), "add up"),
    (dict(atom_types={"Xe": (1, None)}), "unknown atom type"), (dict(atom_types={7: (1, None)}), "outside"),
    (dict(bonds={"QUADRUPLE": 0}), "unknown bond type"), (dict(charges={2: 0}), "unknown formal charge")])
def test_layout_refusals(kw, match):
    from graphinvent_b200.generation import Constraints
    with pytest.raises(ValueError, match=match):
        Constraints(**kw, constants=GDB13).values((A, CH, 0, 0), N, Ef)


def test_names_need_constants():
    from graphinvent_b200.generation import Constraints
    with pytest.raises(ValueError, match="names need constants"):
        Constraints(atom_types={"N": (1, None)}).values((A, CH, 0, 0), N, Ef)


def test_setter_refusals_need_no_device():
    """gib_constraints_set refuses before any CUDA call"""
    from graphinvent_b200._lib import lib
    dummy = ctypes.c_void_p(16)                                      # never dereferenced: refused first
    for edit in ({1: 14}, {0: 5, 1: 4}, {4: 2}, {4: 1}, {2: 3, 3: 2}, {8: -1}, {8 + A: -2}, {1: -2},
                 {8: 7, 9: 7, 1: 12}, {0: 14}, {8 + 2 * A + CH: -5}):
        v = R.off_values(A, CH, Ef)
        for k, x in edit.items():
            v[k] = x
        assert lib.gib_constraints_set(dummy, v.ctypes.data_as(ctypes.c_void_p), N, A, CH, Ef, None) == -1, edit
        assert b"refused" in lib.gib_last_error()
    v = R.off_values(A, CH, Ef)
    assert lib.gib_constraints_set(None, v.ctypes.data_as(ctypes.c_void_p), N, A, CH, Ef, None) == -1
    assert lib.gib_constraints_set(dummy, None, N, A, CH, Ef, None) == -1
    assert lib.gib_constraints_set(dummy, v.ctypes.data_as(ctypes.c_void_p), 128, A, CH, Ef, None) == -1
    assert lib.gib_constraints_ints(A, CH, Ef) == 8 + 2 * A + CH + Ef and lib.gib_constraints_ints(0, CH, Ef) == 0


def test_constraints_without_an_action_mask_bring_the_structural_rule():
    from graphinvent_b200.generation import Constraints, make_action_mask
    assert make_action_mask(None, None, GDB13, (A, CH, 0, 0), N, A + CH, Ef, APD, "cpu") is None
    with pytest.raises(TypeError):
        make_action_mask(None, None, GDB13, (A, CH, 0, 0), N, A + CH, Ef, APD, "cpu", constraints={"atoms": (1, 2)})
