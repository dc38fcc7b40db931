"""CPU: the restatement of the scaffold-first decoding order (tests/scaffold_match_reference.py) and the C-ABI of
`gib_scaffold_first`.

  1. the restated search equals brute force over every injective map (itertools.permutations) on small random
     molecules and scaffolds -- the same embedding, "none" included -- across the four action layouts, Ef = 1-4, with
     and without attachment points;
  2. every restated output begins with its scaffold (the conditional route plan's prefix rule), its route never
     disconnects, and with attachment points no conditional action is one the generator's rule forbids;
  3. the budget: a long path scaffold absent from a ladder of identical atoms runs out at a small budget and is
     "none" at a large one;
  4. the new symbols are bound, the ABI version is still 206, and the host-side refusals.
"""
import ctypes

import numpy as np
import pytest

from tests import preprocess_reference as P
from tests import scaffold_match_reference as SM
from tests import scaffold_oracle as SO
from tests import scaffold_route_reference as SR

LAYOUTS = {"gdb13": (5, 3, 0, 0), "imp_H": (5, 3, 4, 0), "chirality": (5, 3, 0, 3), "imp_H+chirality": (4, 3, 4, 3)}


def random_case(rng, layout, Ef, N=8, max_atoms=7):
    """a shuffled molecule and a scaffold cut from it (60 %) or from another molecule"""
    X, E = SM.random_molecule(rng, int(rng.integers(1, max_atoms + 1)), N, layout, Ef)
    src = (X, E) if rng.random() < 0.6 else SM.random_molecule(rng, int(rng.integers(1, max_atoms + 1)), N, layout, Ef)
    k = int(rng.integers(1, SM.n_atoms(src[0]) + 1))
    SX, SE = SM.cut_scaffold(*src, k, rng)
    X, E = SM.shuffle(X, E, rng)
    return X, E, SX, SE


@pytest.mark.parametrize("attachment", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("Ef", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_search_equals_brute_force(layout, Ef, attachment):
    rng = np.random.default_rng(hash((layout, Ef, attachment)) % 2**32)
    found = 0
    for _ in range(40):
        X, E, SX, SE = random_case(rng, LAYOUTS[layout], Ef)
        protect = rng.random(X.shape[0]) < 0.5 if attachment else None
        want = SM.brute_force(X, E, SX, SE, protect)
        res, phi = SM.search(X, E, SX, SE, protect)
        if want is None:
            assert res == "none"
        else:
            assert res == "found" and phi == want
            found += 1
    assert 5 <= found < 40          # both answers occur


def _scaffold_set(rng, layout, Ef, M=24, S=6, N=9):
    mols = [SM.random_molecule(rng, int(rng.integers(2, 9)), N, layout, Ef) for _ in range(M)]
    sc = [SM.cut_scaffold(*mols[int(rng.integers(0, M))], int(rng.integers(1, 5)), rng) for _ in range(S)]
    mols = [SM.shuffle(x, e, rng) for x, e in mols]
    nodes, edges = np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])
    sn, se = np.stack([s[0] for s in sc]), np.stack([s[1] for s in sc])
    rankings = np.full((M, N), -1, np.int32)
    for m in range(M):
        n = SM.n_atoms(nodes[m])
        rankings[m, :n] = rng.permutation(n)
    return nodes, edges, sn, se, rankings


@pytest.mark.parametrize("attachment", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_restated_output_is_a_scaffold_prefix(layout, attachment):
    rng = np.random.default_rng(7)
    L = LAYOUTS[layout]
    nodes, edges, sn, se, rankings = _scaffold_set(rng, L, 3)
    protect = None
    if attachment:
        k = [SM.n_atoms(x) for x in sn]
        protect = (np.arange(sn.shape[1])[None] < np.array(k)[:, None]) & (rng.random(sn.shape[:2]) < 0.5)
    on, oe, order, ids, status = SM.scaffold_first(nodes, edges, sn, se, rankings, protect)
    assert status == (0, SM.NO_MOLECULE)
    assert (ids >= 0).sum() >= 4
    segs = P.segments(*L)
    for m in range(nodes.shape[0]):
        n = SM.n_atoms(nodes[m])
        assert sorted(order[m, :n].tolist()) == list(range(n)) and (order[m, n:] == -1).all()
        X, E = SM.reorder(nodes[m], edges[m], order[m, :n])
        assert np.array_equal(X, on[m]) and np.array_equal(E, oe[m])
        s = int(ids[m])
        if s < 0:                                         # no embedding: the input as it is
            assert np.array_equal(order[m, :n], np.arange(n))
            continue
        P.route(on[m], oe[m], segs)                       # raises on a route that disconnects
        k = SM.n_atoms(sn[s])
        X, E = SR.prefix(on[m], oe[m], k)
        assert np.array_equal(X, sn[s]) and np.array_equal(E, se[s]), m
        # the first scaffold that embeds: no earlier one does
        for t in range(s):
            assert SM.brute_force(nodes[m], edges[m], sn[t], se[t], None if protect is None else protect[t]) is None
    if attachment:
        # every conditional action against the generator's rule (tests/scaffold_oracle.forbidden): slot 1 of an
        # oracle state decorating scaffold sid with the state's atom count
        N, Ef = nodes.shape[1], edges.shape[3]
        hit = ids >= 0                                    # the others keep their input order, which may disconnect
        _, _, acts, _, sid, n_at = SR.conditional_states(on[hit], oe[hit], ids[hit], sn, segs)
        A, CH, H, C = L
        state = SO.ScaffoldState(2, N, A, CH, Ef, H, C, sn, se)
        for a, s, n in zip(acts, sid, n_at):
            state.slot_ids[1], state.n_nodes[1] = s, n
            assert not SO.forbidden(state, 1, protect)[a], (a, s, n)
        assert len(acts) > 0


def test_ids_mode():
    rng = np.random.default_rng(3)
    nodes, edges, sn, se, rankings = _scaffold_set(rng, LAYOUTS["gdb13"], 2)
    ids_in = rng.integers(-1, sn.shape[0], nodes.shape[0])
    _, _, _, ids, status = SM.scaffold_first(nodes, edges, sn, se, rankings, ids=ids_in)
    assert status[0] == 0
    for m in range(nodes.shape[0]):
        s = int(ids_in[m])
        want = s if s >= 0 and SM.brute_force(nodes[m], edges[m], sn[s], se[s]) is not None else -1
        assert ids[m] == want


def ladder(rungs, N, Ef=1):
    """a ladder graph of 2 * rungs identical atoms (type 0), padded to N"""
    F = 8
    X = np.zeros((N, F), np.int8)
    E = np.zeros((N, N, Ef), np.int8)
    n = 2 * rungs
    X[:n, 0] = 1
    X[:n, 5] = 1
    for r in range(rungs):
        a, b = 2 * r, 2 * r + 1
        E[a, b, 0] = E[b, a, 0] = 1
        if r + 1 < rungs:
            E[a, a + 2, 0] = E[a + 2, a, 0] = 1
            E[b, b + 2, 0] = E[b + 2, b, 0] = 1
    return X, E


def path_scaffold(length, N, Ef=1):
    """a path of `length` type-0 atoms ending in a type-1 atom: absent from a ladder of type-0 atoms, found only at the
    last depth"""
    X = np.zeros((N, 8), np.int8)
    E = np.zeros((N, N, Ef), np.int8)
    X[:length, 0] = 1
    X[length - 1, 0], X[length - 1, 1] = 0, 1
    X[:length, 5] = 1
    for a in range(length - 1):
        E[a, a + 1, 0] = E[a + 1, a, 0] = 1
    return X, E


def search_nodes(X, E, SX, SE, protect=None):
    """the smallest budget with which the search completes: its number of search-tree nodes (assignments)"""
    lo, hi = 1, 1 << 20
    assert SM.search(X, E, SX, SE, protect, budget=hi)[0] != "budget"
    while lo < hi:
        mid = (lo + hi) // 2
        if SM.search(X, E, SX, SE, protect, budget=mid)[0] == "budget":
            lo = mid + 1
        else:
            hi = mid
    return lo


def test_budget():
    X, E = ladder(12, 24)
    SX, SE = path_scaffold(14, 24)
    assert SM.search(X, E, SX, SE, budget=200) == ("budget", None)
    assert SM.search(X, E, SX, SE) == ("none", None)
    # the node count: a budget of exactly the search's nodes is enough, one less is not
    count = search_nodes(X, E, SX, SE)
    assert count > 200
    assert SM.search(X, E, SX, SE, budget=count) == ("none", None)
    assert SM.search(X, E, SX, SE, budget=count - 1) == ("budget", None)
    # a search that finds its embedding: the leaf is the count-th node
    SX2, SE2 = path_scaffold(14, 24)
    SX2[13] = SX2[12]                                       # all type 0: the path embeds
    count = search_nodes(X, E, SX2, SE2)
    assert SM.search(X, E, SX2, SE2, budget=count)[0] == "found"
    assert SM.search(X, E, SX2, SE2, budget=count - 1) == ("budget", None)


def test_symbols_and_abi():
    from graphinvent_b200 import _lib
    assert _lib.ABI_VERSION == 206 and _lib.lib.gib_version() == 206
    for name in ("gib_scaffold_first", "gib_scaffold_first_ws_bytes"):
        assert name in _lib.exported_symbols()
        assert getattr(_lib.lib, name) is not None
    assert _lib.PP_MATCH_BUDGET == 32


def test_host_refusals():
    from graphinvent_b200._lib import PPDims, Scaffolds, lib
    d = PPDims(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert lib.gib_scaffold_first_ws_bytes(ctypes.byref(d), 10, 4) > 0
    assert lib.gib_scaffold_first_ws_bytes(ctypes.byref(d), 0, 4) == 0
    assert lib.gib_scaffold_first_ws_bytes(ctypes.byref(d), 10, 0) == 0
    fake = ctypes.c_void_p(256)          # never dereferenced: every refusal below returns before a launch

    def call(dims, sc, budget=100, n=4):
        return lib.gib_scaffold_first(ctypes.byref(dims), fake, fake, n, ctypes.byref(sc), None, 1, 0, 0, 0, fake,
                                      budget, fake, fake, fake, fake, fake, fake, None)

    sc = Scaffolds(nodes=256, edges=256, n_atoms=256, protect=None, S=2)
    assert call(d, sc, budget=0) < 0 and b"budget" in lib.gib_last_error()
    assert call(d, sc, n=0) < 0
    assert call(d, Scaffolds(nodes=256, edges=256, n_atoms=256, S=0)) < 0
    wide = PPDims(N=10, F=8, Ef=300, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert call(wide, sc) < 0 and b"Ef * N * ceil(N / 32) <= 2048" in lib.gib_last_error()
    d128 = PPDims(N=128, F=8, Ef=1, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert call(d128, Scaffolds(nodes=256, edges=256, n_atoms=256, protect=256, S=2)) < 0
    assert b"N <= 127" in lib.gib_last_error()
