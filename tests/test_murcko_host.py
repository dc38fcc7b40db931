"""CPU: the restatement of the Murcko scaffolds (tests/murcko_reference.py) and the C-ABI of `gib_murcko`.

  1. hand-worked molecules in the gdb13 layout with their kept atoms written out (ring, exocyclic double bonds kept
     one level deep, linkers, spiro and fused systems, no ring), an explicit-H molecule, and bond types other than
     double (aromatic, Ef = 1) that the double-bond clause does not keep;
  2. RDKit's form (ring atoms and shortest paths between them) and the 2-core form agree on gdb13_1K/train and on
     random ring-rich molecules, and the canonical order's every prefix is connected;
  3. the hash: decalin and bicyclopentyl collide and are not isomorphic; a molecule and an atom-shuffled copy hash
     equal; the restated dedup gives the same ids for shuffled molecules and for calls chained with `known`;
  4. the new symbols are bound and the host-side limits refuse.
"""
import ctypes
import os

import numpy as np
import pytest

from tests import murcko_reference as MR
from tests import scaffold_match_reference as SM
from tests.conftest import GOLDEN

GDB13 = (5, 3, 0, 0)          # C N O S Cl | charge -1 0 +1
EXPLICIT_H = (6, 3, 0, 0)     # C N O S Cl H | charge
ATOM = {"C": 0, "N": 1, "O": 2, "H": 5}
SINGLE, DOUBLE, TRIPLE, AROMATIC = 0, 1, 2, 3


def mol(atoms, bonds, N=16, Ef=3, n_types=5):
    """int8 (nodes [N, n_types + 3], edges [N, N, Ef]): uncharged atoms `atoms` (a string of C N O H), bonds
    (a, b, type)"""
    X = np.zeros((N, n_types + 3), np.int8)
    E = np.zeros((N, N, Ef), np.int8)
    for i, a in enumerate(atoms):
        X[i, ATOM[a]] = 1
        X[i, n_types + 1] = 1
    for a, b, t in bonds:
        E[a, b, t] = E[b, a, t] = 1
    return X, E


def ring(atoms, t=SINGLE):
    return [(atoms[i], atoms[(i + 1) % len(atoms)], t) for i in range(len(atoms))]


HAND = {
    # CC1CCCCC1: the methyl goes
    "methylcyclohexane": (mol("CCCCCCC", [(0, 1, SINGLE)] + ring([1, 2, 3, 4, 5, 6])), {1, 2, 3, 4, 5, 6}),
    # O=C1CCCCC1: the exocyclic double bond to a ring atom stays
    "cyclohexanone": (mol("OCCCCCC", [(0, 1, DOUBLE)] + ring([1, 2, 3, 4, 5, 6])), {0, 1, 2, 3, 4, 5, 6}),
    # CC(=O)C1CCCC1: the carbonyl carbon is not core, so it goes and its O with it
    "acetylcyclopentane": (mol("CCOCCCCC", [(0, 1, SINGLE), (1, 2, DOUBLE), (1, 3, SINGLE)] + ring([3, 4, 5, 6, 7])),
                           {3, 4, 5, 6, 7}),
    # C=C1CCCC1
    "methylenecyclopentane": (mol("CCCCCC", [(0, 1, DOUBLE)] + ring([1, 2, 3, 4, 5])), {0, 1, 2, 3, 4, 5}),
    # C1CC1C(C)C1CC1: the linker stays, its methyl goes
    "dicyclopropylethane": (mol("CCCCCCCC", ring([0, 1, 2]) + [(2, 3, SINGLE), (3, 4, SINGLE), (3, 5, SINGLE)]
                                + ring([5, 6, 7])), {0, 1, 2, 3, 5, 6, 7}),
    # CC1CC12CC2: spiro[2.2]pentane with a methyl
    "spiro": (mol("CCCCCC", [(0, 1, SINGLE)] + ring([1, 2, 3]) + ring([3, 4, 5])), {1, 2, 3, 4, 5}),
    # a fused 6-5 system with an OH on the five-ring and a ring C=O: OC1CC2CC(=O)CCC2C1 in another numbering
    "fused": (mol("OCCCCCCCCCO", [(0, 1, SINGLE)] + ring([2, 3, 4, 5, 6, 7]) + [(6, 8, SINGLE), (8, 9, SINGLE),
                                                                              (9, 1, SINGLE), (1, 7, SINGLE),
                                                                              (3, 10, DOUBLE)]),
              set(range(1, 11))),
    # CCO
    "ethanol": (mol("CCO", [(0, 1, SINGLE), (1, 2, SINGLE)]), set()),
    # C#CC1CC1: a triple bond out of the ring is not the double-bond clause
    "ethynylcyclopropane": (mol("CCCCC", [(0, 1, TRIPLE), (1, 2, SINGLE)] + ring([2, 3, 4])), {2, 3, 4}),
}


def _check_keep(X, E, want):
    got_core, got_rdkit = MR.keep_core(X, E), MR.keep_rdkit(X, E)
    assert set(np.flatnonzero(got_core).tolist()) == want
    assert np.array_equal(got_core, got_rdkit)


@pytest.mark.parametrize("name", list(HAND))
def test_hand_worked(name):
    (X, E), want = HAND[name]
    _check_keep(X, E, want)
    SX, SE, order, keep = MR.scaffold(X, E)
    assert sorted(order) == sorted(want)
    assert SM.n_atoms(SX) == len(want)
    if want:                                     # node rows byte for byte, every bond among the kept atoms
        o = np.array(order)
        assert np.array_equal(SX[:len(o)], X[o]) and np.array_equal(SE[:len(o), :len(o)], E[o][:, o])
        assert order[0] == min(want)


def test_explicit_h():
    """OC1CC1 with every hydrogen explicit: H atoms and the OH go like any substituent"""
    bonds = ring([0, 1, 2]) + [(0, 3, SINGLE), (3, 4, SINGLE), (0, 5, SINGLE)] + \
        [(1, 6, SINGLE), (1, 7, SINGLE), (2, 8, SINGLE), (2, 9, SINGLE)]
    X, E = mol("CCCOHHHHHH", bonds, n_types=6)
    _check_keep(X, E, {0, 1, 2})


def test_other_bond_types():
    """the clause is edge feature 1 only: an aromatic exocyclic bond (Ef = 4) is not kept; with Ef = 1 the double
    bond is not representable and the clause never applies"""
    X, E = mol("CCCC", [(0, 1, AROMATIC)] + ring([1, 2, 3]), Ef=4)
    _check_keep(X, E, {1, 2, 3})
    X, E = mol("OCCC", [(0, 1, DOUBLE)] + ring([1, 2, 3]), Ef=4)
    _check_keep(X, E, {0, 1, 2, 3})
    X1, E1 = mol("OCCC", [(0, 1, SINGLE)] + ring([1, 2, 3]), Ef=1)
    _check_keep(X1, E1, {1, 2, 3})


def _gdb13():
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]


def ring_rich(rng, M, N, layout, Ef, lo=3, hi=None):
    """random connected molecules with about as many extra bonds (rings) as 1/2 of their atoms, atoms shuffled"""
    hi = hi or N
    out = [SM.shuffle(*SM.random_molecule(rng, int(rng.integers(lo, hi + 1)), N, layout, Ef, n_types=2,
                                          extra_bonds=1.0), rng) for _ in range(M)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def _prefixes_connected(SE, k):
    bonded = SE[:k, :k].any(-1)
    return all(bonded[i, :i].any() for i in range(1, k))


def test_formulations_agree_gdb13():
    nodes, edges = _gdb13()
    rings = 0
    for X, E in zip(nodes, edges):
        core = MR.keep_core(X, E)
        assert np.array_equal(core, MR.keep_rdkit(X, E))
        SX, SE, order, _ = MR.scaffold(X, E, core)
        assert _prefixes_connected(SE, len(order))
        rings += core.any()
    assert 100 < rings < nodes.shape[0]


@pytest.mark.parametrize("Ef", [1, 2, 3, 4])
def test_formulations_agree_random(Ef):
    rng = np.random.default_rng(Ef)
    nodes, edges = ring_rich(rng, 60, 24, GDB13, Ef)
    doubles = 0
    for X, E in zip(nodes, edges):
        core = MR.keep_core(X, E)
        assert np.array_equal(core, MR.keep_rdkit(X, E))
        SX, SE, order, _ = MR.scaffold(X, E, core)
        assert _prefixes_connected(SE, len(order))
        doubles += Ef > 1 and bool(SE[:, :, 1].any())
    assert Ef == 1 or doubles > 0


def decalin_and_bicyclopentyl(N=16):
    decalin = mol("C" * 10, ring([0, 1, 2, 3, 4, 5]) + [(5, 6, SINGLE), (6, 7, SINGLE), (7, 8, SINGLE),
                                                         (8, 9, SINGLE), (9, 0, SINGLE)], N=N)
    bicyclopentyl = mol("C" * 10, ring([0, 1, 2, 3, 4]) + ring([5, 6, 7, 8, 9]) + [(0, 5, SINGLE)], N=N)
    return decalin, bicyclopentyl


def test_wl_collision():
    (dX, dE), (bX, bE) = decalin_and_bicyclopentyl()
    assert MR.wl_hash(dX, dE) == MR.wl_hash(bX, bE)
    assert SM.search(dX, dE, bX, bE)[0] == "none" and SM.search(bX, bE, dX, dE)[0] == "none"
    ids = MR.murcko(np.stack([dX, bX, dX]), np.stack([dE, bE, dE]))[1]
    assert ids.tolist() == [0, 1, 0]


def test_hash_ignores_atom_order():
    rng = np.random.default_rng(3)
    nodes, edges = ring_rich(rng, 20, 20, (5, 3, 4, 0), 3)
    for X, E in zip(nodes, edges):
        SX, SE, _, _ = MR.scaffold(X, E)
        X2, E2 = SM.shuffle(X, E, rng)
        SX2, SE2, _, _ = MR.scaffold(X2, E2)
        assert MR.wl_hash(SX, SE) == MR.wl_hash(SX2, SE2)


def test_restated_dedup_invariance_and_chaining():
    rng = np.random.default_rng(5)
    nodes, edges = _gdb13()
    nodes, edges = nodes[:200], edges[:200]
    table, ids, keep, status = MR.murcko(nodes, edges)
    assert status == (0, SM.NO_MOLECULE)
    shuf = [SM.shuffle(x, e, rng) for x, e in zip(nodes, edges)]
    _, ids2, _, _ = MR.murcko(np.stack([s[0] for s in shuf]), np.stack([s[1] for s in shuf]))
    assert np.array_equal(ids, ids2)
    first, ids_a, _, _ = MR.murcko(nodes[:77], edges[:77])
    whole, ids_b, _, _ = MR.murcko(nodes[77:], edges[77:], known=first)
    assert np.array_equal(np.concatenate([ids_a, ids_b]), ids)
    for u, v in zip(table, whole):
        assert np.array_equal(u, v)
    assert table[2].sum() == (ids >= 0).sum()


def test_symbols_and_limits():
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import exported_symbols, lib
    assert {"gib_murcko", "gib_murcko_ws_bytes"} <= set(exported_symbols())
    d = PP._pp_dims(38, 8, 3, GDB13)
    assert lib.gib_murcko_ws_bytes(ctypes.byref(d), 10, 4) > 0
    assert lib.gib_murcko_ws_bytes(ctypes.byref(d), 0, 4) == 0
    assert lib.gib_murcko_ws_bytes(ctypes.byref(d), 10, -1) == 0
    big = PP.PPDims(N=182, F=8, Ef=1, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert lib.gib_murcko_ws_bytes(ctypes.byref(big), 10, 0) == 0
    X, E = HAND["methylcyclohexane"][0]
    with pytest.raises(ValueError, match="budget"):
        PP.murcko_scaffolds(X[None], E[None], layout=GDB13, budget=0)
