"""CPU: the restatement of the molecule set (tests/molecule_set_reference.py) and the host side of its C-ABI.

  1. identity against brute-force permutation isomorphism on random molecules of <= 7 atoms, over the four action
     layouts and Ef 1-4 (shuffled copies and near misses);
  2. ids invariant under atom shuffles; decalin / bicyclopentyl: one hash, two entries; the empty molecule;
  3. the uniqueness rule of util.write_molecules restated on lists, with a valid mask;
  4. gdb13_1K/train: 979 molecules, 979 entries, 979 distinct hashes;
  5. the new symbols, the size query and the host-side refusals.
"""
import ctypes
import os

import numpy as np
import pytest

from tests import molecule_set_reference as MS
from tests import murcko_reference as MR
from tests import scaffold_match_reference as SM
from tests.conftest import GOLDEN
from tests.test_murcko_host import GDB13, decalin_and_bicyclopentyl
from tests.test_scaffold_match_host import LAYOUTS


def _gdb13():
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]


def _near_miss(X, E, rng):
    """the molecule with one bond's type changed (or, with Ef = 1, one atom's first segment index changed)"""
    X, E = X.copy(), E.copy()
    n = SM.n_atoms(X)
    bonds = np.argwhere(np.triu(E[:n, :n].any(-1)))
    if E.shape[2] > 1 and len(bonds):
        a, b = bonds[rng.integers(len(bonds))]
        t = int(np.flatnonzero(E[a, b])[0])
        E[a, b] = E[b, a] = 0
        E[a, b, (t + 1) % E.shape[2]] = E[b, a, (t + 1) % E.shape[2]] = 1
    else:
        a = int(rng.integers(n))
        t = int(np.flatnonzero(X[a])[0])
        X[a, t] = 0
        X[a, 1 - t if t < 2 else 0] = 1
    return X, E


@pytest.mark.parametrize("Ef", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_identity_is_isomorphism(layout, Ef):
    rng = np.random.default_rng(100 * list(LAYOUTS).index(layout) + Ef)
    mols = []
    for _ in range(14):
        X, E = SM.random_molecule(rng, int(rng.integers(1, 8)), 8, LAYOUTS[layout], Ef, n_types=2, extra_bonds=0.6)
        mols.append((X, E))
        mols.append(SM.shuffle(X, E, rng))
        mols.append(SM.shuffle(*_near_miss(X, E, rng), rng))
    order = rng.permutation(len(mols))
    mols = [mols[i] for i in order]
    s = MS.MoleculeSet()
    ids, new, first = s.add(np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols]))
    for i in range(len(mols)):
        for j in range(i):
            assert (ids[i] == ids[j]) == MS.brute_isomorphic(*mols[i], *mols[j]), (i, j)
    assert (new == (ids >= 0)).all() and first.sum() == len(s)
    assert (np.asarray(s.counts) == np.bincount(ids, minlength=len(s))).all()
    for X, E in zip(s.nodes, s.edges):                      # canonical: every prefix connected
        k = SM.n_atoms(X)
        assert all(E[i, :i].any() for i in range(1, k))


def test_shuffle_invariance_and_collision():
    rng = np.random.default_rng(7)
    nodes, edges = _gdb13()
    nodes, edges = nodes[:150], edges[:150]
    a = MS.MoleculeSet()
    ids, _, _ = a.add(nodes, edges)
    shuf = [SM.shuffle(x, e, rng) for x, e in zip(nodes, edges)]
    ids2, new2, first2 = a.find(np.stack([s[0] for s in shuf]), np.stack([s[1] for s in shuf]))
    assert np.array_equal(ids, ids2) and not new2.any() and first2.all()
    (dX, dE), (bX, bE) = decalin_and_bicyclopentyl()
    assert MR.wl_hash(*MS.canonical(dX, dE)) == MR.wl_hash(*MS.canonical(bX, bE))
    s = MS.MoleculeSet()
    ids, new, first = s.add(np.stack([dX, bX, SM.shuffle(dX, dE, rng)[0]]),
                            np.stack([dE, bE, SM.shuffle(dX, dE, np.random.default_rng(7))[1]]))
    assert len(s) == 2 and ids[:2].tolist() == [0, 1] and s.hash[0] == s.hash[1]


def test_empty_molecule_is_one_entry():
    (dX, dE), _ = decalin_and_bicyclopentyl()
    z = np.zeros_like(dX), np.zeros_like(dE)
    s = MS.MoleculeSet()
    ids, new, first = s.add(np.stack([z[0], dX, z[0]]), np.stack([z[1], dE, z[1]]))
    assert ids.tolist() == [0, 1, 0] and first.tolist() == [True, True, False] and s.counts == [2, 1]


def test_uniqueness_rule_with_valid():
    rng = np.random.default_rng(3)
    nodes, edges = _gdb13()
    pick = rng.integers(0, 40, 120)                         # many repeats
    X, E = nodes[pick], edges[pick]
    valid = rng.random(120) < 0.7
    s = MS.MoleculeSet()
    ids, new, first = s.add(X, E, valid)
    got = np.where(valid, first, True).astype(np.float32)
    want = MS.write_molecules_uniqueness(pick.tolist(), valid.tolist())
    assert np.array_equal(got, want)
    assert (ids[~valid] == -1).all() and not new[~valid].any() and not first[~valid].any()


def test_gdb13_all_distinct():
    nodes, edges = _gdb13()
    s = MS.MoleculeSet()
    ids, new, first = s.add(nodes, edges)
    assert len(s) == nodes.shape[0] == 979 and ids.tolist() == list(range(979)) and new.all() and first.all()
    assert len(set(s.hash)) == 979


def test_symbols_and_size_query():
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import exported_symbols, lib
    assert {"gib_molset_bytes", "gib_molset_slots", "gib_molset_init", "gib_molset_ws_bytes", "gib_molset_identify",
            "gib_molset_from_float"} <= set(exported_symbols())
    d = PP._pp_dims(13, 8, 3, GDB13)
    per_entry = 13 * 8 + 13 * 13 * 3 + 8 + 4 + 4 + 8 + 4        # bytes, hash, atoms, bonds, count, next
    for C in (1, 1000, 1 << 20):
        slots = lib.gib_molset_slots(C)
        assert slots >= 2 * C and slots & (slots - 1) == 0 and slots < 4 * C + 2
        assert lib.gib_molset_bytes(ctypes.byref(d), C) == per_entry * C + 12 * slots + 4
    assert lib.gib_molset_bytes(ctypes.byref(d), 0) == 0 and lib.gib_molset_slots(0) < 0
    assert lib.gib_molset_ws_bytes(ctypes.byref(d), 1000) > 0 and lib.gib_molset_ws_bytes(ctypes.byref(d), 0) == 0
    big = PP.PPDims(N=182, F=8, Ef=1, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert lib.gib_molset_bytes(ctypes.byref(big), 10) == 0 and b"N=182" in lib.gib_last_error()
    wide = PP.PPDims(N=4, F=8, Ef=600, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=1)
    assert lib.gib_molset_ws_bytes(ctypes.byref(wide), 10) == 0 and b"2048" in lib.gib_last_error()


def test_python_refusals_before_the_device():
    from graphinvent_b200.molecules import MoleculeSet
    with pytest.raises(ValueError, match="capacity"):
        MoleculeSet(13, 8, 3, 0, layout=GDB13)
    with pytest.raises(ValueError, match="budget"):
        MoleculeSet(13, 8, 3, 10, layout=GDB13, budget=0)
    with pytest.raises(ValueError, match="N=182"):
        MoleculeSet(182, 8, 1, 10, layout=GDB13)
