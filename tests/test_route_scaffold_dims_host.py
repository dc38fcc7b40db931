"""CPU: the N <= 127 limit of attachment points, refused by name before any launch (gib_route_plan_scaffold, both mask
entry points, generation.ScaffoldTable), and the molecule builders of tests/test_gpu_route_scaffold_dims.py: each a
valid decoding order whose restated route has n_bonds + 2 states."""
import ctypes

import numpy as np
import pytest

from tests import preprocess_reference as P
from tests.test_gpu_route_scaffold_dims import (GRID, LAYOUTS, chain, complete, molecule, molecule_set, segs_of, star,
                                                tree_with_rings)


def _dims(N, Ef=1, layout="gdb13"):
    from graphinvent_b200._lib import PPDims
    A, Fc, H, C = LAYOUTS[layout]
    return PPDims(N=N, F=A + Fc + H + C, Ef=Ef, n_atom_types=A, n_formal_charge=Fc, n_imp_H=H, n_chirality=C,
                  batch_size=64)


@pytest.mark.parametrize("N", [128, 181])
def test_plan_refuses_attachment_points_beyond_127(N):
    """protect != null at N > 127 is refused with the limit in the message; without protect words the same call gets
    past that check (here it stops at n_molecules = 0, which comes first only when the table has no protect words)"""
    from graphinvent_b200._lib import Scaffolds, lib
    d = _dims(N)
    p = ctypes.c_void_p(64)
    with_protect = Scaffolds(nodes=64, edges=64, n_atoms=64, protect=64, S=2)
    rc = lib.gib_route_plan_scaffold(ctypes.byref(d), p, p, 5, 10, ctypes.byref(with_protect), p, p, p, p, None)
    err = lib.gib_last_error()
    assert rc < 0 and b"gib_route_plan_scaffold" in err and b"N <= 127" in err and f"N={N}".encode() in err, err
    free = Scaffolds(nodes=64, edges=64, n_atoms=64, S=2)
    rc = lib.gib_route_plan_scaffold(ctypes.byref(d), p, p, 0, 10, ctypes.byref(free), p, p, p, p, None)
    assert rc < 0 and b"n_molecules" in lib.gib_last_error()


@pytest.mark.parametrize("N", [128, 181])
def test_masks_refuse_n_beyond_127(N):
    from graphinvent_b200._lib import Scaffolds, lib
    p = ctypes.c_void_p(64)
    sc = ctypes.byref(Scaffolds(nodes=64, edges=64, n_atoms=64, protect=64, S=2))
    apd = N * (5 * 3 * 1 + 1) + 1
    assert lib.gib_route_mask_logits(4, N, 1, apd, sc, p, p, p, None) < 0
    assert b"gib_route_mask_logits" in lib.gib_last_error()
    assert lib.gib_generation_mask_logits(4, N, 1, apd, sc, p, p, None, None, None, p, None) < 0
    assert b"gib_generation_mask_logits" in lib.gib_last_error()


@pytest.mark.parametrize("N", [128, 129, 181])
def test_scaffold_table_names_the_limit(N):
    """attachment points at N > 127, as index lists or as a bool array: a ValueError naming N <= 127 (not a numpy
    broadcast error, nor a C error at the first conditional score)"""
    from graphinvent_b200.generation import ScaffoldTable, scaffold_table
    lay = LAYOUTS["gdb13"]
    rng = np.random.default_rng(N)
    x, e = molecule(40, N, segs_of("gdb13"), 1, chain(40, 1, rng), rng)
    sn, se = x[None], e[None]
    for attach in ([[0, 39]], np.ones((1, N), bool)):
        with pytest.raises(ValueError, match="N <= 127") as err:
            ScaffoldTable(sn, se, attach, N, 8, 1, lay, "cpu")
        assert f"N = {N}" in str(err.value)
        with pytest.raises(ValueError, match="N <= 127"):
            scaffold_table((sn, se), attach, N, 8, 1, lay, "cpu")


@pytest.mark.parametrize("N,Ef,layout", sorted({g[:3] for g in GRID}))
def test_builders_make_valid_decoding_orders(N, Ef, layout):
    """every atom i >= 1 bonds to an earlier atom, bonds are symmetric single-type, and the restated route has
    n_bonds + 2 states ending in the empty graph"""
    nodes, edges = molecule_set(min(N, 64), segs_of(layout), Ef, seed=N)
    rng = np.random.default_rng(0)
    n = min(N, 20)
    extra = [molecule(n, N, segs_of(layout), Ef, b(n, Ef, rng), rng) for b in (chain, star, complete, tree_with_rings)]
    mols = list(zip(nodes, edges)) + extra
    for x, e in mols:
        k = P.n_atoms(x)
        bonded = e.any(-1)
        assert (e == e.transpose(1, 0, 2)).all() and (e.sum(-1) <= 1).all() and not bonded.diagonal().any()
        assert all(bonded[i, :i].any() for i in range(1, k))
        st = P.route(x, e, segs_of(layout))
        assert len(st) == int(e.sum()) // 2 + 2 and not st[-1][0].any() and not st[-1][1].any()
    c = molecule(n, N, segs_of(layout), Ef, complete(n, Ef, rng), rng)[1]
    assert int(c.sum()) // 2 == n * (n - 1) // 2
