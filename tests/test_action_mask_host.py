"""CPU: the action mask's rule (tests/action_mask_reference.py) against the unmodified reference's verdicts, the
valence table (`config.action_rule_table`) and the refusals of `gib_action_mask_logits` and `generation.ActionMask`."""
import ctypes
import os
from collections import namedtuple

import numpy as np
import pytest

from tests import action_mask_reference as R
from tests.conftest import ROOT

FIXTURE = os.path.join(ROOT, "tests", "golden", "action_mask_invalid.npz")


def _cases():
    z = np.load(FIXTURE)
    return z, [tuple(int(v) for v in c) for c in z["cases"]]


def test_structure_equals_the_reference_verdict_on_every_action():
    """every (state, action) pair of the fixture: the oracle's structural rule is the reference's get_invalid_actions,
    except adds into a full graph outside L0, which the reference cannot judge (it raises IndexError next)"""
    z, cases = _cases()
    n_checked = n_forbidden = n_deviation = 0
    layouts = set()
    for k, (N, A, CH, H, C, Ef) in enumerate(cases):
        layouts.add((H > 0, C > 0))
        per = A * CH * max(H, 1) * max(C, 1) * Ef
        for n, e, ref in zip(z[f"n_{k}"], z[f"edges_{k}"], z[f"invalid_{k}"]):
            got = R.structure(int(n), e, N, A, CH, H, C, Ef)
            assert got.shape == ref.shape
            skip = np.zeros_like(ref)
            if (H or C) and n == N:
                skip[:N * per] = True                       # the documented deviation
                assert got[:N * per].all()
                n_deviation += int((got[:N * per] != ref[:N * per]).sum())
            diff = np.flatnonzero((got != ref) & ~skip)
            assert diff.size == 0, f"case {k} n={int(n)}: indices {diff[:10]}"
            assert not got[-1]                              # terminate is never forbidden
            n_checked += int((~skip).sum())
            n_forbidden += int(got.sum())
    assert layouts == {(False, False), (True, False), (False, True), (True, True)}
    assert n_checked > 20000 and n_forbidden > 5000 and n_deviation > 0


def test_the_fixture_reaches_the_quirks():
    """the element-5 rule fires on bond types / chiralities at tiny N, and bonds exist to be refused"""
    z, cases = _cases()
    seen_e5 = seen_dup = seen_multi = False
    for k, (N, A, CH, H, C, Ef) in enumerate(cases):
        per = A * CH * max(H, 1) * max(C, 1) * Ef
        for n, e, ref in zip(z[f"n_{k}"], z[f"edges_{k}"], z[f"invalid_{k}"]):
            if (H or C) and 0 < n < N:
                kind, to, *_ = R.decode(ref.size, N, A, CH, H, C, Ef)
                ok_to = (kind == 0) & (to < n)
                seen_e5 |= bool(ref[:N * per][ok_to[:N * per]].any())
            seen_dup |= bool((e.sum(-1) == 1).any() and n > 1)
            seen_multi |= bool((e.sum(-1) > 1).any())
    assert seen_e5 and seen_dup and seen_multi


def test_valence_rule_on_hand_built_states():
    """carbon chain C-C=C in L0: the double-bonded end takes at most one more single bond; O caps at 2"""
    N, A, CH, H, C, Ef = 5, 5, 3, 0, 0, 3
    from graphinvent_b200.config import DEFAULT_MAX_VALENCE, action_rule_table
    Cst = namedtuple("C", "atom_types formal_charge")(["C", "N", "O", "S", "Cl"], [-1, 0, 1])
    V, order, imp = action_rule_table(A, CH, Ef, 0, None, Cst)
    assert V[0, 1] == DEFAULT_MAX_VALENCE[("C", 0)] == 4 and V[2, 1] == 2 and V[4, 0] == 0
    nodes = np.zeros((N, A + CH), np.int8)
    nodes[:3, 0] = 1
    nodes[:3, A + 1] = 1                                   # neutral carbons
    e = np.zeros((N, N, Ef), np.int8)
    e[0, 1, 0] = e[1, 0, 0] = 1
    e[1, 2, 1] = e[2, 1, 1] = 1
    f = R.forbidden(nodes, e, 3, N, A, CH, H, C, Ef, V, order, imp)
    per = A * CH * Ef
    add = lambda to, t, q, bt: to * per + (t * CH + q) * Ef + bt
    conn = lambda to, bt: N * per + to * Ef + bt
    # atom 2 holds a double bond (4 of 8 half-bond units): a second double reaches the limit, a triple passes it
    assert not f[add(2, 0, 1, 0)] and not f[add(2, 0, 1, 1)]
    assert f[add(2, 0, 1, 2)]
    assert f[add(1, 0, 1, 1)]                               # atom 1: 2 + 4 used, + 4 > 8
    assert not f[add(1, 0, 1, 0)]                           # + 2 = 8
    assert f[add(0, 4, 0, 0)]                               # Cl- has limit 0: no bond at all
    assert not f[add(0, 2, 1, 1)] and f[add(0, 2, 1, 2)]    # O=C allowed, O#C not
    assert not f[conn(0, 0)] and f[conn(0, 2)]              # ring closure 0-2 single ok, triple not
    assert f[conn(1, 0)]                                    # bond 1-2 exists
    assert not f[-1]
    empty = R.forbidden(nodes, np.zeros_like(e), 0, N, A, CH, H, C, Ef, V, order, imp)
    assert not empty[add(0, 4, 0, 0)]                       # a first atom has no bond: even Cl- may start


def test_valence_rule_counts_implicit_hydrogens():
    N, A, CH, H, C, Ef = 4, 1, 1, 4, 0, 3
    V = np.array([[4]])
    nodes = np.zeros((N, A + CH + H), np.int8)
    nodes[0, :2] = 1
    nodes[0, 2 + 3] = 1                                    # CH3
    e = np.zeros((N, N, Ef), np.int8)
    f = R.forbidden(nodes, e, 1, N, A, CH, H, C, Ef, V)
    per = A * CH * H * Ef
    add = lambda to, h, bt: to * per + h * Ef + bt
    assert not f[add(0, 3, 0)] and f[add(0, 3, 1)]          # CH3-CH3 ok, CH3=... no (atom 0: 6 + 4 > 8)
    assert not f[add(0, 2, 0)]
    first = R.forbidden(nodes, e, 0, N, A, CH, H, C, Ef, np.array([[2]]))
    assert first[add(0, 3, 0)] and not first[add(0, 2, 0)]  # a first atom with 3 H over a limit of 2


def test_valence_table_defaults_overrides_and_refusals():
    from graphinvent_b200.config import action_rule_table
    Cst = namedtuple("C", "atom_types formal_charge imp_H int_to_bondtype")
    c = Cst(["C", "N", "O", "S", "Cl"], [-1, 0, 1], [0, 1, 2, 3], {0: "SINGLE", 1: "DOUBLE", 2: "TRIPLE"})
    V, order, imp = action_rule_table(5, 3, 3, 4, None, c)
    assert V.dtype == np.int32 and V.shape == (5, 3)
    assert V.tolist() == [[3, 4, 3], [2, 3, 4], [1, 2, 3], [5, 6, 7], [0, 1, 2]]
    assert order.tolist() == [2, 4, 6] and imp.tolist() == [0, 1, 2, 3]
    V2, _, _ = action_rule_table(5, 3, 3, 4, {"S": 2, ("S", 1): 3, ("C", 0): 5}, c)
    assert V2[3].tolist() == [2, 2, 3] and V2[0].tolist() == [3, 5, 3]
    arr = np.arange(15).reshape(5, 3)
    assert action_rule_table(5, 3, 3, 0, arr, None)[0].tolist() == arr.tolist()
    assert action_rule_table(2, 1, 4, 0, [[1], [2]], None)[1].tolist() == [2, 4, 6, 3]      # default bond order
    assert action_rule_table(1, 1, 2, 3, [[4]], None)[2].tolist() == [0, 1, 2]             # index = count

    class BT:                                               # an rdkit-like BondType: name attribute
        def __init__(self, name):
            self.name = name
    c4 = c._replace(int_to_bondtype={0: BT("SINGLE"), 1: BT("AROMATIC"), 2: "rdkit.Chem.rdchem.BondType.DOUBLE"})
    assert action_rule_table(5, 3, 3, 0, None, c4)[1].tolist() == [2, 3, 4]
    with pytest.raises(ValueError, match=r"'Xe' with formal charge \+0"):
        action_rule_table(2, 1, 3, 0, None, c._replace(atom_types=["C", "Xe"], formal_charge=[0]))
    with pytest.raises(ValueError, match=r"'N' with formal charge \+2"):
        action_rule_table(1, 1, 3, 0, {"C": 4}, c._replace(atom_types=["N"], formal_charge=[2]))
    assert action_rule_table(1, 1, 3, 0, {"N": 5}, c._replace(atom_types=["N"], formal_charge=[2]))[0][0, 0] == 5
    with pytest.raises(ValueError, match="int array"):
        action_rule_table(5, 3, 3, 0, np.zeros((3, 5), np.int32), None)
    with pytest.raises(ValueError, match="needs constants"):
        action_rule_table(5, 3, 3, 0, None, None)
    with pytest.raises(ValueError, match="names 3 bond types"):
        action_rule_table(5, 3, 4, 0, None, c)
    with pytest.raises(ValueError, match="has no order"):
        action_rule_table(5, 3, 3, 0, None, c._replace(int_to_bondtype={0: "SINGLE", 1: "DATIVE", 2: "TRIPLE"}))
    with pytest.raises(ValueError, match="lists 4 counts"):
        action_rule_table(5, 3, 3, 3, None, c)


def test_action_mask_object_refusals():
    from graphinvent_b200.generation import ActionMask, make_action_mask
    assert make_action_mask(None, None, None, (5, 3, 0, 0), 13, 8, 3, 625, "cpu") is None
    with pytest.raises(ValueError, match="needs action_mask='valence'"):
        make_action_mask(None, {"C": 4}, None, (5, 3, 0, 0), 13, 8, 3, 625, "cpu")
    with pytest.raises(ValueError, match="'structure' or 'valence'"):
        ActionMask("valid", None, None, (5, 3, 0, 0), 13, 8, 3, 625, "cpu")
    with pytest.raises(ValueError, match="read by action_mask='valence' only"):
        ActionMask("structure", {"C": 4}, None, (5, 3, 0, 0), 13, 8, 3, 625, "cpu")
    with pytest.raises(ValueError, match="N <= 127"):
        ActionMask("structure", None, None, (1, 1, 0, 0), 128, 2, 1, 128 * 2 + 1, "cpu")
    m = ActionMask("valence", np.full((5, 3), 4), None, (5, 3, 0, 0), 13, 8, 3, 625, "cpu")
    assert m.table.tolist() == [4] * 15 + [2, 4, 6] and m.code == 2


def test_abi_refuses_bad_arguments():
    from graphinvent_b200._lib import Scaffolds, lib
    assert hasattr(lib, "gib_action_mask_logits")
    fake = ctypes.c_void_p(1 << 20)       # never dereferenced: every call below is refused before any launch

    def call(B=4, N=13, F=8, Ef=3, A=5, CH=3, H=0, C=0, apd=625, mode=1, table=None, nodes=fake, edges=fake,
             n8=None, e8=None, n_nodes=fake, sc=None, slot_ids=None, row=None, state=None, counters=None,
             logits=fake, first_slot=1):
        return lib.gib_action_mask_logits(B, N, F, Ef, A, CH, H, C, apd, mode, table, nodes, edges, n8, e8, n_nodes,
                                          sc, slot_ids, row, state, counters, logits, first_slot, None)

    for kw in (dict(B=0), dict(N=0), dict(N=128, apd=128 * 48 + 1), dict(F=9), dict(A=0), dict(Ef=0), dict(H=-1),
               dict(A=256, F=259), dict(apd=624), dict(mode=0), dict(mode=3), dict(mode=2), dict(nodes=None),
               dict(n8=fake), dict(nodes=None, edges=None), dict(nodes=None, n8=fake),
               dict(logits=None), dict(state=fake), dict(counters=fake), dict(first_slot=2), dict(first_slot=-1)):
        assert call(**kw) < 0, kw
        assert b"gib_action_mask_logits" in lib.gib_last_error()
    sc = Scaffolds(protect=1 << 20, n_atoms=None, S=1)
    assert call(sc=ctypes.byref(sc), slot_ids=fake) < 0
    assert b"attachment points" in lib.gib_last_error()
    sc = Scaffolds(protect=1 << 20, n_atoms=1 << 20, S=1)
    assert call(sc=ctypes.byref(sc)) < 0                   # no slot_ids


def test_route_check_refuses_bad_arguments():
    from graphinvent_b200._lib import PPDims, lib
    fake = ctypes.c_void_p(1 << 20)
    pd = PPDims(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=256)

    def call(d=pd, n=4, max_m=8, ws=fake, offsets=fake, mode=1, table=None, result=fake):
        return lib.gib_route_check_actions(ctypes.byref(d), fake, fake, n, max_m, ws, offsets, mode, table, result,
                                           None)

    for kw in (dict(n=0), dict(n=9), dict(ws=None), dict(offsets=None), dict(result=None), dict(mode=0),
               dict(mode=2), dict(d=PPDims(N=128, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, batch_size=256))):
        assert call(**kw) < 0, kw
        assert b"gib_route_check_actions" in lib.gib_last_error()


def test_rl_record_bytes_counts_the_atom_counts():
    from graphinvent_b200.graphed import rl_record_bytes
    base = rl_record_bytes(100, 13, 8, 3)
    assert rl_record_bytes(100, 13, 8, 3, action_mask=True) == base + 26 * 100 * 4
    assert rl_record_bytes(100, 13, 8, 3, masked=True, action_mask=True) == rl_record_bytes(100, 13, 8, 3, masked=True)
