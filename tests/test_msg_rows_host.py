"""CPU: the numpy restatement of the message-row table (tests/msg_rows_reference.py) on K0's numpy restatement, checked
against what the table is for -- every dst slot aggregates the same (source slot, bond value, type) terms as over the
bond entries, every message row is the message of each entry it stands for, and every row goes back to its source."""
from collections import Counter

import numpy as np
import pytest

from tests.k0_reference import k0_reference
from tests.msg_rows_reference import MR_COUNT, msg_rows_reference


def _bonds(kind, B, N, Ef, seed):
    rng = np.random.default_rng(seed)
    e = np.zeros((B, N, N, Ef), np.float32)
    b, i, j = np.nonzero(rng.random((B, N, N)) < 0.25)
    e[b, i, j, rng.integers(0, Ef, b.size)] = 1.0
    b, i, j = np.nonzero(rng.random((B, N, N)) < 0.05)               # a second bond type on some cells
    e[b, i, j, rng.integers(0, Ef, b.size)] = 1.0
    if kind == "values":                                              # non-binary values, some equal to 1
        nz = np.nonzero(e)
        e[nz] = rng.choice(np.array([0.5, 2.0, 1.0, 1.0, -3.0, np.nan], np.float32), nz[0].size)
    e[0] = 0.0                                                        # an empty molecule
    e[:, N - 1] = 0.0                                                 # an atom without bonds in every molecule
    e[:, :, N - 1] = 0.0
    return e


def _type_of(p, tb, G):
    return max(t for t in range(G) if tb[t] <= p)


def table(e, capacity=None):
    r = k0_reference(e, True, capacity)
    E = r.cap_E
    t = msg_rows_reference(r.ent_src, r.ent_dst, r.ent_w, r.dst_ptr, r.dst_ent, r.src_ptr, r.src_ent, r.type_base,
                           r.G, E)
    return r, t


CASES = [("binary", 7, 9, 3, 0), ("binary", 5, 6, 1, 1), ("values", 6, 8, 4, 2), ("values", 4, 11, 2, 3)]


@pytest.mark.parametrize("kind,B,N,Ef,seed", CASES)
def test_message_rows_restate_the_bond_entries(kind, B, N, Ef, seed):
    e = _bonds(kind, B, N, Ef, seed)
    r, t = table(e)
    tb, G, S = list(r.type_base), r.G, r.S
    key = lambda w: np.float32(w).view(np.int32).item()               # NaN-safe, bitwise
    # every dst slot: the same (source, value, type) terms in the same order
    for s in range(S):
        q = range(r.dst_ptr[s], r.dst_ptr[s + 1])
        want = [(r.ent_src[r.dst_ent[k]], key(r.ent_w[r.dst_ent[k]]), _type_of(r.dst_ent[k], tb, G)) for k in q]
        got = [(t["u_src"][t["dst_u"][k]], key(t["u_w"][t["dst_u"][k]]), _type_of(t["dst_u"][k], tb, G)) for k in q]
        assert got == want, s
    # every message row: the entries it stands for (u_ptr / u_dst) are the entries mapped to it
    dst_of_row = {}
    for p in range(r.P):
        if r.ent_src[p] >= 0:
            dst_of_row.setdefault(t["ent_u"][p], []).append(r.ent_dst[p])
            assert t["u_src"][t["ent_u"][p]] == r.ent_src[p]
    for u in range(r.P):
        seg = list(t["u_dst"][t["u_ptr"][u]:t["u_ptr"][u + 1]])
        assert sorted(seg) == sorted(dst_of_row.get(u, [])), u
        if t["u_src"][u] < 0:
            assert seg == [] and t["u_w"][u] == 0
    # the slot CSR lists exactly the rows of each source slot; no row is shared by two (source, type, value) keys
    for s in range(S):
        rows = t["s_u"][t["s_ptr"][s]:t["s_ptr"][s + 1]]
        assert sorted(rows) == sorted(np.flatnonzero(t["u_src"] == s)), s
    live = t["u_src"] >= 0
    keys = Counter((t["u_src"][u], _type_of(u, tb, G)) for u in np.flatnonzero(live & (t["u_w"] == 1)))
    assert max(keys.values(), default=1) == 1
    # fewer rows than entries in every type, each group inside its entry group
    for g in range(G):
        assert t["meta"][MR_COUNT + g] <= r.type_count[g]
    if kind == "binary":
        assert live.sum() < r.E


def test_capacity_mode_lists_the_kept_entries_only():
    """an overflowing capacity: K0 lists row 0 for the entries it dropped; the table leaves them out and stays inside its
    arrays, and a capacity that fits gives the exact table"""
    e = _bonds("binary", 9, 8, 3, 4)
    r0, t0 = table(e)
    r1, t1 = table(e, capacity=r0.E + 50)
    for k in ("u_src", "u_w", "ent_u"):
        assert np.array_equal(t1[k][:r0.P], t0[k]), k
    r2, t2 = table(e, capacity=int(r0.E * 0.7))
    assert r2.overflow
    kept = (r2.ent_src >= 0)
    assert set(np.flatnonzero(t2["ent_u"] >= 0)) <= set(np.flatnonzero(kept))
    assert (t2["s_ptr"] <= r2.cap_E).all() and t2["u_ptr"].max() <= r2.cap_E
