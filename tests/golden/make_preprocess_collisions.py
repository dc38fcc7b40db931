"""Writes tests/golden/preprocess_collisions.npz: gdb13-layout molecules (N = 13, F = 8, Ef = 3) whose route states
collide in the training-set construction's 64-bit state hash (tests/preprocess_reference.state_hash, the key of
gib_preprocess_chunk's dedup table) while their bytes differ.

    python tests/golden/make_preprocess_collisions.py

The hash is a sum mod 2^64 of per-byte mixes, so a collision is a generalized birthday problem, solved here with
Wagner's four-list algorithm.  Every molecule is a complete graph of 13 atoms (one atom type and one charge for all).
The base has single bonds only; each other molecule changes the bond types of some of 56 pairs among atoms 0-11.  The
pairs are split into four lists of 14, each list holding the 3^14 hash changes of its pairs' type choices.  The
lists are joined pairwise on the low 22 bits and the two joins on all 64 bits, to a target sum:
  - 0: colliders, whose full graph has the base's hash (the all-single-bond solution, the base itself, is dropped);
  - 2^64 - 1 - h(base) and 2^64 - 2 - h(base): the full graphs whose hash is the table's empty-slot key, which the
    route kernel stores as 2^64 - 2, and a full graph whose hash really is 2^64 - 2.
Atom 12 keeps single bonds to every atom, so the route removes the same bytes in the same order from every molecule
for 12 steps: by additivity the first 13 route states (the full graph, then atom 12's 12 bond removals) collide
across the base and its colliders, and so does a later state k of two colliders whose routes happen to have removed
the same bytes by step k.  The wrap pair: two molecules that vary one list's pairs only, whose full-graph
hashes differ but have their low 20 bits all ones, so they take the last slot of any table of up to 2^20 slots and
the second one inserted wraps around to slot 0.

Everything claimed above is asserted before anything is written.  The search is seeded and the npz is written
uncompressed with fixed zip timestamps, so a rerun reproduces the file byte for byte (a few minutes on a CPU).

Stored: nodes int8 [M, 13, 8], edges int8 [M, 13, 13, 3], hashes uint64 [M, 80] (every route state's state_hash,
truncation order, not remapped); molecule 0 is the base, `colliders` its colliders, `reserved` the molecules of full
hash 2^64 - 1 and 2^64 - 2, `wrap` the wrap pair; `collide_states` = 13.
"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import preprocess_reference as P  # noqa: E402

SEED = 2024
N, F, EF = 13, 8, 3
SEGS = P.segments(5, 3)
NB = N * F
S_MAX = N * (N - 1) // 2 + 2
COLLIDE = 13                        # route states 0..12: the full graph and atom 12's bond removals
LIST = 14                           # pairs per list: 3^14 = 4 782 969 sums
LOW = np.uint64((1 << 22) - 1)      # the first join's bits
WRAP_BITS = 20
U = np.uint64


def base_molecule():
    X = np.zeros((N, F), np.int8)
    X[:, 0] = 1                     # atom type 0
    X[:, 6] = 1                     # the neutral charge
    E = np.zeros((N, N, EF), np.int8)
    for i in range(N):
        for j in range(N):
            if i != j:
                E[i, j, 0] = 1
    return X, E


def edge_pos(i, j, t):
    return NB + (i * N + j) * EF + t


def delta(i, j, t):
    """the state-hash change of bond (i, j) going from type 0 to type t"""
    pos = [edge_pos(i, j, t), edge_pos(j, i, t), edge_pos(i, j, 0), edge_pos(j, i, 0)]
    h = P.byte_hash(pos, [1, 1, 1, 1])
    with np.errstate(over="ignore"):
        return h[0] + h[1] - h[2] - h[3]


def list_sums(pairs):
    """the 3^len(pairs) hash changes of the pairs' type choices; index digit k (base 3, most significant first) is
    pair k's type"""
    s = np.zeros(1, U)
    for i, j in pairs:
        d = np.array([0, delta(i, j, 1), delta(i, j, 2)], U)
        with np.errstate(over="ignore"):
            s = (s[:, None] + d[None, :]).ravel()
    return s


def choices(idx):
    out = []
    for _ in range(LIST):
        out.append(idx % 3)
        idx //= 3
    return out[::-1]


def join(a, b, mask):
    """every index pair (ia, ib) with (a[ia] + b[ib]) & mask == 0, in the order of ia then b's stable sort"""
    ka = a & mask
    with np.errstate(over="ignore"):
        kb = (U(0) - b) & mask
    ob = np.argsort(kb, kind="stable")
    kbs = kb[ob]
    lo = np.searchsorted(kbs, ka, "left")
    hi = np.searchsorted(kbs, ka, "right")
    cnt = hi - lo
    ia = np.repeat(np.arange(a.size), cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    ib = ob[np.repeat(lo, cnt) + (np.arange(int(cnt.sum())) - start)]
    return ia, ib


def variant(lists_pairs, idx):
    """the base with each list's pairs set to the types its index encodes"""
    X, E = base_molecule()
    for pairs, ix in zip(lists_pairs, idx):
        for (i, j), t in zip(pairs, choices(int(ix))):
            if t:
                E[i, j, 0] = E[j, i, 0] = 0
                E[i, j, t] = E[j, i, t] = 1
    return X, E


def solve(lists, z, b3, b4, target):
    """index quadruples whose four list sums add up to target mod 2^64 (z, b3, b4: the join of lists 2 and 3)"""
    with np.errstate(over="ignore"):
        l0 = lists[0] - U(target)
        a1, a2 = join(l0, lists[1], LOW)
        y = l0[a1] + lists[1][a2]
    iy, iz = join(y, z, U(0xFFFFFFFFFFFFFFFF))
    return sorted(zip(a1[iy].tolist(), a2[iy].tolist(), b3[iz].tolist(), b4[iz].tolist()))


def check_molecule(X, E):
    assert X.shape == (N, F) and E.shape == (N, N, EF)
    assert (X[:, :5].sum(1) == 1).all() and (X[:, 5:].sum(1) == 1).all()
    assert np.array_equal(E, E.transpose(1, 0, 2)) and set(np.unique(E)) <= {0, 1}
    bonded = E.sum(2)
    assert (np.diag(bonded) == 0).all() and (bonded + np.eye(N, dtype=np.int8) == 1).all()   # complete, one type
    assert (E[12, :12, 0] == 1).all()          # atom 12: single bonds to every atom, in every molecule


def states_bytes(X, E):
    return [x.tobytes() + e.tobytes() for x, e, _ in P.route(X, E, SEGS)]


def removed(full, state):
    """the (position, byte) pairs a route has zeroed between its full graph and a later state"""
    f, s = np.frombuffer(full, np.int8), np.frombuffer(state, np.int8)
    q = np.flatnonzero(f != s)
    return tuple(zip(q.tolist(), f[q].tolist()))


def main():
    rng = np.random.default_rng(SEED)
    all_pairs = [(i, j) for i in range(12) for j in range(i + 1, 12)]
    pick = rng.permutation(len(all_pairs))[:4 * LIST]
    lists_pairs = [[all_pairs[k] for k in pick[q * LIST:(q + 1) * LIST]] for q in range(4)]
    lists = [list_sums(p) for p in lists_pairs]
    b3, b4 = join(lists[2], lists[3], LOW)
    with np.errstate(over="ignore"):
        z = lists[2][b3] + lists[3][b4]
    X0, E0 = base_molecule()
    h0 = P.state_hash(X0, E0)

    with np.errstate(over="ignore"):
        sols = [s for s in solve(lists, z, b3, b4, 0) if any(s)]
        top = solve(lists, z, b3, b4, P.RESERVED - h0)
        below = solve(lists, z, b3, b4, P.RESERVED - U(1) - h0)
    print(f"colliders {len(sols)}, hash 2^64-1: {len(top)}, hash 2^64-2: {len(below)}")
    assert len(sols) >= 6 and top and below

    mask = U((1 << WRAP_BITS) - 1)
    wraps = []
    for q in range(4):
        with np.errstate(over="ignore"):
            full = h0 + lists[q]
        for ix in np.flatnonzero((full & mask) == mask).tolist():
            if full[ix] not in (P.RESERVED, P.RESERVED - U(1)) and all(full[ix] != w[2] for w in wraps):
                wraps.append((q, ix, full[ix]))
    assert len(wraps) >= 2, wraps
    wrap_idx = []
    for q, ix, _ in wraps[:2]:
        idx = [0, 0, 0, 0]
        idx[q] = ix
        wrap_idx.append(idx)

    mols = [(X0, E0)] + [variant(lists_pairs, s) for s in sols]
    mols += [variant(lists_pairs, top[0]), variant(lists_pairs, below[0])]
    mols += [variant(lists_pairs, w) for w in wrap_idx]
    M = len(mols)
    colliders = np.arange(1, 1 + len(sols))
    reserved = np.array([M - 4, M - 3])
    wrap = np.array([M - 2, M - 1])
    for X, E in mols:
        check_molecule(X, E)
    hashes = np.stack([P.route_hashes(X, E, SEGS) for X, E in mols])
    assert hashes.shape == (M, S_MAX)
    bytes_ = [states_bytes(X, E) for X, E in mols]

    # the collision class: the first 13 states collide across the base and its colliders, and differ in their bytes
    cls = np.concatenate([[0], colliders])
    for k in range(COLLIDE):
        assert (hashes[cls, k] == hashes[0, k]).all(), k
        assert len({bytes_[m][k] for m in cls}) == cls.size, k
    assert (hashes[cls, COLLIDE] != hashes[0, COLLIDE]).any()
    # the reserved key: raw full hashes 2^64 - 1 and 2^64 - 2, one stored key
    assert hashes[reserved[0], 0] == P.RESERVED and hashes[reserved[1], 0] == P.RESERVED - U(1)
    assert P.stored_hash(hashes[reserved[0], 0]) == P.stored_hash(hashes[reserved[1], 0])
    # the wrap pair: distinct full hashes, low 20 bits all ones
    w0, w1 = hashes[wrap, 0]
    assert w0 != w1 and (w0 & mask) == mask and (w1 & mask) == mask
    # no chance collision: states of one stored hash and different bytes are the reserved pair's full graphs, or the
    # same state k of colliders whose routes have removed the same bytes by then (by additivity: the first 13 states
    # of every collider, and later ones where two colliders' removals happen to coincide)
    seen = {}
    for m in range(M):
        for k, h in enumerate(P.stored_hash(hashes[m]).tolist()):
            seen.setdefault(h, {}).setdefault(bytes_[m][k], []).append((m, k))
    for h, contents in seen.items():
        if len(contents) < 2:
            continue
        members = [mk for v in contents.values() for mk in v]
        if sorted(members) == [(int(reserved[0]), 0), (int(reserved[1]), 0)]:
            continue
        assert all(m in cls for m, _ in members) and len({k for _, k in members}) == 1, members
        assert len({removed(bytes_[m][0], bytes_[m][k]) for m, k in members}) == 1, members
    assert sum(len(c) > 1 for c in seen.values()) >= COLLIDE + 1

    out = dict(nodes=np.stack([m[0] for m in mols]), edges=np.stack([m[1] for m in mols]), hashes=hashes,
               colliders=colliders, reserved=reserved, wrap=wrap, collide_states=np.int64(COLLIDE))
    path = os.path.join(HERE, "preprocess_collisions.npz")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as zf:
        for name in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(out[name]), allow_pickle=False)
            zf.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue())
    print(f"{M} molecules: the base, {len(sols)} colliders, the reserved-key pair, the wrap pair -> {path}")


if __name__ == "__main__":
    main()
