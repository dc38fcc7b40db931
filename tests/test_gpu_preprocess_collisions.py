"""GPU: the training-set construction's per-group deduplication (csrc/preprocess.cu, pp_group_kernel) on route states
whose 64-bit hashes collide while their bytes differ (tests/golden/preprocess_collisions.npz), against the byte-keyed
restatement (tests/preprocess_reference.groups): rows, APD counts, group ranges and counters, bit for bit.

The group kernel keys its table by the state hash and compares the bytes of hash-equal states: on a mismatch
(warp_states_equal false) warp_first_equal scans the group's earlier states of that hash.  Ordinary molecules never
collide, so only these inputs reach that path, the hash 2^64 - 1 that the table reserves for an empty slot, and the
probe's wrap from the table's last slot to slot 0.  Each scenario first checks on the host, from the restated hashes,
that its input takes the path it is named after."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests.conftest import GOLDEN
from tests.guarded import Guarded
from tests.test_gpu_preprocess import LAYOUTS, assert_same, device_groups

pytestmark = pytest.mark.gpu

N, F, EF = 13, 8, 3
LAYOUT = LAYOUTS["gdb13"]
SEGS = P.segments(*LAYOUT)
S_MAX = N * (N - 1) // 2 + 2
TILE = 1024                                   # the group kernel's states per tile (kGroupNT)
ONE_GROUP = 4000                              # a batch_size no scenario below fills


@pytest.fixture(scope="module")
def fx():
    z = np.load(os.path.join(GOLDEN, "preprocess_collisions.npz"))
    mols = [(x, e) for x, e in zip(z["nodes"], z["edges"])]
    c = z["colliders"].tolist()
    r, w = z["reserved"].tolist(), z["wrap"].tolist()
    return dict(base=mols[0], col=[mols[i] for i in c], top=mols[r[0]], below=mols[r[1]], w1=mols[w[0]],
                w2=mols[w[1]], all=mols, hashes=z["hashes"])


@pytest.fixture(scope="module")
def gdb13():
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return {k: [(x, e) for x, e in zip(z[f"gdb13_1K_{k}/nodes"], z[f"gdb13_1K_{k}/edges"])]
            for k in ("debug_train", "train")}


def single_atom():
    X = np.zeros((N, F), np.int8)
    X[0, 0] = X[0, 6] = 1
    return X, np.zeros((N, N, EF), np.int8)


def truncated(mol, k):
    """route state k of a molecule, as a molecule of its own (its route is the rest of the molecule's route)"""
    X, E, _ = P.route(*mol, SEGS)[k]
    return X, E


def stack(mols):
    return np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])


def trace(mols):
    """per state of the molecules read as one group, in state order: the earliest state of its stored hash, the
    earliest of its bytes, the hash-equal states before it, and whether the reference appends it again as a repeat
    whose first match is the last row"""
    earliest, first, cands, quirk, rows_after = [], [], [], [], []
    by_hash, by_bytes, row_of, rows = {}, {}, {}, 0
    i = 0
    for X0, E0 in mols:
        for X, E, _ in P.route(X0, E0, SEGS):
            h = int(P.stored_hash(P.state_hash(X, E)))
            b = X.tobytes() + E.tobytes()
            cands.append(list(by_hash.get(h, [])))
            by_hash.setdefault(h, []).append(i)
            earliest.append(by_hash[h][0])
            first.append(by_bytes.setdefault(b, i))
            r = row_of.get(b)
            again = r is not None and r == rows - 1
            quirk.append(again)
            if r is None:
                row_of[b] = rows
            if r is None or again:
                rows += 1
            i += 1
        rows_after.append(rows)
    return dict(earliest=np.array(earliest), first=np.array(first), cands=cands, quirk=np.array(quirk), rows=rows,
                rows_after=np.array(rows_after))


def mismatches(t):
    """states whose hash-earliest state differs from them in content: the warp_first_equal path"""
    return np.flatnonzero(t["earliest"] != t["first"])


def check(mols, B, chunk=4096):
    nodes, edges = stack(mols)
    ref = list(P.groups(nodes, edges, B, SEGS))
    assert_same(device_groups(nodes, edges, B, LAYOUT, chunk_molecules=chunk), ref)
    return ref


def test_device_hashes_are_the_restated_ones(fx, gdb13):
    """Through gib_test_route_plan_offsets: every state's hash, APD index, node count and molecule in a
    gib_route_plan workspace (the count / scan / route kernels of gib_preprocess_chunk) equal the restatement, for the
    fixture and the gdb13_1K-debug training molecules -- the collisions are real on the device"""
    from graphinvent_b200._lib import PPDims, check as ok, lib
    mols = fx["all"] + gdb13["debug_train"]
    nodes, edges = stack(mols)
    M = len(mols)
    d = PPDims(N=N, F=F, Ef=EF, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=64)
    out = (ctypes.c_longlong * 4)()
    assert lib.gib_test_route_plan_offsets(ctypes.byref(d), M, out) == 0
    ws = Guarded(lib.gib_route_plan_ws_bytes(ctypes.byref(d), M))
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    off, st = Guarded(4 * (M + 1)), Guarded(4 * 8)
    ok(lib.gib_route_plan(ctypes.byref(d), gn.ptr(), ge.ptr(), M, M, ws.ptr(), off.ptr(), st.ptr(), None),
       "gib_route_plan")
    torch.cuda.synchronize()
    status = st.view(torch.int32).cpu().numpy()
    offsets = off.view(torch.int32).cpu().numpy()
    S = int(offsets[M])
    assert status[3] == 0 and status[5] == S
    raw = ws.t.cpu().numpy()
    h_dev = raw[out[0]:out[0] + 8 * S].view(np.uint64)
    apd, nn, mol = (raw[o:o + 4 * S].view(np.int32) for o in out[1:])
    for m, (X0, E0) in enumerate(mols):
        states = P.route(X0, E0, SEGS)
        a, b = offsets[m], offsets[m + 1]
        assert b - a == len(states), m
        want = P.stored_hash([P.state_hash(X, E) for X, E, _ in states])
        assert np.array_equal(h_dev[a:b], want), m
        assert np.array_equal(apd[a:b], [s[2] for s in states]), m
        assert np.array_equal(nn[a:b], [P.n_atoms(s[0]) for s in states]), m
        assert (mol[a:b] == m).all()
        if m < len(fx["all"]):
            assert np.array_equal(want, P.stored_hash(fx["hashes"][m])), m
    for g in (ws, gn, ge, off, st):
        assert g.intact(), g.damage()


def test_adjacent_colliders(fx):
    """The base, then its colliders: each collider's first 13 states sit in one warp and all take the mismatch
    path, scanning past every earlier collider's state of that hash"""
    mols = [fx["base"]] + fx["col"]
    t = trace(mols)
    mis = mismatches(t)
    assert mis.size >= 13 * len(fx["col"])
    assert np.bincount(mis // 32).max() >= 13           # the first group's tiles start at state 0
    ref = check(mols, ONE_GROUP)
    assert len(ref) == 1
    assert len(check(mols, 300)) > 2                    # groups cut inside colliders


def test_colliders_across_tiles(fx, gdb13):
    """Colliders more than a tile of states apart in one group, copies of one filler molecule between them"""
    filler = gdb13["debug_train"][0]
    gap = -(-(TILE + 1) // len(P.route(*filler, SEGS)))
    mols = [fx["base"]]
    for c in fx["col"][:3]:
        mols += [filler] * gap + [c]
    t = trace(mols)
    mis = mismatches(t)
    far = [i for i in mis if i // TILE != t["earliest"][i] // TILE and i - t["earliest"][i] > TILE]
    assert len(far) >= 3 * 13
    ref = check(mols, ONE_GROUP)
    assert len(ref) == 1 and ref[0]["nodes"].shape[0] < ONE_GROUP


def three_way(fx):
    """base, X, Y, a copy of Y, a copy of the base; then Z truncated to its state 12, Z and a copy of Z"""
    base, (X, Y, Z) = fx["base"], fx["col"][:3]
    return [base, X, Y, Y, base, truncated(Z, 12), Z, Z]


def test_three_way(fx):
    """The copy of Y finds Y behind the base's and X's states of its hash; the copy of the base takes the equal
    path to the base.  Z's truncation puts Z's state 11 last among the rows before Z's copy, so the copy's state 11 --
    whose hash-earliest state is the base's -- is appended again by the reference's last-row rule"""
    mols = three_way(fx)
    t = trace(mols)
    y2, b2, z2 = 3 * S_MAX, 4 * S_MAX, 5 * S_MAX + (S_MAX - 12) + S_MAX
    assert t["earliest"][y2] == 0 and t["first"][y2] == 2 * S_MAX
    assert [c for c in t["cands"][y2] if t["first"][c] != t["first"][y2]] == [0, S_MAX]
    assert t["earliest"][b2] == t["first"][b2] == 0
    assert t["quirk"][z2 + 11] and t["earliest"][z2 + 11] == 11 and t["first"][z2 + 11] != 11
    ref = check(mols, ONE_GROUP)
    assert len(ref) == 1 and t["rows"] == ref[0]["nodes"].shape[0]


def carried(ref, M, B, chunk):
    """groups that reach the end of a chunk call's molecules unfilled inside their window of B molecules: the call
    leaves them to the next call, which starts at their first molecule (preprocess.groups' chunk walk)"""
    pos, gi, n = 0, 0, 0
    while gi < len(ref):
        end = min(pos + chunk, M)
        while gi < len(ref):
            g = ref[gi]
            if end == M or g["start"] + B <= end or (g["full"] and g["stop"] <= end):
                gi += 1
            else:
                n += 1
                break
        pos = ref[gi]["start"] if gi < len(ref) else M
    return n


def lifetime_molecules(fx, gdb13, B):
    """a group cut inside the base, the next one starting at a collider, later copies of the base and the colliders,
    and groups that start mid-chunk and run out of the chunk's molecules before they fill (single atoms add a row or
    two per group)"""
    base, (X, Y) = fx["base"], fx["col"][:2]
    S = single_atom()
    if B < S_MAX:
        return [S, base, X, S, S, base, X, Y, S, S, S, Y, X]
    # gdb13 molecules filling all but the last part of the base's route
    lead = gdb13["train"][:200]
    k = int(np.searchsorted(trace(lead)["rows_after"], B - S_MAX // 2))
    return lead[:k] + [base, X, base, Y, Y] + [S] * B + [X, base]


@pytest.mark.parametrize("B", [5, 1000])
def test_table_lifetime(fx, gdb13, B):
    """A group cut between the base and a collider, so the next group starts from a cleared table, with copies of
    the base in later groups; chunks of B molecules with a group whose window crosses a chunk's end, so the next call
    rebuilds the table.  B = 5: a table of 1024 slots"""
    mols = lifetime_molecules(fx, gdb13, B)
    nodes, edges = stack(mols)
    ref = list(P.groups(nodes, edges, B, SEGS))
    base_at = [i for i, m in enumerate(mols) if m is fx["base"]]
    col_at = {i for i, m in enumerate(mols) if any(m is c for c in fx["col"])}
    cut = [g for g in ref if g["full"] and g["stop"] - 1 == base_at[0] and g["stop"] in col_at]
    assert len(cut) == 1
    assert any(g["index"] > cut[0]["index"] and g["start"] <= b < g["stop"] for g in ref for b in base_at[1:])
    assert carried(ref, len(mols), B, B) >= 1
    if B < S_MAX:
        assert 2 * B * S_MAX <= 1024
    assert_same(device_groups(nodes, edges, B, LAYOUT, chunk_molecules=B), ref)


def test_reserved_key(fx):
    """The state of hash 2^64 - 1, stored as 2^64 - 2, then a state whose hash is 2^64 - 2, then copies of each"""
    top, below = fx["top"], fx["below"]
    h = [P.state_hash(*m) for m in (top, below)]
    assert h[0] == P.RESERVED and h[1] == P.RESERVED - np.uint64(1)
    mols = [top, below, top, below]
    t = trace(mols)
    assert t["earliest"][S_MAX] == 0 and t["first"][S_MAX] == S_MAX
    assert t["earliest"][3 * S_MAX] == 0 and t["first"][3 * S_MAX] == S_MAX
    check(mols, ONE_GROUP)


def test_probe_wraps_to_slot_0(fx, gdb13):
    """Two full graphs whose distinct hashes end in 20 one-bits: the first takes the table's last slot, the second,
    a tile later, wraps to slot 0, where a copy of it must find it"""
    w1, w2 = fx["w1"], fx["w2"]
    filler = gdb13["debug_train"][1]
    gap = -(-(TILE + 1) // len(P.route(*filler, SEGS)))
    mols = [w1] + [filler] * gap + [w2, w2, w1]
    M = len(mols)
    table = 1024
    while table < 2 * min(M, ONE_GROUP) * S_MAX:       # the group kernel's table for a chunk of M molecules
        table *= 2
    mask = np.uint64(table - 1)
    assert table <= 1 << 20
    hw = [P.state_hash(*m) for m in (w1, w2)]
    assert hw[0] != hw[1] and all(h & mask == mask for h in hw)
    w2_at = S_MAX + gap * len(P.route(*filler, SEGS))
    assert w2_at // TILE > 0
    t = trace(mols)
    assert t["first"][w2_at + S_MAX] == w2_at
    check(mols, ONE_GROUP)


def test_poisoned_workspace(fx):
    """The three-way scenario through the C ABI on a poisoned, guard-banded workspace and outputs, twice (the
    second call finds the first call's workspace)"""
    from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, lib
    mols = three_way(fx)
    nodes, edges = stack(mols)
    M, B = len(mols), ONE_GROUP
    max_rows = B
    ref = list(P.groups(nodes, edges, B, SEGS))
    rows = sum(r["nodes"].shape[0] for r in ref)
    d = PPDims(N=N, F=F, Ef=EF, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=B)
    apd = lib.gib_preprocess_apd_length(ctypes.byref(d))
    ws = Guarded(lib.gib_preprocess_ws_bytes(ctypes.byref(d), M, max_rows))
    gn = Guarded.like(torch.from_numpy(nodes).cuda())
    ge = Guarded.like(torch.from_numpy(edges).cuda())
    on, oe = Guarded(max_rows * N * F), Guarded(max_rows * N * N * EF)
    oa, og, st = Guarded(4 * max_rows * apd), Guarded(4 * 4 * M), Guarded(4 * PP_STATUS_INTS)
    for _ in range(2):
        rc = lib.gib_preprocess_chunk(ctypes.byref(d), gn.ptr(), ge.ptr(), M, 1, M, max_rows, ws.ptr(), on.ptr(),
                                      oe.ptr(), oa.ptr(), og.ptr(), st.ptr(), None)
        assert rc == 0
        torch.cuda.synchronize()
        status = st.view(torch.int32).cpu().numpy()
        assert status[0] == len(ref) == 1 and status[1] == M and status[2] == rows and status[3] == 0
        assert og.view(torch.int32)[:4].cpu().tolist() == [0, M, 0, rows]
        assert np.array_equal(on.view(torch.int8)[:rows * N * F].cpu().numpy(), ref[0]["nodes"].ravel())
        assert np.array_equal(oe.view(torch.int8)[:rows * N * N * EF].cpu().numpy(), ref[0]["edges"].ravel())
        assert np.array_equal(oa.view(torch.int32)[:rows * apd].cpu().numpy(), ref[0]["apds"].ravel())
        for g in (ws, gn, ge, on, oe, oa, og, st):
            assert g.intact(), g.damage()
