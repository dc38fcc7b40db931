"""GPU: the molecule set (graphinvent_b200.molecules.MoleculeSet, `gib_molset_identify` in csrc/preprocess.cu) against
its restatement (tests/molecule_set_reference.py), bit for bit: ids, new / first flags, counts and entry bytes.

  1. gdb13_1K/train: ids 0..978, all new and first; every molecule again with its atoms shuffled: the same ids, none
     new, counts 2;
  2. generated batches of the pretrained gdb13 GGNN (float32 as sampled) into one set; `uniqueness` with the properly
     terminated mask;
  3. worst-case groups: 1000 shuffled copies of one molecule interleaved with the 1-WL collision pair; chains of
     colliding entries;
  4. one call and several calls give the same set;
  5. `find` leaves every set buffer as it was; novelty against a training set;
  6. the four layouts x Ef 1-4 and ring-rich molecules at N = 38, 127 and 181; int8 and float32 inputs agree;
  7. refusals leave the set byte for byte unchanged; n = 0 and the empty molecule;
  8. guard-banded, poisoned set and workspace buffers.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import molecule_set_reference as MS
from tests import scaffold_match_reference as SM
from tests.conftest import GOLDEN, pretrained_path
from tests.guarded import Guarded
from tests.test_murcko_host import GDB13, decalin_and_bicyclopentyl, ring_rich
from tests.test_scaffold_match_host import LAYOUTS

pytestmark = pytest.mark.gpu


def _gdb13():
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]


def _shuffled(nodes, edges, seed):
    rng = np.random.default_rng(seed)
    pairs = [SM.shuffle(x, e, rng) for x, e in zip(nodes, edges)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def _new_set(N, F, Ef, capacity, layout=GDB13, **kw):
    from graphinvent_b200.molecules import MoleculeSet
    return MoleculeSet(N, F, Ef, capacity, layout=layout, **kw)


def _host(ident):
    return tuple(t.cpu().numpy() for t in ident)


def _assert_identity(got, want):
    for g, w, name in zip(_host(got), want, ("ids", "new", "first")):
        assert np.array_equal(g, w), name


def _assert_entries(s, ref):
    nodes, edges, counts = ref.arrays(s.N, s.F, s.Ef)
    assert len(s) == len(ref)
    en, ee = s.entries()
    assert np.array_equal(en.cpu().numpy(), nodes) and np.array_equal(ee.cpu().numpy(), edges)
    assert np.array_equal(s.counts.cpu().numpy(), counts)


def _snapshot(s):
    return [t.clone() for t in s.buffers()]


def _unchanged(s, snap):
    return all(torch.equal(a, b) for a, b in zip(s.buffers(), snap))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the training set
# ---------------------------------------------------------------------------------------------------------------------
def test_gdb13():
    nodes, edges = _gdb13()
    M, N, F = nodes.shape
    s, ref = _new_set(N, F, edges.shape[3], 2 * M), MS.MoleculeSet()
    got = s.add(nodes, edges)
    _assert_identity(got, ref.add(nodes, edges))
    ids, new, first = _host(got)
    assert ids.tolist() == list(range(M)) and new.all() and first.all()
    X, E = _shuffled(nodes, edges, 3)
    got = s.add(X, E)
    _assert_identity(got, ref.add(X, E))
    ids2, new2, first2 = _host(got)
    assert np.array_equal(ids2, ids) and not new2.any() and first2.all()
    _assert_entries(s, ref)
    assert (s.counts.cpu().numpy() == 2).all()
    assert len(set(s._hash[:len(s)].cpu().numpy().tolist())) == M


# ---------------------------------------------------------------------------------------------------------------------
# 2. generated batches
# ---------------------------------------------------------------------------------------------------------------------
def test_generated_batches_and_uniqueness():
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator
    from graphinvent_b200.molecules import uniqueness
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    C = make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    net = net.cuda().eval()
    B = 1000
    gen = GraphedGenerator(net, B, n_atom_types=5, n_formal_charge=3)
    s, ref = _new_set(13, 8, 3, 4 * B), MS.MoleculeSet()
    repeats = 0
    for seed in range(3):
        U = torch.rand(2 * 13, B, generator=torch.Generator("cuda").manual_seed(seed), device="cuda")
        (nodes, edges, _), _, _, pt = gen.sample(uniforms=U)
        assert nodes.dtype == torch.float32
        hn = nodes.cpu().numpy().astype(np.int8)
        he = edges.cpu().numpy().astype(np.int8)
        got = s.add(nodes, edges)
        _assert_identity(got, ref.add(hn, he))
        repeats += int((~got.first).sum())
        valid = pt.bool()
        u = uniqueness(nodes, edges, valid, layout=GDB13)
        _, _, f = MS.MoleculeSet().add(hn, he, valid.cpu().numpy())
        want = np.where(valid.cpu().numpy(), f, True).astype(np.float32)
        assert u.dtype == torch.float32 and u.is_cuda and np.array_equal(u.cpu().numpy(), want)
    _assert_entries(s, ref)
    assert repeats > 0


# ---------------------------------------------------------------------------------------------------------------------
# 3. worst-case groups and colliding chains
# ---------------------------------------------------------------------------------------------------------------------
def test_worst_case_groups():
    (dX, dE), (bX, bE) = decalin_and_bicyclopentyl(N=13)
    nodes, edges = _gdb13()
    rng = np.random.default_rng(9)
    mols = []
    for i in range(1000):
        mols.append(SM.shuffle(nodes[17], edges[17], rng))
        if i % 50 == 0:
            mols.append(SM.shuffle(*((dX, dE) if i % 100 else (bX, bE)), rng))
    X, E = np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])
    s, ref = _new_set(13, 8, 3, 16), MS.MoleculeSet()
    got = s.add(X, E)
    _assert_identity(got, ref.add(X, E))
    _assert_entries(s, ref)
    assert len(s) == 3 and sorted(s.counts.cpu().numpy().tolist()) == [10, 10, 1000]
    # a set whose chain holds colliding entries: decalin and bicyclopentyl in separate calls, then looked up
    s2, ref2 = _new_set(13, 8, 3, 8), MS.MoleculeSet()
    for Xs, Es in (([bX], [bE]), ([nodes[3]], [edges[3]]), ([dX], [dE])):
        _assert_identity(s2.add(np.stack(Xs), np.stack(Es)), ref2.add(np.stack(Xs), np.stack(Es)))
    h = s2._hash.cpu().numpy()[:3]
    assert h[0] == h[2] and s2._next.cpu().numpy()[0] == 2
    X2, E2 = _shuffled(np.stack([dX, bX, dX]), np.stack([dE, bE, dE]), 4)
    _assert_identity(s2.find(X2, E2), ref2.find(X2, E2))
    assert s2.find(X2, E2).ids.cpu().tolist() == [2, 0, 2]


# ---------------------------------------------------------------------------------------------------------------------
# 4-5. chunking, find, novelty
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_equal_one_call():
    nodes, edges = _gdb13()
    rng = np.random.default_rng(2)
    pick = rng.integers(0, 300, 900)
    X, E = _shuffled(nodes[pick], edges[pick], 5)
    whole = _new_set(13, 8, 3, 1000)
    ids = whole.add(X, E).ids.cpu().numpy()
    parts = _new_set(13, 8, 3, 1000)
    got = [parts.add(torch.from_numpy(X[a:b]).cuda(), torch.from_numpy(E[a:b]).cuda()).ids.cpu().numpy()
           for a, b in ((0, 1), (1, 200), (200, 201), (201, 640), (640, 900))]
    assert np.array_equal(np.concatenate(got), ids)
    for u, v in zip(whole.entries() + (whole.counts,), parts.entries() + (parts.counts,)):
        assert torch.equal(u, v)


def test_find_changes_nothing_and_novelty():
    nodes, edges = _gdb13()
    train = _new_set(13, 8, 3, 1000)
    train.add(nodes, edges)
    snap = _snapshot(train)
    X, E = _shuffled(nodes, edges, 6)
    got = train.find(X, E)
    assert _unchanged(train, snap)
    ids, new, first = _host(got)
    assert ids.tolist() == list(range(979)) and not new.any() and first.all()
    rng = np.random.default_rng(12)
    rnd = [SM.random_molecule(rng, int(rng.integers(9, 14)), 13, GDB13, 3, n_types=5, extra_bonds=0.5)
           for _ in range(400)]
    RX, RE = np.stack([r[0] for r in rnd]), np.stack([r[1] for r in rnd])
    ref = MS.MoleculeSet()
    ref.add(nodes, edges)
    want = ref.find(RX, RE)
    disjoint = want[0] < 0
    assert disjoint.sum() > 350
    got = train.find(RX[disjoint], RE[disjoint])
    assert _unchanged(train, snap)
    _assert_identity(got, tuple(w[disjoint] for w in ref.find(RX[disjoint], RE[disjoint])))
    assert (got.ids == -1).all() and got.new.all()


# ---------------------------------------------------------------------------------------------------------------------
# 6. dims
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Ef", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(layout, Ef):
    rng = np.random.default_rng(10 * list(LAYOUTS).index(layout) + Ef)
    nodes, edges = ring_rich(rng, 48, 38, LAYOUTS[layout], Ef, hi=20)
    X2, E2 = _shuffled(nodes[:16], edges[:16], 1)
    X, E = np.concatenate([nodes, X2]), np.concatenate([edges, E2])
    F = X.shape[2]
    s, ref = _new_set(38, F, Ef, 128, layout=LAYOUTS[layout]), MS.MoleculeSet()
    got = s.add(X, E)
    _assert_identity(got, ref.add(X, E))
    _assert_entries(s, ref)
    f = _new_set(38, F, Ef, 128, layout=LAYOUTS[layout])      # float32 inputs: the same set
    _assert_identity(f.add(torch.from_numpy(X).float().cuda(), torch.from_numpy(E).float().cuda()), _host(got))
    for u, v in zip(s.buffers()[:7], f.buffers()[:7]):
        assert torch.equal(u[:len(s)], v[:len(f)])


@pytest.mark.parametrize("N", [127, 181])
def test_large_n(N):
    rng = np.random.default_rng(N)
    nodes, edges = ring_rich(rng, 4, N, GDB13, 1, lo=N - 40)
    X2, E2 = _shuffled(nodes, edges, 2)
    X, E = np.concatenate([nodes, X2]), np.concatenate([edges, E2])
    s, ref = _new_set(N, 8, 1, 16), MS.MoleculeSet()
    _assert_identity(s.add(X, E), ref.add(X, E))
    _assert_entries(s, ref)
    assert s.counts.cpu().tolist() == [2] * 4


# ---------------------------------------------------------------------------------------------------------------------
# 7. refusals, empty inputs
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_set_unchanged():
    nodes, edges = _gdb13()
    s = _new_set(13, 8, 3, 60)
    s.add(nodes[:20], edges[:20])
    snap = _snapshot(s)
    X, E = nodes[20:60].copy(), edges[20:60].copy()
    cut = E.copy()
    a = SM.n_atoms(X[17]) - 1
    cut[17, a, :] = 0
    cut[17, :, a] = 0
    with pytest.raises(ValueError, match="molecule 17 .*disconnected"):
        s.add(X, cut)
    bad = X.copy()
    bad[23, 0, :5] = 1
    with pytest.raises(ValueError, match="molecule 23 .*node row"):
        s.add(bad, E)
    gap = X.copy()
    gap[5, 1] = 0                                              # a zero row between atoms
    with pytest.raises(ValueError, match="molecule 5 .*zero row"):
        s.add(gap, E)
    fl = torch.from_numpy(X).float().cuda()
    fl[8, 0, 0] = 0.5
    with pytest.raises(ValueError, match="molecule 8 "):
        s.add(fl, torch.from_numpy(E).float().cuda())
    (dX, dE), _ = decalin_and_bicyclopentyl(N=13)
    tiny = _new_set(13, 8, 3, 8, budget=2)
    tiny.add(dX[None], dE[None])
    tiny_snap = _snapshot(tiny)
    with pytest.raises(ValueError, match="molecule 0 .*budget"):
        tiny.add(SM.shuffle(dX, dE, np.random.default_rng(1))[0][None], SM.shuffle(dX, dE, np.random.default_rng(1))[1][None])
    assert _unchanged(tiny, tiny_snap)
    assert _unchanged(s, snap)
    # capacity: 40 new classes fit exactly, 41 do not; the refused call names the molecule of the 41st
    with pytest.raises(ValueError, match="molecule 40 .*full"):
        s.add(nodes[20:61], edges[20:61])
    assert _unchanged(s, snap)
    got = s.add(nodes[20:60], edges[20:60])
    assert len(s) == 60 and got.new.all()
    with pytest.raises(ValueError, match="molecule 0 .*full"):
        s.add(nodes[60:61], edges[60:61])
    snap = _snapshot(s)
    ids = s.add(nodes[:60:3], edges[:60:3]).ids                # known molecules still fit
    assert ids.cpu().tolist() == list(range(0, 60, 3))


def test_empty_inputs():
    nodes, edges = _gdb13()
    s = _new_set(13, 8, 3, 8)
    got = s.add(nodes[:0], edges[:0])
    assert got.ids.shape == (0,) and len(s) == 0
    Z = np.zeros((3, 13, 8), np.int8), np.zeros((3, 13, 13, 3), np.int8)
    X, E = np.concatenate([Z[0], nodes[:2]]), np.concatenate([Z[1], edges[:2]])
    ref = MS.MoleculeSet()
    _assert_identity(s.add(X, E), ref.add(X, E))
    _assert_entries(s, ref)
    assert s.add(X[:1], E[:1]).ids.cpu().tolist() == [0] and s.counts.cpu().tolist()[0] == 4


# ---------------------------------------------------------------------------------------------------------------------
# 8. buffers
# ---------------------------------------------------------------------------------------------------------------------
def test_guarded_buffers():
    """gib_molset_identify on poisoned, guard-banded set and workspace buffers: nothing is written outside them, and
    two inserting calls and a lookup give the Python entry point's results"""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import PP_STATUS_INTS, MolSet, check, lib
    nodes, edges = _gdb13()
    X, E = _shuffled(np.concatenate([nodes[:300], nodes[100:200]]), np.concatenate([edges[:300], edges[100:200]]), 4)
    M, N, F = X.shape
    Ef = E.shape[3]
    want = _new_set(N, F, Ef, 400)
    w1, w2 = want.add(X[:250], E[:250]), want.add(X[250:], E[250:])
    C = 400
    d = PP._pp_dims(N, F, Ef, GDB13)
    slots = lib.gib_molset_slots(C)
    bufs = [Guarded(C * N * F), Guarded(C * N * N * Ef), Guarded(8 * C), Guarded(4 * C), Guarded(4 * C),
            Guarded(8 * C), Guarded(4 * C), Guarded(8 * slots), Guarded(4 * slots), Guarded(4)]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    mset = MolSet(*(g.ptr() for g in bufs), C, slots)
    check(lib.gib_molset_init(ctypes.byref(mset), st), "gib_molset_init")
    status = Guarded(4 * PP_STATUS_INTS)
    outs = []
    for a, b, insert in ((0, 250, 1), (250, M, 1), (0, M, 0)):
        n = b - a
        x, e = Guarded.like(torch.from_numpy(X[a:b]).cuda()), Guarded.like(torch.from_numpy(E[a:b]).cuda())
        ids, new, first = Guarded(4 * n), Guarded(n), Guarded(n)
        ws = Guarded(lib.gib_molset_ws_bytes(ctypes.byref(d), n))
        check(lib.gib_molset_identify(ctypes.byref(d), ctypes.byref(mset), x.ptr(), e.ptr(), None, n, insert, 1 << 20,
                                      ids.ptr(), new.ptr(), first.ptr(), ws.ptr(), status.ptr(), st),
              "gib_molset_identify")
        torch.cuda.synchronize()
        for g in (x, e, ids, new, first, ws, status):
            assert g.intact(), g.damage()
        assert status.view(torch.int32, (PP_STATUS_INTS,)).cpu().numpy()[3] == 0
        outs.append((ids.view(torch.int32, (n,)).cpu().numpy(), new.view(torch.uint8, (n,)).cpu().numpy(),
                     first.view(torch.uint8, (n,)).cpu().numpy()))
    for g in bufs:
        assert g.intact(), g.damage()
    for got, ref in zip(outs[:2], (w1, w2)):
        for u, v in zip(got, _host(ref)):
            assert np.array_equal(u.astype(v.dtype), v)
    assert np.array_equal(outs[2][0], np.concatenate([w1.ids.cpu().numpy(), w2.ids.cpu().numpy()]))
    S = len(want)
    assert bufs[9].view(torch.int32, (1,)).item() == S
    assert np.array_equal(bufs[0].view(torch.int8, (C, N, F))[:S].cpu().numpy(), want.entries()[0].cpu().numpy())
    assert np.array_equal(bufs[1].view(torch.int8, (C, N, N, Ef))[:S].cpu().numpy(), want.entries()[1].cpu().numpy())
    assert np.array_equal(bufs[5].view(torch.int64, (C,))[:S].cpu().numpy(), want.counts.cpu().numpy())
