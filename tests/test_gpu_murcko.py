"""GPU: the Murcko scaffolds (graphinvent_b200.preprocess.murcko_scaffolds, `gib_murcko` in csrc/preprocess.cu)
against their restatement (tests/murcko_reference.py), bit for bit: keep, table bytes, ids, counts, attachment.

  1. gdb13_1K/train; the four action layouts x Ef 1-4 on random ring-rich molecules at N = 38; N = 127 and 181;
  2. every molecule's atoms shuffled: the same ids and counts;
  3. the 1-WL collision: decalin, bicyclopentyl and shuffled copies of both, interleaved, make two entries;
  4. chunking and `known=` over pieces equal one call; against a training table, its molecules keep their ids;
  5. end to end on gdb13_1K/train: scaffold_first with the table and ids returns the ids and begins every molecule
     with its entry, RouteScorer scores the decorations, GraphedGenerator takes the table;
  6. refusals (a disconnected molecule, a bad node row, a tiny budget), M = 0, no ring at all, guard-banded buffers.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import murcko_reference as MR
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


def _device(nodes, edges, layout, **kw):
    from graphinvent_b200 import preprocess as PP
    sc = PP.murcko_scaffolds(nodes, edges, layout=layout, **kw)
    return PP.Murcko(*(t.cpu().numpy() for t in sc))


def _assert_equal(sc, ref):
    table, ids, keep, status = ref
    assert status == (0, SM.NO_MOLECULE)
    assert np.array_equal(sc.keep, keep)
    assert np.array_equal(sc.ids, ids)
    if table is None:
        assert sc.nodes.shape[0] == 0 and sc.counts.shape == (0,)
        return
    assert sc.nodes.shape[0] == table[0].shape[0]
    for got, want in zip((sc.nodes, sc.edges, sc.counts, sc.attachment), table):
        assert np.array_equal(got, want)


def _check(nodes, edges, layout, **kw):
    sc = _device(nodes, edges, layout, **kw)
    _assert_equal(sc, MR.murcko(nodes, edges, budget=kw.get("budget", 1 << 20)))
    return sc


# ---------------------------------------------------------------------------------------------------------------------
# 1. against the restatement
# ---------------------------------------------------------------------------------------------------------------------
def test_gdb13():
    nodes, edges = _gdb13()
    sc = _check(nodes, edges, GDB13)
    assert 20 < sc.nodes.shape[0] < (sc.ids >= 0).sum() and (sc.ids < 0).any()
    assert sc.attachment.any()


@pytest.mark.parametrize("Ef", [1, 2, 3, 4])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts(layout, Ef):
    rng = np.random.default_rng(10 * list(LAYOUTS).index(layout) + Ef)
    nodes, edges = ring_rich(rng, 48, 38, LAYOUTS[layout], Ef, hi=20)
    X2, E2 = _shuffled(nodes[:16], edges[:16], 1)          # repeats: every one joins its original's entry
    nodes, edges = np.concatenate([nodes, X2]), np.concatenate([edges, E2])
    sc = _check(nodes, edges, LAYOUTS[layout])
    assert (sc.counts >= 2).any()


@pytest.mark.parametrize("N", [127, 181])
def test_large_n(N):
    rng = np.random.default_rng(N)
    nodes, edges = ring_rich(rng, 4, N, GDB13, 1, lo=N - 40)
    X2, E2 = _shuffled(nodes, edges, 2)
    sc = _check(np.concatenate([nodes, X2]), np.concatenate([edges, E2]), GDB13)
    assert sc.ids[:4].tolist() == sc.ids[4:].tolist()


# ---------------------------------------------------------------------------------------------------------------------
# 2-3. invariance, the collision path
# ---------------------------------------------------------------------------------------------------------------------
def test_shuffle_invariance():
    nodes, edges = _gdb13()
    a = _device(nodes, edges, GDB13)
    b = _device(*_shuffled(nodes, edges, 7), GDB13)
    assert np.array_equal(a.ids, b.ids) and np.array_equal(a.counts, b.counts)
    rng = np.random.default_rng(11)
    X, E = ring_rich(rng, 64, 38, LAYOUTS["imp_H+chirality"], 3, hi=24)
    a = _device(X, E, LAYOUTS["imp_H+chirality"])
    b = _device(*_shuffled(X, E, 8), LAYOUTS["imp_H+chirality"])
    assert np.array_equal(a.ids, b.ids) and np.array_equal(a.counts, b.counts)


def test_wl_collision():
    (dX, dE), (bX, bE) = decalin_and_bicyclopentyl(N=16)
    assert MR.wl_hash(*MR.scaffold(dX, dE)[:2]) == MR.wl_hash(*MR.scaffold(bX, bE)[:2])    # they really collide
    rng = np.random.default_rng(3)
    mols = []
    for i in range(12):
        X, E = (dX, dE) if i % 2 else (bX, bE)
        mols.append(SM.shuffle(X, E, rng) if i > 1 else (X, E))
    nodes, edges = np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])
    sc = _check(nodes, edges, GDB13)
    assert sc.ids.tolist() == [0, 1] * 6 and sc.counts.tolist() == [6, 6]


# ---------------------------------------------------------------------------------------------------------------------
# 4. chunks, known tables, novelty
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_and_known():
    from graphinvent_b200 import preprocess as PP
    nodes, edges = _gdb13()
    whole = _device(nodes, edges, GDB13)
    small = _device(torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda(), GDB13, chunk_molecules=37)
    for u, v in zip(whole, small):
        assert np.array_equal(u, v)
    sc, ids = None, []
    for a, b in ((0, 100), (100, 101), (101, 640), (640, nodes.shape[0])):
        sc = PP.murcko_scaffolds(nodes[a:b], edges[a:b], layout=GDB13, known=sc)
        ids.append(sc.ids.cpu().numpy())
    assert np.array_equal(np.concatenate(ids), whole.ids)
    for name in ("nodes", "edges", "counts", "attachment"):
        assert np.array_equal(getattr(sc, name).cpu().numpy(), getattr(whole, name))


def test_novelty_against_a_training_table():
    from graphinvent_b200 import preprocess as PP
    nodes, edges = _gdb13()
    train = PP.murcko_scaffolds(nodes[:600], edges[:600], layout=GDB13)
    S = train.nodes.shape[0]
    pick = np.r_[np.arange(0, 600, 7), np.arange(600, nodes.shape[0])]
    np.random.default_rng(0).shuffle(pick)
    X, E = _shuffled(nodes[pick], edges[pick], 5)
    gen = PP.murcko_scaffolds(X, E, layout=GDB13, known=train)
    ids = gen.ids.cpu().numpy()
    old = pick < 600
    assert np.array_equal(ids[old], train.ids.cpu().numpy()[pick[old]])
    kn = tuple(t.cpu().numpy() for t in (train.nodes, train.edges, train.counts, train.attachment))
    table, rids, _, status = MR.murcko(X, E, known=kn)
    assert status == (0, SM.NO_MOLECULE) and np.array_equal(ids, rids)
    for got, want in zip((gen.nodes, gen.edges, gen.counts, gen.attachment), table):
        assert np.array_equal(got.cpu().numpy(), want)
    novel = ids >= S
    assert novel.any() and (ids[old] < S).all()
    assert np.array_equal(gen.counts.cpu().numpy()[:S] - train.counts.cpu().numpy(),
                          np.bincount(ids[(ids >= 0) & ~novel], minlength=S))


# ---------------------------------------------------------------------------------------------------------------------
# 5. end to end
# ---------------------------------------------------------------------------------------------------------------------
def test_end_to_end_gdb13():
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator, RouteScorer
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    nodes, edges = _gdb13()          # decoding order: a molecule without a ring (id -1) is scored as it comes
    sc = PP.murcko_scaffolds(nodes, edges, layout=GDB13)
    on, oe, order, ids = PP.scaffold_first(nodes, edges, (sc.nodes, sc.edges), attachment=sc.attachment,
                                           scaffold_ids=sc.ids, layout=GDB13)
    assert torch.equal(ids, sc.ids)
    on_h, oe_h, ids_h = on.cpu().numpy(), oe.cpu().numpy(), ids.cpu().numpy()
    tn, te = sc.nodes.cpu().numpy(), sc.edges.cpu().numpy()
    for m in np.flatnonzero(ids_h >= 0):
        k = SM.n_atoms(tn[ids_h[m]])
        assert np.array_equal(on_h[m, :k], tn[ids_h[m], :k])
        assert np.array_equal(oe_h[m, :k, :k], te[ids_h[m], :k, :k])
    C = make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    net = net.cuda().eval()
    kw = dict(n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0)
    scorer = RouteScorer(net, 256, scaffolds=(sc.nodes, sc.edges), attachment=sc.attachment, **kw)
    out = scorer.score(on, oe, scaffold_ids=ids)
    assert torch.isfinite(out.nll).all() and torch.isfinite(out.likelihoods).all()
    gen = GraphedGenerator(net, 64, scaffolds=(sc.nodes, sc.edges), attachment=sc.attachment, **kw)
    assert gen.build_graphs() > 0


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals, empty inputs, buffers
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals():
    from graphinvent_b200 import preprocess as PP
    nodes, edges = _gdb13()
    nodes, edges = nodes[:40].copy(), edges[:40].copy()
    cut = edges.copy()
    n = SM.n_atoms(nodes[17])
    a = n - 1
    cut[17, a, :] = 0
    cut[17, :, a] = 0                                       # its last atom loses every bond
    with pytest.raises(ValueError, match="molecule 17 .*disconnected"):
        PP.murcko_scaffolds(nodes, cut, layout=GDB13)
    bad = nodes.copy()
    bad[23, 0, :5] = 1                                      # every atom type on one row
    with pytest.raises(ValueError, match="molecule 23 "):
        PP.murcko_scaffolds(bad, edges, layout=GDB13)
    (dX, dE), (bX, bE) = decalin_and_bicyclopentyl(N=13)
    with pytest.raises(ValueError, match="molecule 1 .*budget"):
        PP.murcko_scaffolds(np.stack([dX, dX]), np.stack([dE, dE]), layout=GDB13, budget=2)


def test_empty_and_acyclic():
    from graphinvent_b200 import preprocess as PP
    nodes, edges = _gdb13()
    sc = PP.murcko_scaffolds(nodes[:0], edges[:0], layout=GDB13)
    assert sc.nodes.shape == (0, 13, 8) and sc.edges.shape == (0, 13, 13, 3) and sc.ids.shape == (0,)
    assert sc.counts.shape == (0,) and sc.attachment.shape == (0, 13) and sc.keep.shape == (0, 13)
    acyclic = np.flatnonzero([not MR.keep_core(x, e).any() for x, e in zip(nodes, edges)])[:50]
    sc = _check(nodes[acyclic], edges[acyclic], GDB13)
    assert sc.nodes.shape[0] == 0 and (sc.ids == -1).all() and not sc.keep.any()


def test_guarded_buffers():
    """gib_murcko on poisoned, guard-banded buffers: nothing is written outside them and the results are the Python
    entry point's"""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import PP_STATUS_INTS, check, lib
    nodes, edges = _shuffled(*(t[:300] for t in _gdb13()), 4)
    want = _device(nodes, edges, GDB13)
    M, N, F = nodes.shape
    Ef = edges.shape[3]
    d = PP._pp_dims(N, F, Ef, GDB13)
    x, e = Guarded.like(torch.from_numpy(nodes).cuda()), Guarded.like(torch.from_numpy(edges).cuda())
    tn, te = Guarded(M * N * F), Guarded(M * N * N * Ef)
    counts, attach = Guarded(8 * M, fill="zero"), Guarded(M * N, fill="zero")
    keep, ids, st = Guarded(M * N), Guarded(4 * M), Guarded(4 * PP_STATUS_INTS)
    ws = Guarded(lib.gib_murcko_ws_bytes(ctypes.byref(d), M, 0))
    check(lib.gib_murcko(ctypes.byref(d), x.ptr(), e.ptr(), M, 0, tn.ptr(), te.ptr(), counts.ptr(), attach.ptr(),
                         1 << 20, keep.ptr(), ids.ptr(), ws.ptr(), st.ptr(),
                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "gib_murcko")
    torch.cuda.synchronize()
    for g in (x, e, tn, te, counts, attach, keep, ids, ws, st):
        assert g.intact(), g.damage()
    status = st.view(torch.int32, (PP_STATUS_INTS,)).cpu().numpy()
    S = int(status[5])
    assert status[3] == 0 and S == want.nodes.shape[0]
    assert np.array_equal(tn.view(torch.int8, (M, N, F)).cpu().numpy()[:S], want.nodes)
    assert np.array_equal(te.view(torch.int8, (M, N, N, Ef)).cpu().numpy()[:S], want.edges)
    assert np.array_equal(counts.view(torch.int64, (M,)).cpu().numpy()[:S], want.counts)
    assert np.array_equal(attach.view(torch.uint8, (M, N)).cpu().numpy()[:S].astype(bool), want.attachment)
    assert np.array_equal(keep.view(torch.uint8, (M, N)).cpu().numpy().astype(bool), want.keep)
    assert np.array_equal(ids.view(torch.int32, (M,)).cpu().numpy(), want.ids)
