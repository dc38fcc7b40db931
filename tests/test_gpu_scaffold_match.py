"""GPU: the scaffold-first decoding order (graphinvent_b200.preprocess.scaffold_first, `gib_scaffold_first` in
csrc/preprocess.cu) against its restatement (tests/scaffold_match_reference.py), byte for byte: stacks, order, ids.

  1. gdb13_1K/train with its atoms shuffled, scaffolds cut from molecules' k-atom prefixes (k = 1, 3, 5, 8), in both
     id modes; `order` applied to the input reproduces the output stacks;
  2. adversarial cases: symmetric scaffolds (rings, stars), a scaffold equal to the whole molecule, an extra bond among
     the image, a different bond type, protected atoms carrying a decoration, molecules smaller than the scaffold,
     N = 127 with attachment points and N = 181 without;
  3. the budget: a path scaffold absent from a ladder of identical atoms names its molecule at a small budget and
     equals the restatement at a large one; the kernel's node count equals the restatement's to the node; the
     refusals, and a molecule the input checks refuse is left alone (zero outputs, id -1, no flag of the search);
  4. poisoned, guard-banded outputs; identical results across chunk sizes and for host and device input;
  5. end to end: RouteScorer.score(..., scaffold_ids=ids) on the output plans every molecule (no NOT_PREFIX, no
     MASKED), its likelihoods are finite and equal the scores of the restated bytes;
  6. GraphedGenerator's decorations of a table ordered larger scaffolds first, with and without attachment points,
     shuffled and searched: the output equals the restatement and each molecule comes back with its own scaffold's
     id unless an earlier scaffold of the table embeds in it too.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests import scaffold_match_reference as SM
from tests import scaffold_route_reference as SR
from tests.conftest import GOLDEN
from tests.guarded import Guarded
from tests.test_scaffold_match_host import LAYOUTS, ladder, path_scaffold, search_nodes

pytestmark = pytest.mark.gpu

GDB13 = LAYOUTS["gdb13"]


def _gdb13(M=None):
    import os
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"][:M], z["gdb13_1K_train/edges"][:M]


def _shuffled(nodes, edges, seed):
    rng = np.random.default_rng(seed)
    pairs = [SM.shuffle(nodes[m], edges[m], rng) for m in range(nodes.shape[0])]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def _run(nodes, edges, sn, se, layout, protect=None, ids=None, seed=5, epoch=2, **kw):
    """device output and restatement, both as numpy"""
    from graphinvent_b200 import preprocess as PP
    attach = None
    if protect is not None:
        attach = [np.flatnonzero(~protect[s, :SM.n_atoms(sn[s])]).tolist() for s in range(sn.shape[0])]
    out = PP.scaffold_first(nodes, edges, (sn, se), attach, ids, seed=seed, epoch=epoch, layout=layout, **kw)
    out = [t.cpu().numpy() for t in out]
    n_at = [SM.n_atoms(x) for x in np.asarray(nodes)]
    rk = PP.rankings(n_at, nodes.shape[1], seed=seed, epoch=epoch).cpu().numpy()
    ref = SM.scaffold_first(np.asarray(nodes), np.asarray(edges), sn, se, rk, protect, ids,
                            kw.get("budget", 1 << 20))
    return out, ref


def _assert_equal(out, ref):
    on, oe, order, ids = out
    rn, re_, rorder, rids, status = ref
    assert status == (0, SM.NO_MOLECULE)
    assert np.array_equal(ids, rids)
    assert np.array_equal(order, rorder)
    assert np.array_equal(on, rn) and np.array_equal(oe, re_)


def _protect(sn, rng, p=0.5):
    k = [SM.n_atoms(x) for x in sn]
    return (np.arange(sn.shape[1])[None] < np.array(k)[:, None]) & (rng.random(sn.shape[:2]) < p)


# ---------------------------------------------------------------------------------------------------------------------
# 1. gdb13
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["ids", "search"])
@pytest.mark.parametrize("k", [1, 3, 5, 8])
def test_gdb13_prefix_scaffolds(k, mode):
    nodes, edges = _gdb13(None if mode == "ids" else 300)
    M = nodes.shape[0]
    ks = np.array([min(k, SM.n_atoms(nodes[m])) for m in range(M)])
    if mode == "ids":
        sn, se = SR.prefix_scaffolds(nodes, edges, ks)
        rng = np.random.default_rng(k)
        ids = np.arange(M)
        ids[rng.random(M) < 0.1] = -1
        other = rng.random(M) < 0.2                       # another molecule's scaffold: often no embedding
        ids[other] = rng.integers(0, M, int(other.sum()))
    else:
        pick = np.flatnonzero(ks == k)[:20] if (ks == k).any() else np.arange(20)
        sn, se = SR.prefix_scaffolds(nodes[pick], edges[pick], ks[pick])
        ids = None
    X, E = _shuffled(nodes, edges, seed=k)
    out, ref = _run(X, E, sn, se, GDB13, ids=ids)
    _assert_equal(out, ref)
    on, oe, order, got = out
    assert (got >= 0).sum() >= M // 10
    for m in range(M):                                    # order applied to the input reproduces the output
        n = SM.n_atoms(X[m])
        Xr, Er = SM.reorder(X[m], E[m], order[m, :n])
        assert np.array_equal(Xr, on[m]) and np.array_equal(Er, oe[m]), m


# ---------------------------------------------------------------------------------------------------------------------
# 2. adversarial cases
# ---------------------------------------------------------------------------------------------------------------------
def _graph(n, N, bonds, types=None, Ef=3, F=8):
    """atoms of type types[i] (default 0, uncharged) and bonds [(a, b, t)]"""
    X = np.zeros((N, F), np.int8)
    E = np.zeros((N, N, Ef), np.int8)
    for i in range(n):
        X[i, 0 if types is None else types[i]] = 1
        X[i, 5] = 1
    for a, b, t in bonds:
        E[a, b, t] = E[b, a, t] = 1
    return X, E


def _ring(n, start=0, t=0):
    return [(start + i, start + (i + 1) % n, t) for i in range(n)]


def _adversarial(N=16):
    ring6 = _graph(6, N, _ring(6))
    star = _graph(5, N, [(0, i, 0) for i in range(1, 5)])
    path3 = _graph(3, N, [(0, 1, 0), (1, 2, 0)])
    double_path3 = _graph(3, N, [(0, 1, 1), (1, 2, 1)])
    scaffolds = [ring6, star, path3, double_path3]
    mols = [
        _graph(10, N, _ring(6) + [(5, 6, 0), (6, 7, 0), (7, 8, 0), (8, 9, 0), (9, 4, 0)]),    # fused rings
        _graph(9, N, [(0, i, 0) for i in range(1, 9)]),                                        # a big star
        _graph(6, N, _ring(6)),                                                                # the whole molecule
        _graph(3, N, _ring(3)),                                                                # a triangle: induced?
        _graph(3, N, [(0, 1, 1), (1, 2, 1)]),                                                  # another bond type
        _graph(4, N, [(0, 1, 1), (1, 2, 1), (2, 3, 0)]),                                       # decorated path
        _graph(2, N, [(0, 1, 0)]),                                                             # fewer atoms
        _graph(1, N, []),
        _graph(8, N, [(0, 1, 0), (1, 2, 0), (2, 3, 0), (3, 4, 0), (4, 5, 0), (5, 6, 0), (6, 7, 0)],
               types=[0, 1, 0, 0, 0, 0, 1, 0]),
    ]
    sn, se = np.stack([s[0] for s in scaffolds]), np.stack([s[1] for s in scaffolds])
    return np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols]), sn, se


@pytest.mark.parametrize("attachment", [False, True], ids=["free", "attachment"])
@pytest.mark.parametrize("mode", ["ids", "search"])
def test_adversarial(mode, attachment):
    nodes, edges, sn, se = _adversarial()
    X, E = _shuffled(nodes, edges, seed=1)
    protect = _protect(sn, np.random.default_rng(2), 0.6) if attachment else None
    ids = None
    if mode == "ids":
        ids = np.array([0, 1, 0, 2, 2, 3, 0, 1, 2])
    out, ref = _run(X, E, sn, se, GDB13, protect, ids)
    _assert_equal(out, ref)
    if mode == "ids" and not attachment:
        # ring in fused rings, star in star, ring as the whole molecule; no path3 in a triangle (an extra bond among
        # the image) nor in a path of double bonds (another type); molecules smaller than their scaffold: none
        assert out[3].tolist() == [0, 1, 0, -1, -1, 3, -1, -1, 2]


@pytest.mark.parametrize("N, attachment", [(127, True), (181, False)])
def test_large_n(N, attachment):
    rng = np.random.default_rng(N)
    layout = LAYOUTS["gdb13"]
    mols = [SM.random_molecule(rng, int(n), N, layout, 1, n_types=2) for n in (N, N - 3, 90, 40, 7)]
    sc = [SM.cut_scaffold(*mols[i % 3], k, rng) for i, k in enumerate((3, 6, 12, 30))]
    mols = [SM.shuffle(x, e, rng) for x, e in mols]
    nodes, edges = np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])
    sn, se = np.stack([s[0] for s in sc]), np.stack([s[1] for s in sc])
    protect = _protect(sn, rng, 0.3) if attachment else None
    for ids in (None, np.array([3, 2, 1, 0, 0])):
        out, ref = _run(nodes, edges, sn, se, layout, protect, ids)
        _assert_equal(out, ref)


def test_molecule_decorated_at_a_protected_atom_is_not_matched_there():
    """the scaffold (path a-b, both protected except b) occurs twice; the first occurrence carries a decoration on a,
    so the embedding is the second one"""
    N = 12
    X, E = _graph(6, N, [(0, 1, 0), (0, 2, 0), (2, 3, 0), (3, 4, 0), (4, 5, 0)], types=[1, 0, 0, 0, 0, 1])
    SX, SE = _graph(2, N, [(0, 1, 0)], types=[1, 0])
    protect = np.zeros((1, N), bool)
    protect[0, 0] = True
    out, ref = _run(X[None], E[None], SX[None], SE[None], GDB13, protect)
    _assert_equal(out, ref)
    assert out[2][0, :2].tolist() == [5, 4]
    free, ref = _run(X[None], E[None], SX[None], SE[None], GDB13)
    assert free[2][0, :2].tolist() == [0, 1]


# ---------------------------------------------------------------------------------------------------------------------
# 3. the budget
# ---------------------------------------------------------------------------------------------------------------------
def test_budget():
    from graphinvent_b200 import preprocess as PP
    N = 24
    small = _graph(3, N, [(0, 1, 0), (1, 2, 0)], Ef=1)
    lad = ladder(12, N)
    nodes = np.stack([small[0]] * 3 + [lad[0], small[0]])
    edges = np.stack([small[1]] * 3 + [lad[1], small[1]])
    SX, SE = path_scaffold(14, N)
    with pytest.raises(ValueError, match=r"molecule 3 .*budget"):
        PP.scaffold_first(nodes, edges, (SX[None], SE[None]), layout=GDB13, budget=200)
    out, ref = _run(nodes, edges, SX[None], SE[None], GDB13)
    _assert_equal(out, ref)
    # the kernel counts search-tree nodes as the restatement does: exactly the restated count is enough, one less
    # is not -- for a search that exhausts and for one that finds its embedding at its last node
    SX2 = SX.copy()
    SX2[13] = SX2[12]
    for sx in (SX, SX2):
        count = search_nodes(lad[0], lad[1], sx, SE)
        out, ref = _run(nodes, edges, sx[None], SE[None], GDB13, budget=count)
        _assert_equal(out, ref)
        with pytest.raises(ValueError, match=r"molecule 3 .*budget"):
            PP.scaffold_first(nodes, edges, (sx[None], SE[None]), layout=GDB13, budget=count - 1)
    assert out[3][3] == 0


def test_refusals():
    from graphinvent_b200 import preprocess as PP
    nodes, edges, sn, se = _adversarial()
    with pytest.raises(ValueError, match="molecule 2: scaffold id 4"):
        PP.scaffold_first(nodes, edges, (sn, se), scaffold_ids=[0, 0, 4, 0, 0, 0, 0, 0, 0], layout=GDB13)
    lone = edges.copy()
    lone[0, 9], lone[0, :, 9] = 0, 0                      # atom 9 of the fused rings loses both its bonds
    with pytest.raises(ValueError, match="molecule 0 .*disconnected"):
        PP.scaffold_first(nodes, lone, (sn, se), layout=GDB13)
    asym = edges.copy()
    asym[6, 0, 1, 0] = 0
    with pytest.raises(ValueError, match="molecule 6 "):
        PP.scaffold_first(nodes, asym, (sn, se), layout=GDB13)
    rk = np.zeros((nodes.shape[0], nodes.shape[1]), np.int32)
    with pytest.raises(ValueError, match="molecule 0 .*permutation"):
        PP.scaffold_first(nodes, edges, (sn, se), rankings=rk, layout=GDB13)


def test_molecules_the_input_checks_refuse_are_left_alone():
    """through the C-ABI (the Python entry point raises first): a molecule pp_count refuses is not searched -- its
    order is -1, its stacks zero, its id -1, and it raises no flag of the search -- while the others are unaffected"""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import PP_BAD_EDGES
    X, E, sn, se = _gdb13_case(32)
    want = [t.cpu().numpy() for t in PP.scaffold_first(X, E, (sn, se), seed=9, epoch=1, layout=GDB13)]
    assert want[3][5] >= 0
    bad = E.copy()
    a, b = np.argwhere(bad[5].any(-1))[0]
    bad[5, a, b] = 0                                       # one half of a bond: asymmetric edges
    got, status = _raw_call(X, bad, sn, se)
    assert status[3] == PP_BAD_EDGES and status[4] == 5
    for w, g in zip(want, got):
        keep = np.arange(X.shape[0]) != 5
        assert np.array_equal(w[keep], g[keep])
    assert (got[0][5] == 0).all() and (got[1][5] == 0).all() and (got[2][5] == -1).all() and got[3][5] == -1


# ---------------------------------------------------------------------------------------------------------------------
# 4. buffers, chunks, host and device input
# ---------------------------------------------------------------------------------------------------------------------
def _gdb13_case(M, k=3, S=8, seed=3):
    nodes, edges = _gdb13(M)
    sn, se = SR.prefix_scaffolds(nodes[:S], edges[:S], [min(k, SM.n_atoms(x)) for x in nodes[:S]])
    X, E = _shuffled(nodes, edges, seed)
    return X, E, sn, se


def _raw_call(X, E, sn, se, seed=9, epoch=1):
    """gib_scaffold_first on guard-banded, poisoned buffers (draw mode); every band is checked.  Returns the outputs
    (nodes, edges, order, ids) as numpy and the status words"""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200._lib import PP_STATUS_INTS, check, lib
    from graphinvent_b200.generation import ScaffoldTable
    M, N, F = X.shape
    Ef = E.shape[3]
    table = ScaffoldTable(sn, se, None, N, F, Ef, GDB13, "cuda")
    d = PP._pp_dims(N, F, Ef, GDB13)
    x, e = Guarded.like(torch.from_numpy(X).cuda()), Guarded.like(torch.from_numpy(E).cuda())
    on, oe = Guarded(M * N * F), Guarded(M * N * N * Ef)
    order, ids, rk = Guarded(4 * M * N), Guarded(4 * M), Guarded(4 * M * N)
    ws = Guarded(lib.gib_scaffold_first_ws_bytes(ctypes.byref(d), M, table.S))
    st = Guarded(4 * PP_STATUS_INTS)
    sc = table.struct()
    check(lib.gib_scaffold_first(ctypes.byref(d), x.ptr(), e.ptr(), M, ctypes.byref(sc), None, 1,
                                 ctypes.c_ulonglong(seed), epoch, 0, rk.ptr(), 1 << 20, order.ptr(), ids.ptr(),
                                 on.ptr(), oe.ptr(), ws.ptr(), st.ptr(),
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "gib_scaffold_first")
    torch.cuda.synchronize()
    for g in (x, e, on, oe, order, ids, rk, ws, st):
        assert g.intact(), g.damage()
    n_at = [SM.n_atoms(r) for r in X]
    assert np.array_equal(rk.view(torch.int32, (M, N)).cpu().numpy(),
                          PP.rankings(n_at, N, seed=seed, epoch=epoch).cpu().numpy())
    out = (on.view(torch.int8, (M, N, F)).cpu().numpy(), oe.view(torch.int8, (M, N, N, Ef)).cpu().numpy(),
           order.view(torch.int32, (M, N)).cpu().numpy(), ids.view(torch.int32, (M,)).cpu().numpy())
    return out, st.view(torch.int32, (PP_STATUS_INTS,)).cpu().numpy()


def test_guarded_outputs():
    from graphinvent_b200 import preprocess as PP
    X, E, sn, se = _gdb13_case(64)
    want = [t.cpu().numpy() for t in PP.scaffold_first(X, E, (sn, se), seed=9, epoch=1, layout=GDB13)]
    got, status = _raw_call(X, E, sn, se)
    for w, g in zip(want, got):
        assert np.array_equal(w, g)
    assert status[3] == 0 and status[4] == SM.NO_MOLECULE


def test_chunks_and_device_input():
    from graphinvent_b200 import preprocess as PP
    X, E, sn, se = _gdb13_case(200, k=4, S=10)
    a = PP.scaffold_first(X, E, (sn, se), seed=3, epoch=4, layout=GDB13, chunk_molecules=1000)
    b = PP.scaffold_first(torch.from_numpy(X).cuda(), torch.from_numpy(E).cuda(), (sn, se), seed=3, epoch=4,
                          layout=GDB13, chunk_molecules=7)
    rk = PP.rankings([SM.n_atoms(r) for r in X], X.shape[1], seed=3, epoch=4)
    c = PP.scaffold_first(X, E, (sn, se), rankings=rk, layout=GDB13, chunk_molecules=64)
    for u, v, w in zip(a, b, c):
        assert torch.equal(u, v) and torch.equal(u, w)
    assert (a[3] >= 0).any()


# ---------------------------------------------------------------------------------------------------------------------
# 5. end to end
# ---------------------------------------------------------------------------------------------------------------------
def test_route_scorer_end_to_end():
    """search mode over prefix scaffolds with their decoration points as attachment points, then every atom row of
    the set as a one-atom scaffold (all an attachment point) so that every molecule embeds one"""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200.generation import ScaffoldTable
    from graphinvent_b200.graphed import RouteScorer
    from tests.test_gpu_route_nll import GDB13 as GDB13_KW
    from tests.test_gpu_route_nll import _net
    nodes, edges = _gdb13(96)
    rng = np.random.default_rng(4)
    S = 24
    ks = np.array([rng.integers(2, SM.n_atoms(nodes[m]) + 1) for m in range(S)])
    sn, se = SR.prefix_scaffolds(nodes[:S], edges[:S], ks)
    attach = [SR.decoration_points(nodes[m], edges[m], int(ks[m])) for m in range(S)]
    rows = np.unique(nodes.reshape(-1, nodes.shape[2]), axis=0)
    rows = rows[rows.any(1)]
    one_n = np.zeros((rows.shape[0],) + sn.shape[1:], np.int8)
    one_n[:, 0] = rows
    sn = np.concatenate([sn, one_n])
    se = np.concatenate([se, np.zeros((rows.shape[0],) + se.shape[1:], np.int8)])
    attach += [[0]] * rows.shape[0]
    X, E = _shuffled(nodes, edges, seed=6)
    N, F, Ef = X.shape[1], X.shape[2], E.shape[3]
    table = ScaffoldTable(sn, se, attach, N, F, Ef, GDB13, "cuda")
    on, oe, order, ids = PP.scaffold_first(X, E, table, seed=2, epoch=7, layout=GDB13)
    assert (ids >= 0).all() and (ids < S).sum() >= 24
    rk = PP.rankings([SM.n_atoms(r) for r in X], N, seed=2, epoch=7).cpu().numpy()
    rn, re_, _, rids, status = SM.scaffold_first(X, E, sn, se, rk, table.protect_mask)
    assert status[0] == 0 and np.array_equal(ids.cpu().numpy(), rids)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 64, scaffolds=(sn, se), attachment=attach, **GDB13_KW)
    out = scorer.score(on.cpu().numpy(), oe.cpu().numpy(), scaffold_ids=ids.cpu().numpy())
    assert torch.isfinite(out.likelihoods).all() and torch.isfinite(out.nll).all()
    again = scorer.score(rn, re_, scaffold_ids=rids)
    assert torch.equal(out.likelihoods, again.likelihoods) and torch.equal(out.nll, again.nll)


# ---------------------------------------------------------------------------------------------------------------------
# 6. the generator's own decorations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["free", "attachment"])
def test_generator_decorations_come_back_with_their_scaffold(masked):
    """GraphedGenerator decorates a table ordered larger scaffolds first; its molecules, atoms shuffled, go through
    the search.  The output equals the restatement.  A molecule that begins with its generating scaffold s (with
    attachment points every one does: the mask closes bonds among scaffold atoms) gets an id <= s, and exactly s
    unless an earlier scaffold of the table embeds in it too (the search takes the first that embeds).  Without
    attachment points the generator may bond two scaffold atoms to each other; scaffold s then no longer embeds as
    an induced subgraph and the restatement decides.  With the generating ids given, every molecule that begins
    with its scaffold gets that id."""
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200.generation import ScaffoldTable
    from graphinvent_b200.graphed import GraphedGenerator
    from tests.test_gpu_scaffold_generation import _gdb13_constants, attachment_lists, gdb13_scaffolds
    from tests.test_gpu_generation_layouts import _seeded_model
    sn, se = gdb13_scaffolds(sizes=(9, 6, 4, 2, 1))
    att = attachment_lists(sn) if masked else None
    C = _gdb13_constants()
    net, _ = _seeded_model("GGNN", C, 11)
    net.eval()
    B = 300
    gen = GraphedGenerator(net, B, constants=C, scaffolds=(sn, se), attachment=att, action_mask="structure")
    got = gen.build_graphs(uniforms=torch.rand(26, B, generator=torch.Generator(device="cuda").manual_seed(3),
                                               device="cuda"))
    n = min(got, B)
    keep = (gen.properly_terminated[:n].cpu().numpy() != 0) & (gen.generated_n_nodes[:n].cpu().numpy() > 0)
    nodes = gen.generated_nodes[:n].to(torch.int8).cpu().numpy()[keep]
    edges = gen.generated_edges[:n].to(torch.int8).cpu().numpy()[keep]
    gen_ids = gen.generated_scaffolds[:n].cpu().numpy()[keep].astype(np.int64)
    M = nodes.shape[0]
    assert M >= B // 2 and len(set(gen_ids.tolist())) == sn.shape[0]
    table = ScaffoldTable(sn, se, att, 13, 8, 3, GDB13, "cuda")
    protect = table.protect_mask
    k = [SM.n_atoms(x) for x in sn]
    begins = np.array([all(np.array_equal(a, b) for a, b in zip(SR.prefix(nodes[m], edges[m], k[s]), (sn[s], se[s])))
                       for m, s in enumerate(gen_ids)])
    if masked:
        assert begins.all()
    X, E = _shuffled(nodes, edges, seed=4)
    for ids_in in (None, gen_ids):
        out, ref = _run(X, E, sn, se, GDB13, protect, ids_in)
        _assert_equal(out, ref)
        ids = out[3]
        if ids_in is not None:
            assert (ids[begins] == gen_ids[begins]).all()
            continue
        assert (ids[begins] >= 0).all() and (ids[begins] <= gen_ids[begins]).all()
        earlier = np.array([any(SM.choose(X[m], E[m], sn, se, protect, t)[0] == "found" for t in range(s))
                            for m, s in enumerate(gen_ids)])
        own = begins & ~earlier
        assert (ids[own] == gen_ids[own]).all()
        assert own.sum() >= M // 2, (own.sum(), M)
