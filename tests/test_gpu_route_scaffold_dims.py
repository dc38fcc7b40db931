"""GPU: the route-scorer and scaffold kernels across the dimensions they accept, not only gdb13's (N = 13, Ef = 3).

A. Kernel level through the C ABI on guard-banded, poisoned buffers, no model:
   - gib_route_plan / gib_route_fill and their _scaffold forms over N = 1 .. 181, Ef = 1 .. 4, the four action layouts
     (node and edge rows of many residues mod 16, rows shorter than 16 bytes), batches of 1, 7, 256 and 263 and
     chunks that split the molecules, against the restatements (tests/preprocess_reference.py,
     tests/scaffold_route_reference.py) byte for byte; scaffolds of 1 .. n atoms with attachment points in all four
     protect words; the GIB_ROUTE_MASKED / GIB_ROUTE_NOT_PREFIX refusals naming the first molecule;
   - gib_route_mask_logits and gib_generation_mask_logits (plain and round-gated) against mask_row, N up to 127;
   - gib_route_probs / gib_route_dlogits at apd 2 .. 52 201 against an fp64 softmax;
   - gib_route_reduce / gib_route_grad_coef on routes of 1 .. 16 292 states (one warp walks 32 states per pass).
B. The generator's round kernels, mask and start state with scaffolds of 1 .. N - 1 atoms at N = 38 / 90 / 127
   against the scaffold oracle bit for bit; the captured generator and a masked RL rollout plus backward at N = 38.
C. RouteScorer at (N = 38, Ef = 4, implicit H + chirality) and (N = 64, Ef = 1) against the fp64 restatements.

Molecules come from seeded builders (chains, stars, complete graphs, trees with ring bonds, single atoms), each a
valid decoding order: every atom i >= 1 bonds to some j < i."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R
from tests import scaffold_oracle as SO
from tests import scaffold_route_reference as SR
from tests.guarded import Guarded
from tests.test_gpu_preprocess import LAYOUTS
from tests.test_route_grad_host import coef_restated

pytestmark = pytest.mark.gpu

# the scaffold atoms whose protect bits sit at the edges of the four 32-bit words
WORD_EDGES = (0, 31, 32, 63, 64, 95, 96, 126)


# ---- molecule builders ---------------------------------------------------------------------------------------------
def molecule(n, N, segs, Ef, bonds, rng):
    """int8 nodes [N, F] (n atoms, a random one-hot per segment) and edges [N, N, Ef] with the bonds (i, j, type)"""
    X = np.zeros((N, sum(segs)), np.int8)
    for i in range(n):
        base = 0
        for w in segs:
            X[i, base + int(rng.integers(w))] = 1
            base += w
    E = np.zeros((N, N, Ef), np.int8)
    for i, j, t in bonds:
        E[i, j, t] = E[j, i, t] = 1
    return X, E


def chain(n, Ef, rng):
    return [(i - 1, i, int(rng.integers(Ef))) for i in range(1, n)]


def star(n, Ef, rng):
    return [(0, i, int(rng.integers(Ef))) for i in range(1, n)]


def complete(n, Ef, rng):
    return [(j, i, int(rng.integers(Ef))) for i in range(1, n) for j in range(i)]


def tree_with_rings(n, Ef, rng, p_ring=0.4):
    """atom i bonds to a random earlier atom, and with probability p_ring to a second one"""
    bonds = []
    for i in range(1, n):
        js = {int(rng.integers(i))}
        if i > 1 and rng.random() < p_ring:
            js.add(int(rng.integers(i)))
        bonds += [(j, i, int(rng.integers(Ef))) for j in sorted(js)]
    return bonds


def molecule_set(N, segs, Ef, seed, complete_atoms=48):
    """a single atom, a chain, a star and a tree of N atoms, a complete graph of min(N, complete_atoms) atoms and a
    tree of random size: int8 stacks [M, N, F] / [M, N, N, Ef]"""
    rng = np.random.default_rng(seed)
    specs = [(1, [])]
    if N > 1:
        specs += [(N, chain(N, Ef, rng)), (N, star(N, Ef, rng)), (N, tree_with_rings(N, Ef, rng))]
        nc = min(N, complete_atoms)
        specs += [(nc, complete(nc, Ef, rng))]
        n = int(rng.integers(2, N + 1))
        specs += [(n, tree_with_rings(n, Ef, rng))]
    specs += [(1, [])]
    mols = [molecule(n, N, segs, Ef, b, rng) for n, b in specs]
    return np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])


def layout_kw(layout):
    A, Fc, H, C = LAYOUTS[layout]
    return dict(n_atom_types=A, n_formal_charge=Fc, n_imp_H=H, n_chirality=C)


def segs_of(layout):
    return P.segments(*LAYOUTS[layout])


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _G(a):
    return Guarded.like(torch.from_numpy(np.ascontiguousarray(a)).cuda())


def _p(g):
    return ctypes.c_void_p(g.ptr()) if g is not None else None


def _i32(g, n):
    """the first n int32 words of a guarded buffer"""
    return g.view(torch.int32)[:n].cpu().numpy()


def attachment_points(nodes, edges, k, rng):
    """the decoration's own points (so its route is never masked), the word-edge atoms below k and a random third of
    the rest: every protect word holds both kinds of atom once k reaches it"""
    pts = set(SR.decoration_points(nodes, edges, k)) | {i for i in WORD_EDGES if i < k}
    pts |= {int(i) for i in np.flatnonzero(rng.random(k) < 0.33)}
    return sorted(pts)


# ---- A. plan + fill ------------------------------------------------------------------------------------------------
# (N, Ef, layout, batch, chunk): N*F mod 16 and N*N*Ef mod 16 over {8, 1}, {6, 12}, {12, 9}, {14, 2}, {4, 0}, {0, 0},
# {11, 3}, {12, 0}, {4, 2}, {0, 0}, {6, 9}
GRID = [(1, 1, "gdb13", 1, 1), (2, 3, "chirality", 1, 3), (13, 1, "imp_H", 7, 3), (33, 2, "imp_H+chirality", 256, 4),
        (38, 4, "imp_H+chirality", 263, 3), (64, 4, "gdb13", 256, 5), (65, 3, "chirality", 263, 2),
        (90, 4, "imp_H+chirality", 256, 4), (127, 2, "imp_H", 263, 3), (128, 2, "chirality", 256, 4),
        (181, 1, "imp_H+chirality", 263, 3)]
K_SIZES = (1, 31, 32, 33, 63, 64, 65, 96, 97)


class _MaskRows:
    """SR.state_masks of the states, row by row: mask_row depends on the atom count only through n - 1 < k, so each
    scaffold has two rows (the [S, apd] array would not fit at N = 90, Ef = 4)"""

    def __init__(self, sid, n_at, sn, protect, N, Ef, per_node):
        self.sid, self.n_at, self.sn, self.protect = sid, n_at, sn, protect
        self.args, self.rows = (N, Ef, per_node), {}
        self.apd = N * (per_node + Ef) + 1

    def __getitem__(self, idx):
        out = np.zeros((len(idx), self.apd), bool)
        for r, i in enumerate(idx):
            s = int(self.sid[i])
            if s < 0:
                continue
            k = P.n_atoms(self.sn[s])
            key = (s, int(self.n_at[i]) - 1 < k)
            if key not in self.rows:
                self.rows[key] = SR.mask_row(int(self.n_at[i]), k, self.protect[s], *self.args)
            out[r] = self.rows[key]
        return out


class _Route:
    """one dims case's guarded plan / fill buffers"""

    def __init__(self, N, Ef, layout, B, chunk):
        from graphinvent_b200._lib import PP_STATUS_INTS, PPDims, lib
        self.N, self.Ef, self.B, self.chunk, self.segs = N, Ef, B, chunk, segs_of(layout)
        self.F = sum(self.segs)
        self.d = PPDims(N=N, F=self.F, Ef=Ef, batch_size=B, **layout_kw(layout))
        self.bd = ctypes.byref(self.d)
        self.ws = Guarded(lib.gib_route_plan_ws_bytes(self.bd, chunk))
        self.off, self.status = Guarded(4 * (chunk + 1)), Guarded(4 * PP_STATUS_INTS)
        self.ctl, self.slots = Guarded(8), Guarded(8 * B)
        self.s_ids, self.s_n = Guarded(4 * B), Guarded(4 * B)
        self.on, self.oe = Guarded(B * N * self.F), Guarded(B * N * N * Ef)
        self.bufs = [self.ws, self.off, self.status, self.ctl, self.slots, self.s_ids, self.s_n, self.on, self.oe]
        self.replays = 0

    def plan(self, nodes, edges, ids=None, sc=None):
        """plans one chunk; returns the status words"""
        from graphinvent_b200._lib import PP_STATUS_INTS, check, lib
        M = nodes.shape[0]
        self.gn, self.ge = _G(nodes), _G(edges)
        self.gi = _G(ids.astype(np.int32)) if ids is not None else None
        self.bufs += [self.gn, self.ge] + ([self.gi] if ids is not None else [])
        if ids is None:
            check(lib.gib_route_plan(self.bd, _p(self.gn), _p(self.ge), M, self.chunk, _p(self.ws), _p(self.off),
                                     _p(self.status), _st()), "gib_route_plan")
        else:
            check(lib.gib_route_plan_scaffold(self.bd, _p(self.gn), _p(self.ge), M, self.chunk, ctypes.byref(sc),
                                              _p(self.gi), _p(self.ws), _p(self.off), _p(self.status), _st()),
                  "gib_route_plan_scaffold")
        return _i32(self.status, PP_STATUS_INTS)

    def fill(self):
        from graphinvent_b200._lib import check, lib
        if self.gi is None:
            check(lib.gib_route_fill(self.bd, _p(self.gn), _p(self.ge), self.chunk, _p(self.ws), _p(self.off),
                                     _p(self.status), _p(self.ctl), _p(self.slots), _p(self.on), _p(self.oe), _st()),
                  "gib_route_fill")
        else:
            check(lib.gib_route_fill_scaffold(self.bd, _p(self.gn), _p(self.ge), self.chunk, _p(self.ws), _p(self.off),
                                              _p(self.status), _p(self.gi), _p(self.ctl), _p(self.slots),
                                              _p(self.s_ids), _p(self.s_n), _p(self.on), _p(self.oe), _st()),
                  "gib_route_fill_scaffold")

    def next_round(self):
        from graphinvent_b200._lib import check, lib
        check(lib.gib_rl_next_round(ctypes.c_void_p(self.status.ptr() + 24), _st()), "gib_rl_next_round")

    def run_chunk(self, nodes, edges, ids=None, sn=None, table=None, protect=None):
        """plan + every fill replay of one chunk against the restatement: inputs byte for byte, slot actions, build
        order places, scaffold ids and atom counts exact, padding -1 / zero, offsets and S; with attachment points each
        replay's masked logits against state_masks.  Returns the number of states."""
        from graphinvent_b200._lib import check, lib
        N, F, Ef, B = self.N, self.F, self.Ef, self.B
        M = nodes.shape[0]
        if ids is None:
            X, E, acts, offsets = R.build_order_states(nodes, edges, self.segs)
            sid = n_at = None
        else:
            X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, self.segs)
        S = int(offsets[-1])
        sw = self.plan(nodes, edges, ids, table.struct() if table is not None else None)
        assert sw[3] == 0 and sw[5] == S and sw[6] == 0, sw
        if ids is not None:
            assert sw[1] == 0 and sw[2] == 2 ** 31 - 1, sw
        assert np.array_equal(_i32(self.off, M + 1), offsets)
        masks = None
        if protect is not None:
            per_node = int(np.prod(self.segs)) * Ef
            apd = N * (per_node + Ef) + 1
            masks = _MaskRows(sid, n_at, sn, protect, N, Ef, per_node)
            sc = table.struct()
            logits = Guarded.like(torch.randn(B, apd, device="cuda", generator=torch.Generator("cuda").manual_seed(S)))
            raw = logits.view().clone()
            self.bufs.append(logits)
        for r in range(-(-S // B)):
            self.fill()
            if masks is not None:
                logits.view().copy_(raw)
                check(lib.gib_route_mask_logits(B, N, Ef, apd, ctypes.byref(sc), _p(self.s_ids), _p(self.s_n),
                                                _p(logits), _st()), "gib_route_mask_logits")
            self.next_round()
            self.replays += 1
            live = min(B, S - r * B)
            assert _i32(self.ctl, 2)[0] == live                 # gib_batch_ctl.live
            sl = self.slots.view(torch.int32, (2, B)).cpu().numpy()
            dst = sl[1]
            # states in truncation order: state s0 + b of molecule m sits at off[m] + off[m + 1] - 1 - (s0 + b)
            mol = np.searchsorted(offsets, r * B + np.arange(live), side="right") - 1
            assert np.array_equal(dst[:live], offsets[mol] + offsets[mol + 1] - 1 - (r * B + np.arange(live))), r
            assert (dst[live:] == -1).all() and (sl[0][live:] == -1).all()
            assert np.array_equal(sl[0][:live], acts[dst[:live]])
            xn = self.on.view(torch.int8, (B, N, F)).cpu().numpy()
            xe = self.oe.view(torch.int8, (B, N, N, Ef)).cpu().numpy()
            assert np.array_equal(xn[:live], X[dst[:live]]), r
            assert np.array_equal(xe[:live], E[dst[:live]]), r
            assert not xn[live:].any() and not xe[live:].any()
            if ids is not None:
                si, sn_ = _i32(self.s_ids, B), _i32(self.s_n, B)
                assert np.array_equal(si[:live], sid[dst[:live]]) and (si[live:] == -1).all()
                want_n = np.where(sid[dst[:live]] >= 0, n_at[dst[:live]], -1)
                assert np.array_equal(sn_[:live], want_n) and (sn_[live:] == -1).all()
            if masks is not None:
                lg = logits.view().cpu()
                m = torch.from_numpy(masks[dst[:live]])
                assert torch.equal(torch.isinf(lg[:live]), m), r
                assert torch.equal(lg[:live][~m], raw[:live].cpu()[~m]) and torch.equal(lg[live:], raw[live:].cpu())
        return S

    def intact(self):
        torch.cuda.synchronize()
        for g in self.bufs:
            assert g.intact(), g.damage()


def _chunks(M, chunk):
    return [(a, min(a + chunk, M)) for a in range(0, M, chunk)]


def _conditional_set(nodes, edges, N, seed):
    """(molecule, k) pairs for k in K_SIZES, N - 1 and n (k = n leaves only terminate) with k <= n: the molecules
    repeated, scaffold j = pair j's k-atom prefix, every fifth id -1; and each pair's attachment points"""
    rng = np.random.default_rng(seed)
    pairs = []
    for m in range(nodes.shape[0]):
        n = P.n_atoms(nodes[m])
        pairs += [(m, k) for k in sorted(set(K_SIZES + (N - 1, n))) if 1 <= k <= n]
    idx = np.array([m for m, _ in pairs])
    ks = np.array([k for _, k in pairs])
    mn, me = nodes[idx], edges[idx]
    sn, se = SR.prefix_scaffolds(mn, me, ks)
    ids = np.arange(len(pairs))
    ids[::5] = -1
    attach = [attachment_points(mn[j], me[j], int(ks[j]), rng) for j in range(len(pairs))]
    return mn, me, sn, se, ids, attach


@pytest.mark.parametrize("N,Ef,layout,B,chunk", GRID, ids=[f"N{g[0]}-Ef{g[1]}-{g[2]}-B{g[3]}" for g in GRID])
def test_plan_and_fill_across_dims(N, Ef, layout, B, chunk):
    from graphinvent_b200.generation import ScaffoldTable
    nodes, edges = molecule_set(N, segs_of(layout), Ef, seed=N * 10 + Ef)
    M = nodes.shape[0]
    run = _Route(N, Ef, layout, B, chunk)
    total = 0
    for a, b in _chunks(M, chunk):
        total += run.run_chunk(nodes[a:b], edges[a:b])
    assert total == P.total_subgraphs(edges)
    # conditional: scaffolds of 1 .. n atoms, ids of -1 mixed in; attachment points while N <= 127
    mn, me, sn, se, ids, attach = _conditional_set(nodes, edges, N, seed=N)
    lay = LAYOUTS[layout]
    masked = N <= 127
    table = ScaffoldTable(sn, se, attach if masked else None, N, sum(lay), Ef, lay, "cuda")
    protect = SR.protect_of(sn, attach) if masked else None
    if masked:
        assert (table.protect_mask == protect).all()
    run = _Route(N, Ef, layout, B, chunk)
    for a, b in _chunks(mn.shape[0], chunk):
        run.run_chunk(mn[a:b], me[a:b], ids[a:b], sn, table, protect)
    run.intact()
    if not masked:
        with pytest.raises(ValueError, match="N <= 127"):
            ScaffoldTable(sn, se, attach, N, sum(lay), Ef, lay, "cuda")


def _route_states(nodes, edges, segs):
    """preprocess_reference.route one state at a time (truncation order), for routes too long to hold at once"""
    X, E = nodes.copy(), edges.copy()
    n = P.n_atoms(X)
    yield X.copy(), E.copy(), P.apd_length(E.shape[0], E.shape[2], segs) - 1
    for _ in range(int(E.sum()) // 2 + 1):
        a = P._apd_index(X, E, n, segs)
        n = P._truncate(X, E, n)
        yield X, E, a                                   # the caller copies what it keeps


def test_the_largest_route_plans_at_n_181():
    """a complete graph of 181 atoms (Ef = 1): s_max = 16 292 states, the first and last batches filled"""
    N, Ef, layout, B = 181, 1, "gdb13", 263
    rng = np.random.default_rng(5)
    X, E = molecule(N, N, segs_of(layout), Ef, complete(N, Ef, rng), rng)
    run = _Route(N, Ef, layout, B, 1)
    sw = run.plan(X[None], E[None])
    S = N * (N - 1) // 2 + 2
    assert sw[3] == 0 and sw[5] == S and _i32(run.off, 2).tolist() == [0, S]
    last = -(-S // B) - 1
    want = set(range(0, 2 * B)) | set(range(last * B, S))
    states = {i: (x.copy(), e.copy(), a) for i, (x, e, a) in enumerate(_route_states(X, E, segs_of(layout)))
              if i in want}
    for r in range(last + 1):
        run.fill()
        run.next_round()
        if r not in (0, 1, last):
            continue
        live = min(B, S - r * B)
        sl = run.slots.view(torch.int32, (2, B)).cpu().numpy()
        xn = run.on.view(torch.int8, (B, N, run.F)).cpu().numpy()
        xe = run.oe.view(torch.int8, (B, N, N, Ef)).cpu().numpy()
        for b in range(live):
            x, e, a = states[r * B + b]
            assert sl[0, b] == a and sl[1, b] == S - 1 - (r * B + b)
            assert np.array_equal(xn[b], x) and np.array_equal(xe[b], e), (r, b)
        assert not xn[live:].any() and not xe[live:].any() and (sl[:, live:] == -1).all()
    run.intact()


# ---- A. refusals at large N ----------------------------------------------------------------------------------------
def _chain_with(n, N, segs, Ef, extra, rng, skip=()):
    """a chain of n atoms whose bonds in `skip` are replaced by the (i, j) pairs of `extra`"""
    bonds = [(i, j, t) for i, j, t in chain(n, Ef, rng) if (i, j) not in skip] + [(i, j, 0) for i, j in extra]
    return molecule(n, N, segs, Ef, bonds, rng)


@pytest.mark.parametrize("N,Ef,layout", [(127, 2, "imp_H"), (128, 2, "chirality"), (181, 1, "gdb13")])
def test_refusals_name_the_first_molecule_at_large_n(N, Ef, layout):
    """GIB_ROUTE_MASKED (N = 127: the decoration bonds to protected atom 70 or 102 -- words 2 and 3 -- while atom
    6 = 70 mod 32 = 102 mod 32 is an attachment point) and GIB_ROUTE_NOT_PREFIX (an extra bond between scaffold atoms
    40 and 100, another atom type in row 100), each naming the first such molecule of the chunk"""
    from graphinvent_b200._lib import ROUTE_MASKED, ROUTE_NOT_PREFIX
    from graphinvent_b200.generation import ScaffoldTable
    rng = np.random.default_rng(N)
    segs = segs_of(layout)
    lay = LAYOUTS[layout]
    mols, scafs, attach = [], [], []

    def add(x, e, k, pts):
        mols.append((x, e))
        scafs.append(SR.prefix(x, e, k))
        attach.append(pts)

    for _ in range(3):                                   # valid decorations first
        x, e = _chain_with(120, N, segs, Ef, [], rng)
        add(x, e, 105, [6, 104])
    cases = {}
    if N <= 127:
        x, e = _chain_with(104, N, segs, Ef, [(70, 101)], rng, skip={(100, 101)})
        add(x, e, 101, [6, 38, 100])                     # atom 101 bonds to 70, protected
        cases["masked"] = len(mols) - 1
        x, e = _chain_with(115, N, segs, Ef, [(102, 111)], rng, skip={(110, 111)})
        add(x, e, 111, [6, 110])                          # a later one in word 3
    x, e = _chain_with(112, N, segs, Ef, [(40, 100)], rng)
    sx, se_ = SR.prefix(x, e, 110)
    se_[40, 100] = se_[100, 40] = 0                       # the scaffold lacks that bond
    mols.append((x, e))
    scafs.append((sx, se_))
    attach.append(list(range(110)))
    cases["extra bond"] = len(mols) - 1
    x, e = _chain_with(112, N, segs, Ef, [], rng)
    sx, se_ = SR.prefix(x, e, 110)
    sx = sx.copy()
    t = int(np.argmax(sx[100, :segs[0]]))
    sx[100, :segs[0]] = 0
    sx[100, (t + 1) % segs[0]] = 1
    mols.append((x, e))
    scafs.append((sx, se_))
    attach.append(list(range(110)))
    cases["atom type"] = len(mols) - 1
    nodes, edges = np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])
    sn, se = np.stack([s[0] for s in scafs]), np.stack([s[1] for s in scafs])
    masked = N <= 127
    table = ScaffoldTable(sn, se, attach if masked else None, N, sum(lay), Ef, lay, "cuda")
    run = _Route(N, Ef, layout, 263, nodes.shape[0])
    sw = run.plan(nodes, edges, np.arange(nodes.shape[0]), table.struct())
    flags = ROUTE_NOT_PREFIX | (ROUTE_MASKED if masked else 0)
    assert sw[3] == 0 and sw[1] == flags, sw
    assert sw[2] == min(cases.values()), (sw, cases)
    # each refusal alone names its own molecule
    for case, m in cases.items():
        keep = [0, 1, m]
        run = _Route(N, Ef, layout, 263, 3)
        sub = ScaffoldTable(sn[keep], se[keep], [attach[i] for i in keep] if masked else None, N, sum(lay), Ef, lay,
                            "cuda")
        sw = run.plan(nodes[keep], edges[keep], np.arange(3), sub.struct())
        assert sw[1] == (ROUTE_MASKED if case == "masked" else ROUTE_NOT_PREFIX) and sw[2] == 2, (case, sw)
        run.intact()


@pytest.mark.parametrize("N", [128, 181])
def test_plan_refuses_attachment_points_beyond_127_before_any_launch(N):
    """the plan refuses a table with protect words at N > 127 (it would read past the scaffold's 4 words); the same
    table without them plans"""
    from graphinvent_b200._lib import check, lib
    from graphinvent_b200.generation import ScaffoldTable
    layout, Ef = "gdb13", 1
    lay = LAYOUTS[layout]
    nodes, edges = molecule_set(N, segs_of(layout), Ef, seed=3)
    ks = np.array([max(1, P.n_atoms(x) // 2) for x in nodes])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    table = ScaffoldTable(sn, se, None, N, sum(lay), Ef, lay, "cuda")
    run = _Route(N, Ef, layout, 64, nodes.shape[0])
    sw = run.plan(nodes, edges, np.arange(nodes.shape[0]), table.struct())
    assert sw[1] == 0 and sw[3] == 0
    words = torch.zeros(nodes.shape[0], 4, dtype=torch.int32, device="cuda")
    sc = table.struct()
    sc.protect = words.data_ptr()
    before = run.status.t.clone()
    rc = lib.gib_route_plan_scaffold(run.bd, _p(run.gn), _p(run.ge), nodes.shape[0], run.chunk, ctypes.byref(sc),
                                     _p(run.gi), _p(run.ws), _p(run.off), _p(run.status), _st())
    assert rc < 0 and b"N <= 127" in lib.gib_last_error()
    torch.cuda.synchronize()
    assert torch.equal(run.status.t, before)            # nothing was launched: the status words are as they were
    with pytest.raises(RuntimeError, match="N <= 127"):
        check(rc, "gib_route_plan_scaffold")


# ---- A. the masks --------------------------------------------------------------------------------------------------
def _mask_case(N, Ef, per_node, seed):
    """scaffolds of k in K_SIZES + (N - 1, N), k <= N, random protect bits with the word-edge atoms attachment
    points; one slot per (scaffold, n = k .. N); -1 ids mixed in"""
    rng = np.random.default_rng(seed)
    ks = sorted({k for k in K_SIZES + (N - 1, N) if 1 <= k <= N})
    protect = np.zeros((len(ks), N), bool)
    for s, k in enumerate(ks):
        protect[s, :k] = rng.random(k) < 0.5
        protect[s, [i for i in WORD_EDGES if i < k]] = False
    slots = [(s, n) for s, k in enumerate(ks) for n in range(k, N + 1)]
    slots += [(-1, int(rng.integers(1, N + 1))) for _ in range(len(slots) // 8)]
    order = rng.permutation(len(slots))
    sid = np.array([slots[i][0] for i in order], np.int32)
    n_at = np.array([slots[i][1] for i in order], np.int32)
    apd = N * (per_node + Ef) + 1
    rows = {}
    for s, k in enumerate(ks):                           # the rule depends on n only through n - 1 < k
        rows[s] = (SR.mask_row(k, k, protect[s], N, Ef, per_node), SR.mask_row(k + 1, k, protect[s], N, Ef, per_node))
    want = np.zeros((len(sid), apd), bool)
    for b, (s, n) in enumerate(zip(sid, n_at)):
        if s >= 0:
            want[b] = rows[s][0 if n == ks[s] else 1]
    return np.array(ks, np.int32), protect, sid, n_at, want


def _words(protect):
    bits = np.zeros((protect.shape[0], 128), bool)
    bits[:, :protect.shape[1]] = protect
    w = (bits.reshape(-1, 4, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
    return w.astype(np.uint32).view(np.int32)


@pytest.mark.parametrize("N,Ef,per_node", [(38, 4, 5 * 3 * 4), (90, 1, 4 * 3 * 4 * 3), (127, 2, 5 * 3 * 2)])
def test_masks_against_mask_row(N, Ef, per_node):
    """gib_route_mask_logits (every slot) and gib_generation_mask_logits (slot 0 left alone; plain, and gated by
    row / state / counters) set exactly mask_row's entries to -inf and leave every other entry's bits unchanged"""
    from graphinvent_b200._lib import Scaffolds, check, lib
    ks, protect, sid, n_at, want = _mask_case(N, Ef, per_node, seed=N)
    B, apd = len(sid), want.shape[1]
    gk, gp = _G(ks), _G(_words(protect))
    sc = Scaffolds(n_atoms=gk.ptr(), protect=gp.ptr(), S=len(ks))
    gs, gn = _G(sid), _G(n_at)
    raw = torch.randn(B, apd, generator=torch.Generator().manual_seed(N)) * 3
    lg = _G(raw.numpy())
    check(lib.gib_route_mask_logits(B, N, Ef, apd, ctypes.byref(sc), _p(gs), _p(gn), _p(lg), _st()), "route mask")
    got = lg.view().cpu()
    assert torch.equal(torch.isinf(got), torch.from_numpy(want)) and (got[torch.isinf(got)] < 0).all()
    assert torch.equal(got[~torch.from_numpy(want)], raw[~torch.from_numpy(want)])
    # the generator's form: slot 0 is the dummy slot
    lg2 = _G(raw.numpy())
    check(lib.gib_generation_mask_logits(B, N, Ef, apd, ctypes.byref(sc), _p(gs), _p(gn), None, None, None, _p(lg2),
                                         _st()), "generation mask")
    w2 = want.copy()
    w2[0] = False
    got = lg2.view().cpu()
    assert torch.equal(torch.isinf(got), torch.from_numpy(w2))
    assert torch.equal(got[~torch.from_numpy(w2)], raw[~torch.from_numpy(w2)])
    # gated: row 2 of a [3, B] table of ids / atom counts, live (counters < B, status 0, 0 <= round < 2N) or not
    rng = np.random.default_rng(1)
    table_ids = np.stack([rng.permutation(sid), rng.permutation(sid), sid]).astype(np.int32)
    table_n = np.stack([rng.permutation(n_at), rng.permutation(n_at), n_at]).astype(np.int32)
    gti, gtn, grow = _G(table_ids), _G(table_n), _G(np.array([2], np.int32))
    bufs = [gk, gp, gs, gn, lg, lg2, gti, gtn, grow]
    for state, counters, live in (((0, 0), (0,), True), ((2 * N - 1, 0), (B - 1,), True), ((2 * N, 0), (0,), False),
                                  ((-1, 0), (0,), False), ((3, 1), (0,), False), ((3, 0), (B,), False)):
        gst, gc = _G(np.array(state, np.int32)), _G(np.array(counters + (0,), np.int32))
        lg3 = _G(raw.numpy())
        check(lib.gib_generation_mask_logits(B, N, Ef, apd, ctypes.byref(sc), _p(gti), _p(gtn), _p(grow), _p(gst),
                                             _p(gc), _p(lg3), _st()), "gated generation mask")
        got = lg3.view().cpu()
        if live:
            assert torch.equal(torch.isinf(got), torch.from_numpy(w2)), state
            assert torch.equal(got[~torch.from_numpy(w2)], raw[~torch.from_numpy(w2)])
        else:
            assert torch.equal(got, raw), state
        bufs += [gst, gc, lg3]
    torch.cuda.synchronize()
    for g in bufs:
        assert g.intact(), g.damage()


# ---- A. probabilities and their backward ---------------------------------------------------------------------------
@pytest.mark.parametrize("apd", [2, 33, 625, 4065, 52201])
def test_probs_and_dlogits_against_fp64(apd):
    """52 201 = N * (per_node + Ef) + 1 at N = 90, implicit H + chirality (4 * 3 * 4 * 3 * 4 per node), Ef = 4.  Rows:
    random, masked blocks of -inf, only terminate finite, saturated (p underflows to 0, the row stays finite), and
    every fifth a padding slot (a +0 row, no probability written)"""
    from graphinvent_b200._lib import check, lib
    rng = np.random.default_rng(apd)
    B, S = 40, 64
    logits = (4 * rng.standard_normal((B, apd))).astype(np.float32)
    act = rng.integers(0, apd, B)
    live = np.arange(B) % 5 != 4
    dst = np.full(B, -1, np.int32)
    dst[live] = rng.permutation(S)[:int(live.sum())]
    for b in range(0, B, 7):                             # masked rows: -inf blocks, the action outside them
        lo = int(rng.integers(0, apd))
        logits[b, lo:lo + apd // 3 + 1] = -np.inf
        logits[b, act[b]] = np.float32(rng.standard_normal())
    logits[1, :apd - 1] = -np.inf                        # only terminate may remain
    act[1] = apd - 1
    if apd > 2:
        logits[2] *= 300                                 # saturated: the action sits far below the row's max
        act[2] = int(np.argmin(logits[2]))
    act = np.where(live, act, -1).astype(np.int32)
    coef = rng.standard_normal(S).astype(np.float32)
    gl, gs, gc = _G(logits), _G(np.concatenate([act, dst])), _G(coef)
    lik, dl, pout = Guarded(4 * S), Guarded(4 * B * apd), Guarded(4 * S)
    check(lib.gib_route_probs(B, apd, _p(gl), _p(gs), _p(lik), _st()), "gib_route_probs")
    check(lib.gib_route_dlogits(B, apd, _p(gl), _p(gs), _p(gc), _p(dl), _p(pout), _st()), "gib_route_dlogits")
    sm = torch.softmax(torch.from_numpy(logits).double(), 1)
    d = dl.view(torch.float32, (B, apd)).cpu().double()
    pl, po = lik.view(torch.float32, (S,)).cpu(), pout.view(torch.float32, (S,)).cpu()
    for b in range(B):
        if not live[b]:
            assert (d[b] == 0).all() and not torch.signbit(d[b]).any(), b
            continue
        p64 = sm[b, act[b]].item()
        assert abs(pl[dst[b]].item() - p64) <= 2e-6 * p64 + 1e-37, (b, pl[dst[b]].item(), p64)
        assert po[dst[b]].item() == pl[dst[b]].item(), b   # the backward recomputes the forward's p bit for bit
        onehot = torch.zeros(apd, dtype=torch.float64)
        onehot[act[b]] = 1
        ref = float(coef[dst[b]]) * (onehot - sm[b])
        assert torch.isfinite(d[b]).all() and ((d[b] - ref).abs() <= 4e-6 * abs(float(coef[dst[b]])) + 1e-37).all(), b
    assert pl[dst[1]].item() == 1.0
    if apd > 2:
        assert pl[dst[2]].item() == 0.0
    written = np.zeros(S, bool)
    written[dst[live]] = True
    assert torch.isnan(pl[torch.from_numpy(~written)]).all() and torch.isnan(po[torch.from_numpy(~written)]).all()
    for g in (gl, gs, gc, lik, dl, pout):
        assert g.intact(), g.damage()


# ---- A. reduce and the coefficients --------------------------------------------------------------------------------
def test_reduce_and_grad_coef_on_routes_longer_than_a_warp():
    """routes of 1, 31, 32, 33, 64, 65, 1000 and 16 292 states among 40 short ones, in one call: nll and final in
    fp64 in build order, rounded once; the coefficients against coef_restated with each gradient null in turn; p = 0
    entries (nll = +inf) and an all-zero molecule (final = -inf, g_final = 0 there)"""
    from graphinvent_b200._lib import check, lib
    rng = np.random.default_rng(17)
    long_ = [1, 31, 32, 33, 64, 65, 1000, 16292]
    lengths = np.concatenate([long_, rng.integers(1, 13, 40)])
    lengths = lengths[rng.permutation(len(lengths))]
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    S, M = int(offsets[-1]), len(lengths)
    p = (rng.random(S) ** 3).astype(np.float32)
    p[rng.random(S) < 0.05] = 0.0
    zero = int(np.flatnonzero(lengths == 33)[0])        # an all-zero molecule of 33 states
    p[offsets[zero]:offsets[zero + 1]] = 0.0
    g_lik, g_nll = rng.standard_normal(S).astype(np.float32), rng.standard_normal(M).astype(np.float32)
    g_fin = rng.standard_normal(M).astype(np.float32)
    g_fin[zero] = 0.0
    off, lik, gl, gn, gf = _G(offsets), _G(p), _G(g_lik), _G(g_nll), _G(g_fin)
    nll, fin = Guarded(4 * M), Guarded(4 * M)
    check(lib.gib_route_reduce(M, _p(off), _p(lik), _p(nll), _p(fin), _st()), "gib_route_reduce")
    got_n, got_f = nll.view(torch.float32, (M,)).cpu().numpy(), fin.view(torch.float32, (M,)).cpu().numpy()
    with np.errstate(divide="ignore"):
        for m in range(M):
            q = p[offsets[m]:offsets[m + 1]].astype(np.float64)
            ln, s = 0.0, 0.0
            for v in q:                                  # build order, as the kernel sums
                ln -= np.log(v)
                s += v
            wn, wf = np.float32(ln), np.float32(np.log(s))
            for g, w, what in ((got_n[m], wn, "nll"), (got_f[m], wf, "final")):
                if np.isinf(w):
                    assert g == w, (m, what)
                else:
                    assert abs(g - w) <= 1.2e-7 * abs(w) + 1e-30, (m, what, g, w)
    assert np.isinf(got_n[zero]) and got_f[zero] == -np.inf
    assert all(np.isinf(got_n[m]) == (p[offsets[m]:offsets[m + 1]] == 0).any() for m in range(M))
    bufs = [off, lik, gl, gn, gf, nll, fin]
    for args in ((gl, gn, gf), (None, gn, gf), (gl, None, gf), (gl, gn, None)):
        coef = Guarded(4 * S)
        check(lib.gib_route_grad_coef(M, _p(off), _p(lik), *map(_p, args), _p(coef), _st()), "gib_route_grad_coef")
        want = coef_restated(p, offsets, *(None if a is None else b for a, b in zip(args, (g_lik, g_nll, g_fin))))
        got = coef.view(torch.float32, (S,)).cpu().numpy()
        assert np.all(np.isfinite(got))
        bad = np.abs(got - want) > 2.5e-7 * np.abs(want) + 1e-30
        assert not bad.any(), (np.flatnonzero(bad)[:8], np.searchsorted(offsets, np.flatnonzero(bad)[:8], "right") - 1)
        bufs.append(coef)
    torch.cuda.synchronize()
    for g in bufs:
        assert g.intact(), g.damage()


# ---- B. the generator with scaffolds beyond N = 13 -----------------------------------------------------------------
def _gen_constants(N, layout, Ef, model="GGNN", **kw):
    from graphinvent_b200.config import make_constants
    A, CH, H, C = LAYOUTS[layout]
    return make_constants(model, max_n_nodes=N, n_node_features=A + CH + H + C, n_edge_features=Ef,
                          len_f_add_per_node=A * CH * max(H, 1) * max(C, 1) * Ef, len_f_conn_per_node=Ef,
                          n_atom_types=A, n_formal_charge=CH, n_imp_H=H, n_chirality=C, **kw)


def _gen_scaffolds(N, layout, Ef, seed, sizes):
    """prefixes of one tree with rings of N atoms: scaffolds of `sizes` atoms, and attachment points in every word"""
    rng = np.random.default_rng(seed)
    x, e = molecule(N, N, segs_of(layout), Ef, tree_with_rings(N, Ef, rng), rng)
    ks = [k for k in sizes if 1 <= k < N]
    sn, se = SR.prefix_scaffolds(np.repeat(x[None], len(ks), 0), np.repeat(e[None], len(ks), 0), ks)
    att = [sorted({k - 1} | {i for i in WORD_EDGES if i < k} | {int(i) for i in np.flatnonzero(rng.random(k) < 0.3)})
           for k in ks]
    return sn, se, att


GEN_DIMS = [(38, 4, "imp_H+chirality", 61), (90, 4, "chirality", 48), (127, 2, "imp_H", 40), (127, 2, "gdb13", 33)]


@pytest.mark.parametrize("N,Ef,layout,B", GEN_DIMS, ids=[f"N{g[0]}-{g[2]}" for g in GEN_DIMS])
def test_generator_rounds_and_mask_match_the_oracle(N, Ef, layout, B):
    """GraphGenerator's round kernels on a random action stream from scaffolds of 1 .. N - 1 atoms: the state after
    every round equals the scaffold oracle's bit for bit, and the attachment mask of that state equals
    scaffold_oracle.forbidden for every slot"""
    from graphinvent_b200.generation import GraphGenerator
    from tests.test_gpu_generation_layouts import _layout_stream
    A, CH, H, C = LAYOUTS[layout]
    sn, se, att = _gen_scaffolds(N, layout, Ef, seed=N, sizes=(1, 2, 33, 40, 70, 100, N - 1))
    rng = np.random.default_rng(N + B)
    st = SO.ScaffoldState(B, N, A, CH, Ef, H, C, sn, se)
    gen = GraphGenerator(None, B, constants=_gen_constants(N, layout, Ef), scaffolds=(sn, se), attachment=att)
    protect = SO.protect_of(st.k, att, N)
    assert (gen.scaffolds.protect_mask == protect).all()
    stream = _st()
    for rnd in range(2 * N - 1):
        if st.n_generated > B:
            break
        logits = torch.randn(B, gen.apd, device="cuda", generator=torch.Generator("cuda").manual_seed(rnd))
        raw = logits.clone()
        gen._mask(logits, stream)
        got = torch.isinf(logits).cpu().numpy()
        for b in range(B):
            assert np.array_equal(got[b], SO.forbidden(st, b, protect)), (rnd, b)
        assert torch.equal(logits[~torch.isinf(logits)], raw[~torch.isinf(logits)])
        a, _ = _layout_stream(rng, st)
        lik = rng.random(B).astype(np.float32)
        SO.generation_round(st, rnd, a, lik)
        gen._round(rnd, torch.from_numpy(a).cuda(), torch.from_numpy(lik).cuda(), stream)
        for name in ("nodes", "edges", "n_nodes", "likelihoods"):
            assert (getattr(gen, name).cpu().numpy() == getattr(st, name)).all(), (rnd, name)
        assert int(gen._counters[0]) == st.n_generated
        assert (gen._slot_ids.cpu().numpy() == st.slot_ids).all() and int(gen._started) == st.started
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "generated_likelihoods",
                 "properly_terminated"):
        assert (getattr(gen, name).cpu().numpy() == getattr(st, name)).all(), name
    assert (gen._gen_scaffolds.cpu().numpy() == st.generated_scaffolds).all()
    assert st.n_generated > B // 4


def test_scaffold_init_on_guarded_buffers():
    """gib_generation_scaffold_init at N = 127: slot b >= 1 holds scaffold (b - 1) mod S as the oracle's start state,
    slot_ids / started as the oracle's, slot 0 and everything past the buffers untouched"""
    from graphinvent_b200._lib import check, lib
    from graphinvent_b200.generation import ScaffoldTable
    N, Ef, layout, B = 127, 2, "chirality", 37
    A, CH, H, C = LAYOUTS[layout]
    sn, se, att = _gen_scaffolds(N, layout, Ef, seed=9, sizes=(1, 31, 32, 33, 64, 97, 126))
    table = ScaffoldTable(sn, se, att, N, A + CH + H + C, Ef, LAYOUTS[layout], "cuda")
    F, Lw = A + CH + H + C, 2 * N
    nodes, edges = Guarded(4 * B * N * F), Guarded(4 * B * N * N * Ef)
    n_nodes, lik = Guarded(4 * B), Guarded(4 * B * Lw)
    slot_ids, started, gen_sc = Guarded(4 * B), Guarded(4), Guarded(4 * 2 * B)
    sc = table.struct()
    sc.slot_ids, sc.started, sc.gen_scaffolds = slot_ids.ptr(), started.ptr(), gen_sc.ptr()
    check(lib.gib_generation_scaffold_init(B, N, F, Ef, ctypes.byref(sc), _p(nodes), _p(edges), _p(n_nodes),
                                           _p(lik), _st()), "gib_generation_scaffold_init")
    st = SO.ScaffoldState(B, N, A, CH, Ef, H, C, sn, se)
    gn = nodes.view(torch.float32, (B, N, F)).cpu().numpy()
    ge = edges.view(torch.float32, (B, N, N, Ef)).cpu().numpy()
    assert np.array_equal(gn[1:], st.nodes[1:]) and np.array_equal(ge[1:], st.edges[1:])
    assert np.isnan(gn[0]).all() and np.isnan(ge[0]).all()
    assert np.array_equal(_i32(n_nodes, B)[1:], st.n_nodes[1:]) and _i32(n_nodes, B)[0] == -1
    lk = lik.view(torch.float32, (B, Lw)).cpu().numpy()
    assert (lk[1:] == 0).all() and np.isnan(lk[0]).all()
    assert np.array_equal(_i32(slot_ids, B), st.slot_ids) and _i32(started, 1)[0] == st.started
    assert (_i32(gen_sc, 2 * B) == -1).all()              # untouched: the poison reads as -1
    torch.cuda.synchronize()
    for g in (nodes, edges, n_nodes, lik, slot_ids, started, gen_sc):
        assert g.intact(), g.damage()


def _small_model(N, layout, Ef, seed, model="GGNN"):
    """a seeded model of small widths for the layout: (net, oracle state dict, oracle constants, constants)"""
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = _gen_constants(N, layout, Ef, model=model, **SMALL)
    OC = O.make_constants(**dict(C._asdict(), device="cpu"))
    sd = O.init_state_dict(OC, seed=seed)
    net = mpnn.create(C)
    net.load_state_dict(sd)
    return net.cuda(), sd, OC, C


# small widths: the EMN's per-entry message matrices (message_size x hidden_node_features) at route_entry_capacity --
# 1.03 M bond entries at N = 64, B = 256 -- take 31 GiB of forward workspace at widths of 32
SMALL = dict(hidden_node_features=16, message_size=16, message_passes=2, enn_hidden_dim=32, enn_depth=2,
             msg_hidden_dim=32, msg_depth=2, att_hidden_dim=32, att_depth=2, gather_width=16,
             gather_att_hidden_dim=32, gather_att_depth=2, gather_emb_hidden_dim=32, gather_emb_depth=2,
             mlp1_hidden_dim=32, mlp1_depth=2, mlp2_hidden_dim=32, mlp2_depth=2, edge_emb_size=16,
             edge_emb_hidden_dim=32, edge_emb_depth=2)
CHUNK = 64          # the scorers' chunk_molecules: a few molecules here, so the chunk-sized buffers stay small


def test_captured_generator_and_masked_rl_rollout_at_n_38():
    """GraphedGenerator with attachment points in words 0 and 1 equals the eager loop bit for bit; a masked
    GraphedGeneratorRL rollout's backward recomputes its probabilities bit for bit and matches eager autograd"""
    from graphinvent_b200.generation import GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGenerator, GraphedGeneratorRL
    from tests.test_gpu_rl_graphed import _loss, _run
    from tests.test_gpu_scaffold_generation import STATE, _eager
    N, Ef, layout = 38, 4, "imp_H+chirality"
    sn, se, att = _gen_scaffolds(N, layout, Ef, seed=38, sizes=(1, 5, 31, 33, 36, 37))
    net, _, _, C = _small_model(N, layout, Ef, seed=1)
    net.eval()
    B = 96
    graphed = GraphedGenerator(net, B, constants=C, scaffolds=(sn, se), attachment=att)
    U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(2), device="cuda")
    got = graphed.build_graphs(uniforms=U)
    eager = _eager(net, C, B, U, (sn, se), att)
    assert got == int(eager._counters[0]) and graphed.rounds == eager.rounds
    for name in STATE:
        assert torch.equal(getattr(graphed, name), getattr(eager, name)), name
    assert torch.equal(graphed.generated_scaffolds, eager._gen_scaffolds[:B])
    k = graphed.scaffolds.n_atoms
    ids = graphed.generated_scaffolds.cpu().numpy()
    en = graphed.generated_edges.cpu().numpy()
    protect = SO.protect_of(k, att, N)
    for p in range(B):
        s = ids[p]
        for i in np.flatnonzero(protect[s][:k[s]]):
            assert (en[p, i] == se[s, i]).all(), (p, i)        # protected atoms gain no bond
    # RL: agent and prior, a masked rollout and its backward against eager autograd
    agent, _, _, _ = _small_model(N, layout, Ef, seed=3)
    prior, _, _, _ = _small_model(N, layout, Ef, seed=4)
    gen = GraphedGeneratorRL(agent, B, constants=C, scaffolds=(sn, se), attachment=att)
    for s in range(1, 9):
        U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(10 + s), device="cuda")
        with torch.no_grad():
            if not isinstance(_run(lambda: gen.build_graphs(agent, prior, uniforms=U)), Exception):
                break
    else:
        pytest.fail("no finished rollout among the seeds tried")
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    R_ = gen.rounds
    p_a, p_b, acts = gen.p_a[:R_].clone(), gen.p_b[:R_].clone(), gen.act_rec[:R_].clone()
    gids = gen.generated_scaffolds.clone()
    _loss(agent_ll, prior_ll).backward()
    assert torch.equal(gen.recomputed_p[0][:R_], p_a) and torch.equal(gen.recomputed_p[1][:R_], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    eg = GraphGeneratorRL(agent2, B, constants=C, scaffolds=(sn, se), attachment=att)
    agent2.entry_capacity = prior2.entry_capacity = gen.entry_capacity
    try:
        _, ll_a, ll_p, _ = eg.sample(agent2, prior2, replay=list(acts))
    finally:
        agent2.entry_capacity = prior2.entry_capacity = None
    assert eg.rounds == R_ and torch.equal(eg.generated_scaffolds, gids)
    for name in ("generated_nodes", "generated_edges", "generated_n_nodes", "properly_terminated"):
        assert torch.equal(getattr(gen, name), getattr(eg, name)), name
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


# ---- C. RouteScorer end to end at non-gdb13 dims -------------------------------------------------------------------
E2E = [(38, 4, "imp_H+chirality"), (64, 1, "gdb13")]


def _e2e_molecules(N, layout, Ef, seed):
    """small molecules in decoding order (a chain, a star, a tree with rings, a complete graph of 7 atoms, one atom)
    so the CPU fp64 oracle stays quick, and a chain of N atoms that reaches row N - 1"""
    rng = np.random.default_rng(seed)
    segs = segs_of(layout)
    specs = [(9, chain(9, Ef, rng)), (8, star(8, Ef, rng)), (14, tree_with_rings(14, Ef, rng)),
             (7, complete(7, Ef, rng)), (1, []), (N, chain(N, Ef, rng))]
    mols = [molecule(n, N, segs, Ef, b, rng) for n, b in specs]
    return np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols])


@pytest.mark.parametrize("model", ["GGNN", "EMN"])
@pytest.mark.parametrize("N,Ef,layout", E2E, ids=[f"N{g[0]}-Ef{g[1]}-{g[2]}" for g in E2E])
def test_route_scorer_against_fp64(N, Ef, layout, model):
    """unconditional, conditional without and with attachment points, against route_nll_reference.score and
    scaffold_route_reference.score with assert_within's bounds; bit-identical over batch_size and chunk_molecules"""
    from graphinvent_b200.graphed import RouteScorer
    net, sd, OC, _ = _small_model(N, layout, Ef, seed=5, model=model)
    segs = segs_of(layout)
    nodes, edges = _e2e_molecules(N, layout, Ef, seed=N)
    kw = layout_kw(layout)
    out = RouteScorer(net, 64, chunk_molecules=CHUNK, **kw).score(nodes, edges)
    oracle = R.score(sd, OC, nodes, edges, segs)
    assert torch.equal(out.offsets.cpu(), torch.from_numpy(oracle[1]))
    R.assert_within(out.likelihoods, out.nll, out.final, oracle, f"{model} N={N}")
    rng = np.random.default_rng(N)
    M = nodes.shape[0]
    ks = np.array([max(1, P.n_atoms(nodes[m]) - int(rng.integers(0, 4))) for m in range(M)])
    ks[-1] = 33                                          # attachment points in word 1
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    ids = np.arange(M)
    ids[2] = -1
    attach = [attachment_points(nodes[m], edges[m], int(ks[m]), rng) for m in range(M)]
    for masked in (False, True):
        scorer = RouteScorer(net, 64, scaffolds=(sn, se), attachment=attach if masked else None,
                             chunk_molecules=CHUNK, **kw)
        got = scorer.score(nodes, edges, scaffold_ids=ids)
        protect = SR.protect_of(sn, attach) if masked else None
        R.assert_within(got.likelihoods, got.nll, got.final, SR.score(sd, OC, nodes, edges, ids, sn, segs, protect),
                        f"{model} N={N} masked={masked}")
        if masked:
            for B, chunk in ((1, 2), (256, 1), (7, 5)):
                again = RouteScorer(net, B, scaffolds=(sn, se), attachment=attach, chunk_molecules=chunk,
                                    **kw).score(nodes, edges, scaffold_ids=ids)
                for a, b, name in zip(again, got, got._fields):
                    assert torch.equal(a, b), (B, chunk, name)


def test_route_scorer_gradients_against_fp64_at_n_38():
    """one requires_grad=True conditional score with attachment points against fp64 parameter gradients, with
    test_gpu_route_grad's yardstick (fp64-anchored, SELU kinks bracketed)"""
    from graphinvent_b200.graphed import RouteScorer
    from oracle import mpnn_oracle as O
    from tests.test_gpu_route_grad import KINK_TAU, _assert_fp64_anchored, _weights
    from tests.test_gpu_scaffold_route import _oracle_grads
    N, Ef, layout = 38, 4, "imp_H+chirality"
    net, sd, OC, _ = _small_model(N, layout, Ef, seed=6)
    segs = segs_of(layout)
    nodes, edges = _e2e_molecules(N, layout, Ef, seed=7)
    M = nodes.shape[0]
    rng = np.random.default_rng(8)
    ks = np.array([max(1, P.n_atoms(nodes[m]) // 2) for m in range(M)])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    ids = np.arange(M)
    attach = [attachment_points(nodes[m], edges[m], int(ks[m]), rng) for m in range(M)]
    out = RouteScorer(net, 64, scaffolds=(sn, se), attachment=attach, chunk_molecules=CHUNK, **layout_kw(layout)).score(
        nodes, edges, scaffold_ids=ids, requires_grad=True)
    w = _weights(M, seed=M)
    grads = torch.autograd.grad((w.cuda() * out.nll).sum(), list(net.parameters()))
    protect = SR.protect_of(sn, attach)
    X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, segs)
    masks = SR.state_masks(sid, n_at, sn, protect, N, Ef, OC.len_f_add_per_node)
    w_state = torch.repeat_interleave(w, torch.from_numpy(np.diff(offsets)))
    g = lambda dt: _oracle_grads(sd, OC, X, E, acts, masks, w_state, dt)
    g32, g64 = g(torch.float32), g(torch.float64)
    try:
        O.KINK = (KINK_TAU, "L")
        gL = g(torch.float64)
        O.KINK = (KINK_TAU, "R")
        gR = g(torch.float64)
    finally:
        O.KINK = None
    _assert_fp64_anchored(net, grads, (g32, g64, gL, gR), "N=38 masked")
