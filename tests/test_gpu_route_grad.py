"""GPU: gradients of the decoding-route likelihoods (graphed.RouteScorer.score(..., requires_grad=True)) -- against
fp64 autograd through the oracle for the four models and an implicit-H + chirality layout, against eager autograd
through the module API, the recomputed probabilities and the host loop of the same C-ABI calls, determinism and
chunking, edge cases, guarded buffers, memory, the TF32 / bf16 modes and a short fine-tuning run."""
import ctypes
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R
from tests.conftest import GOLDEN, MODELS
from tests.guarded import Guarded
from tests.test_gpu_route_nll import GDB13, LAYOUTS, SEGS, _fixture, _layout_molecules, _net
from tests.test_route_grad_host import coef_restated

pytestmark = pytest.mark.gpu


def _weights(M, seed=0):
    """non-uniform, non-negative molecule weights"""
    return torch.rand(M, generator=torch.Generator().manual_seed(seed)) * 2 + 0.05


def _flat(grads):
    return torch.cat([g.reshape(-1) for g in grads])


def _route_grads(scorer, net, nodes, edges, loss_fn):
    """(outputs, gradients of loss_fn(outputs) w.r.t. the model's parameters) on the captured path"""
    out = scorer.score(nodes, edges, requires_grad=True)
    return out, torch.autograd.grad(loss_fn(out), list(net.parameters()))


# ---- fp64-anchored gradients ---------------------------------------------------------------------------------------
KINK_TAU, GEMM_EPS = 3e-5, 3e-5        # tests/test_gpu_parity.py: the tensor-core path's SELU band and GEMM arithmetic


def _oracle_route_grads(sd, C, X, E, acts, w_state, dtype, batch=512):
    """gradients of sum_s w_s * -log_softmax(forward(state s))[a_s] through mpnn_oracle.forward in `dtype`"""
    from oracle import mpnn_oracle as O
    leaves = OrderedDict((k, v.to(dtype).detach().clone().requires_grad_(True)) for k, v in sd.items())
    total = OrderedDict((k, torch.zeros_like(v)) for k, v in leaves.items())
    for s in range(0, X.shape[0], batch):
        o = O.forward(leaves, C, torch.from_numpy(X[s:s + batch]).to(dtype), torch.from_numpy(E[s:s + batch]).to(dtype))
        a = torch.from_numpy(acts[s:s + batch]).view(-1, 1)
        loss = (w_state[s:s + batch].to(dtype) * -torch.log_softmax(o, 1).gather(1, a).view(-1)).sum()
        for (k, t), g in zip(total.items(), torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)):
            if g is not None:
                t += g.detach()
    return total


def _oracle_with_kink_band(sd, C, X, E, acts, w_state):
    """(fp32, fp64, fp64 with every SELU within KINK_TAU of 0 on its left / right limit) oracle gradients"""
    from oracle import mpnn_oracle as O
    g32 = _oracle_route_grads(sd, C, X, E, acts, w_state, torch.float32)
    g64 = _oracle_route_grads(sd, C, X, E, acts, w_state, torch.float64)
    try:
        O.KINK = (KINK_TAU, "L")
        gL = _oracle_route_grads(sd, C, X, E, acts, w_state, torch.float64)
        O.KINK = (KINK_TAU, "R")
        gR = _oracle_route_grads(sd, C, X, E, acts, w_state, torch.float64)
    finally:
        O.KINK = None
    return g32, g64, gL, gR


def _assert_fp64_anchored(net, grads, oracle, tag):
    """test_gpu_parity._fp64_anchored's yardstick, per tensor and over all of them"""
    g32, g64, gL, gR = oracle
    got = {k: g.detach().cpu().double() for (k, _), g in zip(net.named_parameters(), grads)}
    assert set(got) == set(g64)
    gscale = max(g.norm().item() for g in g64.values())
    tot = [0.0] * 4
    for k, g in g64.items():
        d_cuda = (got[k] - g).norm().item()
        d_ref = (g32[k].double() - g).norm().item()
        d_kink = (gL[k] - gR[k]).norm().item()
        bound = 2.0 * d_ref + d_kink + GEMM_EPS * g.norm().item() + 1e-7 * gscale
        assert d_cuda <= bound, f"{tag} {k}: |cuda - fp64| {d_cuda:.3e} > bound {bound:.3e} (ref32 {d_ref:.3e}, kink {d_kink:.3e})"
        for i, v in enumerate((d_cuda, d_ref, d_kink, g.norm().item())):
            tot[i] += v * v
    tot = [t ** 0.5 for t in tot]
    assert tot[0] <= 2.0 * tot[1] + tot[2] + GEMM_EPS * tot[3], (tag, tot)


def _fp64_case(net, sd, C, nodes, edges, segs, layout):
    from graphinvent_b200.graphed import RouteScorer
    M = nodes.shape[0]
    w = _weights(M, seed=M)
    X, E, acts, offsets = R.build_order_states(nodes, edges, segs)
    w_state = torch.repeat_interleave(w, torch.from_numpy(np.diff(offsets)))
    scorer = RouteScorer(net, 128, **layout)
    _, grads = _route_grads(scorer, net, nodes, edges, lambda o: (w.cuda() * o.nll).sum())
    return grads, _oracle_with_kink_band(sd, C, X, E, acts, w_state)


@pytest.mark.parametrize("model", MODELS)
def test_gradients_against_fp64(model):
    nodes, edges, _ = _fixture(40)
    net, sd, C = _net(model)
    grads, oracle = _fp64_case(net, sd, C, nodes, edges, SEGS, GDB13)
    _assert_fp64_anchored(net, grads, oracle, model)


def test_gradients_against_fp64_implicit_H_and_chirality():
    from graphinvent_b200.config import layout_dims
    from oracle import mpnn_oracle as O
    A, Fc, H, X = LAYOUTS["imp_H+chirality"]
    L = layout_dims(A, Fc, 3, ignore_H=False, use_chirality=True)
    C = O.make_constants("GGNN", n_node_features=L["n_node_features"], len_f_add_per_node=L["len_f_add_per_node"])
    net, sd, C = _net("GGNN", C)
    nodes, edges = _layout_molecules(LAYOUTS["imp_H+chirality"])
    layout = dict(n_atom_types=A, n_formal_charge=Fc, n_imp_H=L["n_imp_H"], n_chirality=L["n_chirality"])
    grads, oracle = _fp64_case(net, sd, C, nodes, edges, P.segments(A, Fc, H, X), layout)
    _assert_fp64_anchored(net, grads, oracle, "imp_H+chirality")


# ---- against eager autograd through the module API ---------------------------------------------------------------
def _eager_route(net, nodes, edges, B, segs=SEGS):
    """likelihoods, nll and final with autograd through `model(nodes, edges)` in capacity mode at the scorer's
    capacity, batches of B build-order states padded with empty graphs (every forward GEMM on the tensor-core kernel),
    ATen's softmax gather and route_nll_reference.reduce"""
    from graphinvent_b200.graphed import route_entry_capacity
    X, E, acts, offsets = R.build_order_states(nodes, edges, segs)
    S, N, Ef = X.shape[0], X.shape[1], E.shape[3]
    net.entry_capacity = route_entry_capacity(B, N, Ef)
    try:
        ps = []
        for s in range(0, S, B):
            k = min(B, S - s)
            x = torch.zeros(B, *X.shape[1:], device="cuda")
            e = torch.zeros(B, *E.shape[1:], device="cuda")
            x[:k], e[:k] = torch.from_numpy(X[s:s + k]).cuda(), torch.from_numpy(E[s:s + k]).cuda()
            a = torch.from_numpy(acts[s:s + k]).cuda().view(-1, 1)
            ps.append(torch.softmax(net(x, e)[:k], 1).gather(1, a).view(-1))
    finally:
        net.entry_capacity = None
    p = torch.cat(ps)
    nll, final = R.reduce(p, offsets)
    return p, offsets, nll, final


def _mixed_loss(S, M, seed=5):
    g = torch.Generator().manual_seed(seed)
    sign = lambda n: (torch.randint(0, 2, (n,), generator=g) * 2 - 1).float() * (torch.rand(n, generator=g) + 0.5)
    r_lik, r_nll, r_fin = sign(S).cuda(), sign(M).cuda(), sign(M).cuda()
    return lambda lik, nll, final: (r_lik * lik).sum() + (r_nll * nll).sum() + (r_fin * final).sum()


def _assert_close_to_eager(grads, eager_grads, rel=1e-4, what=""):
    total = sum(g.norm().item() ** 2 for g in eager_grads) ** 0.5
    for i, (g, e) in enumerate(zip(grads, eager_grads)):
        assert (g - e).norm().item() <= rel * e.norm().item() + 0.1 * rel * total, f"{what} parameter {i}"


def test_all_three_outputs_match_eager_autograd():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(40)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 256, **GDB13)
    out = scorer.score(nodes, edges, requires_grad=True)
    assert out.likelihoods.requires_grad and out.nll.requires_grad and out.final.requires_grad
    assert not out.offsets.requires_grad
    loss_fn = _mixed_loss(out.likelihoods.numel(), nodes.shape[0])
    grads = torch.autograd.grad(loss_fn(out.likelihoods, out.nll, out.final), list(net.parameters()))
    p, offsets, nll, final = _eager_route(net, nodes, edges, scorer.B)
    assert np.array_equal(out.offsets.cpu().numpy(), offsets)
    assert torch.allclose(p, out.likelihoods, rtol=1e-6, atol=0)
    eager = torch.autograd.grad(loss_fn(p, nll, final), list(net.parameters()))
    _assert_close_to_eager(grads, eager)


# ---- recomputation -----------------------------------------------------------------------------------------------
def test_recomputed_probabilities_and_the_host_loop():
    """chunk by chunk, the backward's recomputed p equals the forward's bit for bit; the captured backward equals
    the same C-ABI calls made one by one from the host, and autograd's gradient"""
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture()
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 256, chunk_molecules=13, **GDB13)
    out = scorer.score(nodes, edges, requires_grad=True)
    w = _weights(nodes.shape[0]).cuda()
    loss = (w * out.nll).sum() + out.final.sum()
    rec, lik, params = out.nll.grad_fn.rec, out.likelihoods.detach(), list(net.parameters())
    assert len(rec.chunks) == -(-nodes.shape[0] // 13)
    b = scorer._bwd
    runs = []
    for eager in (False, True):
        scorer._pack(params)
        b.gflat.zero_()
        for c, (_, base, S) in enumerate(rec.chunks):
            scorer._backward_chunk(rec, c, lik, None, w, torch.ones_like(w), eager=eager)
            assert torch.equal(scorer.lik[:S], lik[base:base + S]), (eager, c)
        runs.append(b.gflat.clone())
    assert torch.equal(runs[0], runs[1])
    grads = torch.autograd.grad(loss, params)
    assert torch.equal(_flat(grads), runs[0])


# ---- determinism and chunking -----------------------------------------------------------------------------------
def test_determinism_chunking_and_several_calls_per_backward():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture()
    net, _, _ = _net("GGNN")
    M = nodes.shape[0]
    w = _weights(M).cuda()
    loss_fn = lambda o: (w * o.nll).sum() - 0.5 * o.final.sum()
    params = list(net.parameters())
    out = RouteScorer(net, 256, **GDB13).score(nodes, edges, requires_grad=True)
    loss = loss_fn(out)
    g1 = _flat(torch.autograd.grad(loss, params, retain_graph=True))
    g2 = _flat(torch.autograd.grad(loss, params))
    assert torch.equal(g1, g2)
    norm = g1.norm().item()
    for B, chunk in ((256, 7), (1000, 4096), (1000, 7)):
        _, g = _route_grads(RouteScorer(net, B, chunk_molecules=chunk, **GDB13), net, nodes, edges, loss_fn)
        # the same per-state terms summed into the bucket in another grouping: fp32 regrouping of the batch sums
        assert (_flat(g) - g1).norm().item() <= 1e-5 * norm, (B, chunk)
    # two score() calls, one backward
    scorer = RouteScorer(net, 256, **GDB13)
    half = M // 2
    singles = []
    for sl in (slice(0, half), slice(half, M)):
        net.zero_grad(set_to_none=True)
        o = scorer.score(nodes[sl], edges[sl], requires_grad=True)
        (w[sl] * o.nll).sum().backward()
        singles.append([p.grad.clone() for p in params])
    net.zero_grad(set_to_none=True)
    oa = scorer.score(nodes[:half], edges[:half], requires_grad=True)
    ob = scorer.score(nodes[half:], edges[half:], requires_grad=True)
    ((w[:half] * oa.nll).sum() + (w[half:] * ob.nll).sum()).backward()
    for p, a, b in zip(params, *singles):
        assert torch.allclose(p.grad, a + b, rtol=1e-6, atol=1e-9)


# ---- edge cases -------------------------------------------------------------------------------------------------
def test_parameter_changed_in_place_raises():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(8)
    net, _, _ = _net("GGNN")
    out = RouteScorer(net, 64, **GDB13).score(nodes, edges, requires_grad=True)
    with torch.no_grad():
        next(net.parameters()).add_(1e-3)
    with pytest.raises(RuntimeError, match="inplace"):
        out.nll.sum().backward()


def test_caller_arrays_changed_after_score_do_not_change_the_gradients():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(16)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 64, **GDB13)
    _, want = _route_grads(scorer, net, nodes, edges, lambda o: o.nll.sum())
    for where in ("host", "device"):
        n, e = nodes.copy(), edges.copy()
        if where == "device":
            n, e = torch.from_numpy(n).cuda(), torch.from_numpy(e).cuda()
        out = scorer.score(n, e, requires_grad=True)
        n[3:] = 0                                   # edits after the call: an empty molecule would be refused
        e[:] = 0
        got = torch.autograd.grad(out.nll.sum(), list(net.parameters()))
        assert all(torch.equal(a, b) for a, b in zip(got, want)), where


def test_plain_calls_keep_no_record_and_equal_the_grad_path():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(16)
    net, _, _ = _net("GGNN")
    ref = RouteScorer(net, 64, **GDB13).score(nodes, edges, requires_grad=True)
    for name in ("default", "no_grad", "frozen"):
        scorer = RouteScorer(net, 64, **GDB13)
        if name == "no_grad":
            with torch.no_grad():
                out = scorer.score(nodes, edges, requires_grad=True)
        elif name == "frozen":
            net.requires_grad_(False)
            try:
                out = scorer.score(nodes, edges, requires_grad=True)
            finally:
                net.requires_grad_(True)
        else:
            out = scorer.score(nodes, edges)
        assert scorer._bwd is None and not any(t.requires_grad for t in out), name
        assert all(t.grad_fn is None for t in out), name
        assert all(torch.equal(a, b.detach()) for a, b in zip(out, ref)), name


def test_no_molecules_and_a_one_atom_molecule():
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(4)
    net, _, _ = _net("GGNN")
    scorer = RouteScorer(net, 64, **GDB13)
    out = scorer.score(nodes[:0], edges[:0], requires_grad=True)
    assert out.likelihoods.numel() == 0 and out.offsets.tolist() == [0]
    g = torch.autograd.grad(out.nll.sum() + out.final.sum(), list(net.parameters()))
    assert all(not t.any() for t in g)
    one_n, one_e = np.zeros_like(nodes[:1]), np.zeros_like(edges[:1])
    one_n[0, 0, 1] = one_n[0, 0, 5 + 1] = 1                 # one atom of type 1, formal charge 0
    out = scorer.score(one_n, one_e, requires_grad=True)
    assert out.offsets.tolist() == [0, 2]
    loss_fn = _mixed_loss(2, 1, seed=9)
    got = torch.autograd.grad(loss_fn(out.likelihoods, out.nll, out.final), list(net.parameters()))
    p, _, nll, final = _eager_route(net, one_n, one_e, scorer.B)
    _assert_close_to_eager(got, torch.autograd.grad(loss_fn(p, nll, final), list(net.parameters())))


# ---- the kernels on guarded buffers -----------------------------------------------------------------------------
def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_kernels_stay_inside_their_buffers():
    from graphinvent_b200._lib import check, lib
    rng = np.random.default_rng(11)
    lengths = rng.integers(1, 12, 50)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    S, M = int(offsets[-1]), len(lengths)
    p = (rng.random(S) ** 3).astype(np.float32)
    p[rng.random(S) < 0.1] = 0.0
    p[offsets[2]:offsets[3]] = 0.0                       # a molecule of zero probabilities: no g_final term there
    g_lik, g_nll = rng.standard_normal(S).astype(np.float32), rng.standard_normal(M).astype(np.float32)
    g_fin = rng.standard_normal(M).astype(np.float32)
    g_fin[[p[a:e].sum() == 0 for a, e in zip(offsets[:-1], offsets[1:])]] = 0.0   # log(0) has no gradient
    G = lambda a: Guarded.like(torch.from_numpy(a).cuda())
    off, lik, gl, gn, gf = G(offsets), G(p), G(g_lik), G(g_nll), G(g_fin)
    q = lambda g: ctypes.c_void_p(g.ptr()) if g is not None else None
    for args in ((gl, gn, gf), (None, gn, None), (gl, None, gf)):
        coef = Guarded(4 * S)
        check(lib.gib_route_grad_coef(M, q(off), q(lik), *map(q, args), q(coef), _st()), "gib_route_grad_coef")
        want = coef_restated(p, offsets, *(None if a is None else b for a, b in zip(args, (g_lik, g_nll, g_fin))))
        got = coef.view(torch.float32, (S,)).cpu().numpy()
        # the kernel may contract a multiply-add in fp64: at most one fp32 rounding step apart
        assert np.all(np.abs(got - want) <= 2.5e-7 * np.abs(want) + 1e-30), np.abs(got - want).max()
        assert coef.intact(), coef.damage()
    # dlogits: 300 slots, every fourth a padding slot; p_out poisoned everywhere but the slots' places
    B, apd = 300, 625
    live = np.arange(B) % 4 != 3
    dst = np.full(B, -1, np.int32)
    dst[live] = rng.permutation(S)[: int(live.sum())]
    act = np.where(live, rng.integers(0, apd, B), -1).astype(np.int32)
    logits = (4 * rng.standard_normal((B, apd))).astype(np.float32)
    logits[5] *= 300                                      # a saturated row: p underflows, the row stays finite
    cf = rng.standard_normal(S).astype(np.float32)
    gl_, gs, gc = G(logits), G(np.concatenate([act, dst])), G(cf)
    dl, pout = Guarded(4 * B * apd), Guarded(4 * S)
    check(lib.gib_route_dlogits(B, apd, q(gl_), q(gs), q(gc), q(dl), q(pout), _st()), "gib_route_dlogits")
    d = dl.view(torch.float32, (B, apd)).cpu().double()
    po = pout.view(torch.float32, (S,)).cpu()
    sm = torch.softmax(torch.from_numpy(logits).double(), 1)
    for b in range(B):
        if not live[b]:
            assert (d[b] == 0).all() and not torch.signbit(d[b]).any(), b
            continue
        onehot = torch.zeros(apd, dtype=torch.float64)
        onehot[act[b]] = 1
        ref = float(cf[dst[b]]) * (onehot - sm[b])
        assert torch.isfinite(d[b]).all() and ((d[b] - ref).abs() <= 4e-6 * abs(float(cf[dst[b]])) + 1e-37).all(), b
        assert abs(po[dst[b]].item() - sm[b, act[b]].item()) <= 2e-6 * sm[b, act[b]].item() + 1e-37, b
    written = np.zeros(S, bool)
    written[dst[live]] = True
    assert torch.isnan(po[torch.from_numpy(~written)]).all()      # the poison of the places no slot owns
    for g in (off, lik, gl, gn, gf, gl_, gs, gc, dl, pout):
        assert g.intact(), g.damage()


# ---- memory -----------------------------------------------------------------------------------------------------
def _bytes(t):
    return t.numel() * t.element_size()


def test_memory_stays_within_the_static_buffers_and_the_record():
    """gdb13_1K/train at B = 1000, GGNN defaults: peak of score(requires_grad=True) + backward is the scorer's buffers,
    the backward's, the record and the gradients, not one forward workspace per batch of states; half the set peaks
    as high but for the smaller record"""
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import RouteScorer
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]
    torch.manual_seed(0)
    net = mpnn.create(make_constants("GGNN")).cuda().eval()
    peaks = []
    for M in (nodes.shape[0], nodes.shape[0] // 2):
        net.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        scorer = RouteScorer(net, 1000, **GDB13)
        out = scorer.score(nodes[:M], edges[:M], requires_grad=True)
        out.nll.mean().backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        static = sum(_bytes(t) for o in (scorer, scorer._bwd) for t in vars(o).values()
                     if isinstance(t, torch.Tensor) and t._base is None)
        S = out.likelihoods.numel()
        record = nodes[:M].nbytes + edges[:M].nbytes + 4 * S + 3 * 4 * M + 8 * (M + 1)
        grads = _bytes(scorer._bwd.gflat)
        assert peak <= static + record + grads + (256 << 20), (peak / 2**30, static / 2**30, S)
        peaks.append((peak, record))
        del scorer, out
    (p_full, r_full), (p_half, r_half) = peaks
    assert p_full - p_half <= (r_full - r_half) + (64 << 20), (p_full / 2**30, p_half / 2**30)


# ---- TF32 and bf16 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["tf32", "bf16"])
def test_reduced_precision_modes(mode):
    from graphinvent_b200.graphed import RouteScorer
    nodes, edges, _ = _fixture(24)
    net, _, _ = _net("GGNN")
    w = _weights(nodes.shape[0]).cuda()
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        if mode == "tf32":
            torch.backends.cuda.matmul.allow_tf32 = True
            scorer = RouteScorer(net, 256, **GDB13)
            p, _, nll, _ = _eager_route(net, nodes, edges, scorer.B)
            eager = torch.autograd.grad((w * nll).sum(), list(net.parameters()))
        else:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                scorer = RouteScorer(net, 256, **GDB13)
                p, _, nll, _ = _eager_route(net, nodes, edges, scorer.B)
                eager = torch.autograd.grad((w * nll).sum(), list(net.parameters()))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert scorer.tf32 == (mode == "tf32") and scorer.autocast_dtype == (torch.bfloat16 if mode == "bf16" else None)
    out, grads = _route_grads(scorer, net, nodes, edges, lambda o: (w * o.nll).sum())
    S = out.likelihoods.numel()
    assert torch.equal(scorer.lik[:S], out.likelihoods.detach())          # one chunk: the backward's recomputed p
    assert torch.allclose(p.float(), out.likelihoods, rtol=1e-5, atol=0)
    _assert_close_to_eager(grads, eager, rel=1e-3, what=mode)


# ---- fine-tuning ------------------------------------------------------------------------------------------------
def test_fine_tuning_tracks_eager_steps_and_lowers_the_nll():
    from graphinvent_b200.graphed import RouteScorer
    from graphinvent_b200.optim import FlatAdam
    z = np.load(os.path.join(GOLDEN, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"][:256], z["gdb13_1K_train/edges"][:256]
    (net, _, _), (twin, _, _) = _net("GGNN", seed=4), _net("GGNN", seed=4)
    opt, opt_e = FlatAdam(net.parameters(), lr=1e-4), FlatAdam(twin.parameters(), lr=1e-4)
    scorer = RouteScorer(net, 1000, **GDB13)
    losses = []
    for step in range(30):
        opt.zero_grad()
        loss = scorer.score(nodes, edges, requires_grad=True).nll.mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if step < 5:
            opt_e.zero_grad()
            _, _, nll, _ = _eager_route(twin, nodes, edges, scorer.B)
            le = nll.mean()
            le.backward()
            opt_e.step()
            assert abs(losses[-1] - le.item()) <= 1e-4 * abs(le.item()), (step, losses[-1], le.item())
    with torch.no_grad():
        final = scorer.score(nodes, edges).nll.mean().item()
    assert final < losses[0], (losses[0], final)
