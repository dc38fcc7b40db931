"""GPU: partial batches in the captured training step (graphed.TrainStep) and the validation pass as captured replays
(graphed.EvalStep).

  a. a stream full -> b -> full -> b' -> full -> b'' -> full, b in {1, 7, B - 1}, for the four models and float / int8
     inputs: the live logits equal a full batch's with the same first b molecules, the loss rows / dlogits / loss equal
     the host-argument entry points on the b live rows, the padding rows are +0, the gradient bucket equals a fresh
     C-ABI run on 0xFF-poisoned buffers, and an eager b-row twin (module API in capacity mode) agrees to rounding;
  b. the batch sizes the reference's BlockDataLoader yields (256 gdb13 rows, block 128, batch 100: 100, 28, 100, 28);
  c. data parallel: a short global batch split by shard_bounds, an empty rank included, two-graph step == one-graph step;
  d. EvalStep sharing a TrainStep: logits / KL / NLL rows against the step and the module-level kernels, both passes
     against restatements of the reference (Analyzer.py:734-778, Workflow.py:813-831), training with passes in between
     bit-identical to training without, check() after an overflowing or multi-type batch, the memory a pass adds, a
     dropout_p > 0 model in eval, and one pass per model against fp64.
"""
import copy
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_buffer_bounds import _bits_equal, _model_case

pytestmark = pytest.mark.gpu

MODELS = ["small_GGNN", "small_MNN", "small_AttGGNN", "small_EMN"]
CASES = [(m, dt) for m in MODELS for dt in (torch.float32, torch.int8)]
B = 32                                       # the small_* fixtures' batch


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _capacity(edges, C):
    from tests.k0_reference import ceil_tile
    e = edges != 0
    return ceil_tile(int(e.sum()) if C.model != "EMN" else int(e.any(-1).sum())) + 128


def _case(name, in_dtype):
    C, net, nodes, edges, target = _model_case(name)
    if in_dtype == torch.int8:
        nodes, edges = nodes.to(torch.int8), edges.to(torch.int8)
    return C, net, nodes, edges, target


def _batches(nodes, edges, target):
    """the stream: full, b, full (rolled), b', full, b'', full -- the short batches' molecules come from the middle"""
    out = []
    for k, b in enumerate((B, 1, B, 7, B, B - 1, B)):
        idx = (torch.arange(B, device=nodes.device) + 5 * k) % B
        out.append((nodes[idx][:b].contiguous(), edges[idx][:b].contiguous(), target[idx][:b].contiguous()))
    return out


def _padded(x, n=B):
    pad = torch.zeros((n - x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    return torch.cat([x, pad])


def fresh_ctl_step(net, nodes, edges, target, cap, live, scale):
    """K0 -> pack -> forward -> _ctl loss -> backward through the C-ABI on freshly allocated 0xFF-poisoned buffers
    (the gradient bucket zeroed): what one replay of TrainStep computes on the padded batch"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import BatchCtl, check, lib
    n = nodes.shape[0]
    d = Fn.make_dims(net, n, Fn.input_dtype_code(nodes, edges))
    bd, st = ctypes.byref(d), _st()
    params = [p.detach() for p in net.parameters()]
    apd = target.shape[1]

    def poison(nbytes):
        return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    cws = poison(lib.gib_graph_count_ws_bytes(bd))
    check(lib.gib_graph_count(bd, Fn._ptr(edges), Fn._ptr(cws), st), "gib_graph_count")
    hdr = np.zeros(16, np.int32)
    check(lib.gib_graph_header_capacity(bd, int(cap), Fn._ptr(cws), hdr.ctypes.data_as(ctypes.c_void_p)), "hdr")
    hp = hdr.ctypes.data_as(ctypes.c_void_p)
    graph = poison(lib.gib_graph_bytes(bd, hp))
    check(lib.gib_graph_fill(bd, Fn._ptr(edges), Fn._ptr(cws), hp, Fn._ptr(graph), st), "gib_graph_fill")
    packed = poison(lib.gib_model_packed_bytes(bd))
    check(lib.gib_model_pack(bd, Fn._ptr_table(params), Fn._ptr(packed), st), "gib_model_pack")
    ws = poison(lib.gib_model_workspace_bytes(bd, hp))
    out = poison(n * apd * 4).view(torch.float32).view(n, apd)
    check(lib.gib_model_forward(bd, hp, Fn._ptr(nodes), Fn._ptr(edges), Fn._ptr(graph), Fn._ptr(packed), Fn._ptr(ws),
                                Fn._ptr(out), st), "gib_model_forward")
    ctl = torch.frombuffer(bytearray(BatchCtl(live, scale)), dtype=torch.uint8).cuda()
    rows = poison(n * 4).view(torch.float32)
    dout = poison(n * apd * 4).view(torch.float32).view(n, apd)
    loss = poison(4).view(torch.float32)
    check(lib.gib_kl_loss_fwd_bwd_ctl(Fn._ptr(out), Fn._ptr(target), n, apd, Fn._ptr(ctl), Fn._ptr(rows), Fn._ptr(dout),
                                      st), "gib_kl_loss_fwd_bwd_ctl")
    check(lib.gib_sum_scaled_ctl(Fn._ptr(rows), n, Fn._ptr(ctl), Fn._ptr(loss), st), "gib_sum_scaled_ctl")
    total = sum(p.numel() for p in params)
    gflat = torch.zeros(total, dtype=torch.float32, device="cuda")
    views, o = [], 0
    for p in params:
        views.append(gflat[o:o + p.numel()])
        o += p.numel()
    scratch = poison(lib.gib_model_bwd_scratch_bytes(bd, hp))
    check(lib.gib_model_backward(bd, hp, Fn._ptr(nodes), Fn._ptr(edges), Fn._ptr(graph), Fn._ptr(packed), Fn._ptr(ws),
                                 Fn._ptr(out), Fn._ptr(dout), Fn._ptr_table(views), Fn._ptr(scratch), st),
          "gib_model_backward")
    torch.cuda.synchronize()
    return dict(out=out, rows=rows, dout=dout, loss=loss, gflat=gflat)


def _host_kl(out, target, scale):
    """gib_kl_loss_fwd_bwd / gib_sum_scaled with host arguments"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import check, lib
    n, apd = out.shape
    rows = torch.empty(n, device="cuda")
    dout = torch.empty_like(out)
    loss = torch.empty(1, device="cuda")
    check(lib.gib_kl_loss_fwd_bwd(Fn._ptr(out), Fn._ptr(target), n, apd, scale, Fn._ptr(rows), Fn._ptr(dout), _st()), "")
    check(lib.gib_sum_scaled(Fn._ptr(rows), n, scale, Fn._ptr(loss), _st()), "")
    return rows, dout, loss


def _zero_bits(t):
    return bool((t.reshape(-1).view(torch.int32) == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# a. partial batches in TrainStep
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,in_dtype", CASES, ids=[f"{m}-{str(d)[6:]}" for m, d in CASES])
def test_partial_batches_in_a_stream(case, in_dtype):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import TrainStep
    C, net, nodes, edges, target = _case(case, in_dtype)
    cap = _capacity(edges, C)
    opt = torch.optim.SGD(net.parameters(), lr=0.0)         # the weights stay: every replay has one fresh reference
    step = TrainStep(net, opt, batch_size=B, entry_capacity=cap, input_dtype=in_dtype)
    eager = copy.deepcopy(net)
    eager.entry_capacity = cap
    for k, (n, e, t) in enumerate(_batches(nodes, edges, target)):
        b = n.shape[0]
        what = f"{case} step {k + 1}, b = {b}"
        loss = step(n, e, t)
        torch.cuda.synchronize()
        step.check()
        scale = float(np.float32(1.0 / b))
        fresh = fresh_ctl_step(net, _padded(n), _padded(e), _padded(t), cap, b, scale)
        for name in ("out", "rows", "dout", "gflat"):
            assert _bits_equal(getattr(step, name), fresh[name]), (what, name)
        assert _bits_equal(loss.view(1), fresh["loss"]), what
        # the live molecules' logits are those of a full batch with the same first b molecules
        full = fresh_ctl_step(net, torch.cat([n, nodes[b:]]), torch.cat([e, edges[b:]]), torch.cat([t, target[b:]]),
                              cap, B, float(np.float32(1.0 / B)))
        assert _bits_equal(step.out[:b], full["out"][:b]), what
        rows, dout, ls = _host_kl(step.out[:b].contiguous(), t, scale)
        assert _bits_equal(step.rows[:b], rows) and _bits_equal(step.dout[:b], dout), what
        assert _bits_equal(loss.view(1), ls), what
        assert _zero_bits(step.rows[b:]) and _zero_bits(step.dout[b:]), what
        # the eager b-row twin plans its GEMMs for b molecules: equal to rounding, not bit for bit
        eager.zero_grad(set_to_none=True)
        out_e = eager(n, e)
        loss_e = Fn.kl_loss(out_e, t)
        loss_e.backward()
        assert torch.allclose(step.out[:b], out_e.detach(), rtol=1e-4, atol=1e-4), what
        assert abs(float(loss) - float(loss_e.detach())) <= 1e-5 * max(1.0, abs(float(loss_e.detach()))), what
        for (name, p), v in zip(eager.named_parameters(), step.views):
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            err = float((v - g).norm()) / max(float(g.norm()), 1e-6)
            assert err <= 1e-3, (what, name, err)


def test_partial_batch_gradients_are_fp64_anchored():
    """the gradients of a 7-row batch run through the padded step, against the fp64 oracle of those 7 rows"""
    from oracle import mpnn_oracle as O
    from graphinvent_b200.graphed import TrainStep
    from tests.test_gpu_parity import FP64_C
    for case in MODELS:
        C, net, nodes, edges, target = _case(case, torch.float32)
        cap = _capacity(edges, C)
        sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
        step = TrainStep(net, torch.optim.SGD(net.parameters(), lr=0.0), batch_size=B, entry_capacity=cap)
        b = 7
        step(nodes[:b], edges[:b], target[:b])
        torch.cuda.synchronize()
        args = (sd, C, nodes[:b].cpu(), edges[:b].cpu(), target[:b].cpu())
        _, _, g32 = O.train_step_grads(*args)
        _, _, g64 = O.train_step_grads(*args, dtype=torch.float64)
        gscale = max(g.norm().item() for g in g64.values())
        for (name, _), v in zip(net.named_parameters(), step.views):
            e_ref = (g32[name].double() - g64[name]).norm().item()
            e_got = (v.detach().cpu().double() - g64[name]).norm().item()
            assert e_got <= FP64_C * e_ref + 1e-4 * gscale, (case, name, e_got, e_ref, gscale)


def _gdb13():
    from oracle import mpnn_oracle as O
    from tests.conftest import load_gdb13
    g = load_gdb13()
    C = O.make_constants("GGNN")
    net = _net(C)
    return C, net, g["nodes"].cuda(), g["edges"].cuda(), g["apds"].cuda()


def _net(C, seed=0):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=seed))
    return net.cuda()


def _block_loader(nodes, edges, target, block=128, batch=100):
    """BlockDataLoader with drop_last=False (its `condition` is False for these sizes): every block's tail batch"""
    out = []
    for s in range(0, nodes.shape[0], block):
        for c in range(s, min(s + block, nodes.shape[0]), batch):
            hi = min(c + batch, s + block, nodes.shape[0])
            out.append((nodes[c:hi], edges[c:hi], target[c:hi]))
    return out


def test_the_reference_loaders_batch_sizes_train():
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    C, net, nodes, edges, target = _gdb13()
    loader = _block_loader(nodes, edges, target)
    assert [x[0].shape[0] for x in loader] == [100, 28, 100, 28]
    twin = copy.deepcopy(net)
    opt = FlatAdam(net.parameters(), lr=1e-4)
    step = TrainStep(net, opt, batch_size=100, entry_capacity=_capacity(edges, C) + 4096)
    for n, e, t in loader:
        with torch.no_grad():
            twin.load_state_dict(net.state_dict())
            want = float(Fn.kl_loss(twin(n, e), t))
        loss = float(step(n, e, t))
        step.check()
        assert np.isfinite(loss) and abs(loss - want) <= 1e-5 * max(1.0, abs(want)), (n.shape[0], loss, want)
    assert all(torch.isfinite(p).all() for p in net.parameters())


# ---------------------------------------------------------------------------------------------------------------------
# c. a short global batch over two ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", [B + 9, 1])
def test_short_global_batch_over_two_ranks(g, monkeypatch):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.parallel import shard_bounds
    C, net, nodes, edges, target = _case("small_GGNN", torch.float32)
    nodes, edges, target = (torch.cat([x, x])[:g] for x in (nodes, edges, target))
    cap = _capacity(edges, C) + 512
    local = (B + 9 + 1) // 2
    dist = torch.distributed
    for rank in range(2):
        lo, hi = shard_bounds(g, rank, 2)
        net1, net2 = copy.deepcopy(net), copy.deepcopy(net)
        one = TrainStep(net1, torch.optim.SGD(net1.parameters(), lr=1e-3), batch_size=local, entry_capacity=cap,
                        global_batch=2 * local, group=False)
        with monkeypatch.context() as mp:
            mp.setattr(dist, "is_initialized", lambda: True)
            mp.setattr(dist, "get_world_size", lambda group=None: 2)
            mp.setattr(dist, "all_reduce", lambda tensor, *a, **kw: None)
            two = TrainStep(net2, torch.optim.SGD(net2.parameters(), lr=1e-3), batch_size=local, entry_capacity=cap,
                            global_batch=2 * local)
            assert two.world == 2
            with pytest.raises(ValueError, match="global batch"):
                two.load(nodes[lo:lo], edges[lo:lo], target[lo:lo])
            l2 = two(nodes[lo:hi], edges[lo:hi], target[lo:hi], global_batch=g)
        l1 = one(nodes[lo:hi], edges[lo:hi], target[lo:hi], global_batch=g)
        torch.cuda.synchronize()
        assert _bits_equal(one.gflat, two.gflat) and _bits_equal(l1.view(1), l2.view(1)), (g, rank)
        for p, q in zip(net1.parameters(), net2.parameters()):
            assert _bits_equal(p.detach(), q.detach()), (g, rank)
        if hi == lo:                                          # the empty rank: loss 0, gradient 0
            assert float(l1) == 0.0 and bool((one.gflat == 0).all()), (g, rank)
        else:
            fresh = fresh_ctl_step(net, _padded(nodes[lo:hi], local), _padded(edges[lo:hi], local),
                                   _padded(target[lo:hi], local), cap, hi - lo, float(np.float32(1.0 / g)))
            assert _bits_equal(one.gflat, fresh["gflat"]), (g, rank)


# ---------------------------------------------------------------------------------------------------------------------
# d. EvalStep
# ---------------------------------------------------------------------------------------------------------------------
class _Loader(list):
    """a list of batches whose len() can claim more batches than it yields (a slot the pass never fills stays 0)"""

    def __init__(self, batches, length=None):
        super().__init__(batches)
        self.length = length

    def __len__(self):
        return self.length if self.length is not None else list.__len__(self)


def ref_validation_likelihood(batches, logits, n_samples, batch_size, N):
    """Analyzer.py:734-778 on precomputed logits, the row values from functional.validation_nll"""
    from graphinvent_b200 import functional as Fn
    n = min(100000, n_samples)
    lik = torch.zeros(n * (N + 5), device="cuda")
    n_structures = torch.zeros(1, device="cuda")
    for idx, ((_, _, t), out) in enumerate(zip(batches, logits)):
        if idx * batch_size > n:
            break
        v = Fn.validation_nll(out, t)
        v = v[~torch.isnan(v)]
        lik[idx * batch_size: idx * batch_size + len(v)] = v
        n_structures += torch.sum(t[:, -1]).unsqueeze(dim=0)
    return lik, torch.sum(lik, dim=0) / n_structures[0], n_structures


def _logits_of(ev, batches):
    """each batch's logits as the captured pass computes them (one single-batch pass each)"""
    out = []
    for bt in batches:
        ev.validation_epoch([bt])
        out.append(ev.out[:bt[0].shape[0]].clone())
    return out


def _eval_batches(nodes, edges, target):
    """five batches of the fixture: NaN rows (all-zero targets) at the start, middle and end of one, an all-NaN batch,
    a short last batch"""
    t1 = target.clone()
    t1[[0, B // 2, B - 1]] = 0
    t2 = torch.zeros_like(target)
    roll = lambda x, s: torch.roll(x, s, 0)                  # noqa: E731
    return [(nodes, edges, target), (roll(nodes, 3), roll(edges, 3), t1), (roll(nodes, 9), roll(edges, 9), t2),
            (roll(nodes, 1), roll(edges, 1), roll(target, 1)), (nodes[:11], edges[:11], target[:11])]


@pytest.mark.parametrize("case,in_dtype", CASES, ids=[f"{m}-{str(d)[6:]}" for m, d in CASES])
def test_eval_step_shares_a_train_step_and_restates_the_reference(case, in_dtype):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import EvalStep, TrainStep
    C, net, nodes, edges, target = _case(case, in_dtype)
    cap = _capacity(edges, C)
    step = TrainStep(net, torch.optim.SGD(net.parameters(), lr=0.0), batch_size=B, entry_capacity=cap,
                     input_dtype=in_dtype)
    ev = EvalStep(net, batch_size=B, entry_capacity=cap, input_dtype=in_dtype, share=step)
    assert ev.out is step.out and ev.ws is step.ws and ev.packed is step.packed and ev.nodes is step.nodes
    # logits, KL and NLL rows against the training step's forward and the module-level kernels
    for b in (B, 7):
        val = ev.validation_epoch([(nodes[:b], edges[:b], target[:b])])
        torch.cuda.synchronize()
        got = ev.out[:b].clone()
        step(nodes[:b], edges[:b], target[:b])
        torch.cuda.synchronize()
        assert _bits_equal(got, step.out[:b]), (case, b)
        rows, _, _ = _host_kl(got.contiguous(), target[:b], 1.0 / b)
        assert _bits_equal(ev.rows[:b], rows) and _zero_bits(ev.rows[b:]), (case, b)
        assert _bits_equal(ev.nll[:b], Fn.validation_nll(got, target[:b])), (case, b)
        exact = float(rows.double().sum()) / b
        assert abs(float(val) - exact) <= 2.0 ** -24 * ((b - 1) * float(rows.double().abs().sum()) / b + 2 * abs(exact))
    batches = _eval_batches(nodes, edges, target)
    logits = _logits_of(ev, batches)
    N = C.max_n_nodes
    # validation_likelihood: several n_samples, none a multiple of B, one that stops before the last batch
    for n_samples in (4 * B + 5, 2 * B - 3, 10 ** 6):
        lik, avg = ev.validation_likelihood(_Loader(batches), n_samples)
        ref, ref_avg, ns = ref_validation_likelihood(batches, logits, n_samples, B, N)
        assert _bits_equal(lik, ref), (case, n_samples)
        off = ev._pass.view(torch.float32)[8]                  # gib_eval_pass.n_structures
        assert float(off) == float(ns[0]), (case, n_samples)
        assert _bits_equal(avg.view(1), ref_avg.view(1)), (case, n_samples)
        ev.check()
    # validation_epoch: each slot to the float32 bound of its row sum; a NaN target row -> NaN; unfilled slots stay 0
    val = ev.validation_epoch(_Loader([batches[0], batches[3], batches[4]], length=5))
    slots = []
    for (_, _, t), out in zip([batches[0], batches[3], batches[4]], [logits[0], logits[3], logits[4]]):
        rows, _, _ = _host_kl(out.contiguous(), t, 1.0)
        slots.append(float(rows.double().sum()) / t.shape[0])
    want = sum(slots) / 5
    assert abs(float(val) - want) <= 1e-6 * abs(want), (case, float(val), want)
    assert torch.isnan(ev.validation_epoch(_Loader(batches[:2]))), case
    with pytest.raises(IndexError):
        ev.validation_epoch(_Loader(batches[:3], length=2))


def test_likelihood_buffer_overflow_raises():
    from graphinvent_b200.graphed import EvalStep
    C, net, nodes, edges, target = _case("small_GGNN", torch.float32)
    ev = EvalStep(net, batch_size=B, entry_capacity=_capacity(edges, C))
    # n_samples = 2: a buffer of 2 * (7 + 5) = 24 floats, the first batch has 32 non-NaN rows
    with pytest.raises(RuntimeError, match="past the end"):
        ev.validation_likelihood([(nodes, edges, target)], 2)
    assert ev.clipped == B - 2 * (C.max_n_nodes + 5)
    lik, _ = ev.validation_likelihood([(nodes[:3], edges[:3], target[:3])], 2)   # 3 rows fit
    assert int((lik != 0).sum()) == 3


def test_training_with_eval_passes_in_between_is_unchanged():
    from graphinvent_b200.graphed import EvalStep, TrainStep
    from graphinvent_b200.optim import FlatAdam
    for case in MODELS:
        C, net, nodes, edges, target = _case(case, torch.float32)
        cap = _capacity(edges, C)
        stream = _batches(nodes, edges, target)
        evb = _eval_batches(nodes, edges, target)
        runs = []
        for with_eval in (False, True):
            m = copy.deepcopy(net)
            opt = FlatAdam(m.parameters(), lr=1e-3)
            step = TrainStep(m, opt, batch_size=B, entry_capacity=cap)
            ev = EvalStep(m, batch_size=B, entry_capacity=cap, share=step) if with_eval else None
            losses = []
            for n, e, t in stream:
                losses.append(step(n, e, t).clone())
                if ev is not None:
                    ev.validation_epoch(evb)
                    ev.validation_likelihood(evb, 3 * B)
            torch.cuda.synchronize()
            runs.append((torch.stack(losses), opt._flat.clone(), opt._m.clone(), opt._v.clone()))
        for name, a, b in zip(("losses", "parameters", "exp_avg", "exp_avg_sq"), *runs):
            assert _bits_equal(a, b), (case, name)


def test_check_raises_after_an_overflowing_or_multitype_pass():
    from graphinvent_b200.graphed import EvalStep
    C, net, nodes, edges, target = _case("small_GGNN", torch.float32)
    assert int((edges[:4] != 0).sum()) <= 128 < int((edges != 0).sum())
    ev = EvalStep(net, batch_size=B, entry_capacity=128)
    ev.validation_epoch([(nodes[:4], edges[:4], target[:4])])
    ev.check()
    ev.validation_epoch([(nodes[:4], edges[:4], target[:4]), (nodes, edges, target), (nodes[:4], edges[:4], target[:4])])
    with pytest.raises(RuntimeError, match="entry_capacity"):
        ev.check()
    ev.validation_epoch([(nodes[:4], edges[:4], target[:4])])
    ev.check()                                              # the next pass starts clean
    C, net, nodes, edges, target = _case("small_AttGGNN", torch.float32)
    e2 = edges.clone()
    b, i, j = [int(x) for x in torch.nonzero(e2[..., 0])[0]]
    e2[b, i, j, 1] = e2[b, j, i, 1] = 1.0                    # a bond of two types
    ev = EvalStep(net, batch_size=B, entry_capacity=_capacity(e2, C))
    ev.validation_likelihood([(nodes, edges, target), (nodes, e2, target)], 10 ** 6)
    with pytest.raises(RuntimeError, match="one bond type"):
        ev.check()


def test_a_shared_pass_adds_only_its_slots_and_likelihood_buffer():
    from graphinvent_b200.graphed import EvalStep, TrainStep
    C, net, nodes, edges, target = _gdb13()
    cap = _capacity(edges, C) + 4096
    step = TrainStep(net, torch.optim.SGD(net.parameters(), lr=0.0), batch_size=100, entry_capacity=cap)
    ev = EvalStep(net, batch_size=100, entry_capacity=cap, share=step)
    loader = _block_loader(nodes, edges, target)
    step(*loader[0])
    ev.validation_epoch(loader)
    ev.validation_likelihood(loader, 250)
    torch.cuda.synchronize()

    def rounded(nbytes):
        return (nbytes + 511) // 512 * 512
    for run, extra in ((lambda: ev.validation_epoch(loader), rounded(4 * len(loader))),
                       (lambda: ev.validation_likelihood(loader, 250), rounded(4 * 250 * (13 + 5)))):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        run()
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base <= extra + 4 * 512, (extra,)


def test_dropout_model_evaluates_as_its_dropout_free_twin():
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import EvalStep
    C0, net0, nodes, edges, target = _case("small_GGNN", torch.float32)
    C1 = C0._replace(enn_dropout_p=0.2, mlp1_dropout_p=0.1, mlp2_dropout_p=0.3, gather_att_dropout_p=0.1)
    net1 = mpnn.create(C1)
    net1.load_state_dict(net0.state_dict())
    net1 = net1.cuda().eval()
    assert any(p > 0 for p in net1._dropout_ps())
    res = []
    for m in (net0.eval(), net1):
        ev = EvalStep(m, batch_size=B, entry_capacity=_capacity(edges, C0))
        val = ev.validation_epoch([(nodes, edges, target)])
        res.append((val.view(1).clone(), ev.out.clone(), ev.validation_likelihood([(nodes, edges, target)], B)[0]))
    for a, b in zip(*res):
        assert _bits_equal(a, b)


@pytest.mark.parametrize("case", MODELS)
def test_eval_pass_is_fp64_anchored(case):
    from oracle import mpnn_oracle as O
    from graphinvent_b200.graphed import EvalStep
    from tests.test_gpu_parity import FP64_C, LOGIT_TOL
    C, net, nodes, edges, target = _case(case, torch.float32)
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    ev = EvalStep(net, batch_size=B, entry_capacity=_capacity(edges, C))
    val = ev.validation_epoch([(nodes, edges, target)])
    out = ev.out.detach().cpu().double()
    l32, o32, _ = O.train_step_grads(sd, C, nodes.cpu(), edges.cpu(), target.cpu())
    l64, o64, _ = O.train_step_grads(sd, C, nodes.cpu(), edges.cpu(), target.cpu(), dtype=torch.float64)
    e_ref = (o32.double() - o64).abs().max(1).values
    e_got = (out - o64).abs().max(1).values
    assert float((e_got - FP64_C * e_ref - LOGIT_TOL).max()) <= 0, case
    assert abs(float(val) - float(l64)) <= FP64_C * abs(float(l32) - float(l64)) + 1e-5, case


def test_share_refuses_a_train_step_of_other_dims():
    from graphinvent_b200.graphed import EvalStep, TrainStep
    C, net, nodes, edges, target = _case("small_GGNN", torch.float32)
    cap = _capacity(edges, C)
    step = TrainStep(net, torch.optim.SGD(net.parameters(), lr=0.0), batch_size=B, entry_capacity=cap)
    for kw in (dict(batch_size=B - 1, entry_capacity=cap), dict(batch_size=B, entry_capacity=cap + 128),
               dict(batch_size=B, entry_capacity=cap, input_dtype=torch.int8)):
        with pytest.raises(ValueError, match="share"):
            EvalStep(net, share=step, **kw)
    with pytest.raises(ValueError, match="up to 32 molecules"):
        step(torch.cat([nodes, nodes[:1]]), torch.cat([edges, edges[:1]]), torch.cat([target, target[:1]]))
