"""GPU: fp16 training in the captured step with dynamic loss scaling on the device (TrainStep(grad_scaler=)).

1. The kernels on their own: the non-finite check (positions, values, guard bands), the scale update against
   torch._amp_update_scale_, and the gated Adam against the host-count gib_adam_step after GradScaler's unscale.
2. The whole step against the eager `scaler.scale(loss).backward(); scaler.step(opt); scaler.update()` loop, bit for bit,
   over a stream with overflowing first steps, a short batch and growth; checkpoint resume; no host synchronisation;
   50 steps near the fp32 loss curve; a shared EvalStep; data parallel on >= 2 GPUs.
"""
import copy
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tests.test_gpu_tf32 as T
from tests.conftest import GOLDEN, MODELS, ROOT, load_small

pytestmark = pytest.mark.gpu
FP16 = torch.float16


def _lib():
    from graphinvent_b200._lib import lib
    return lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.detach().reshape(-1).view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a.float().contiguous()), _bits(b.float().contiguous()))


# ---- 1. kernels ------------------------------------------------------------------------------------------------------
def _check(x, flag):
    assert _lib().gib_nonfinite_check(_p(x), x.numel(), _p(flag), _st()) == 0, _lib().gib_last_error()


@pytest.mark.parametrize("n", [1, 7, 13, 4 * 132 * 8 * 256 * 3 + 7])
def test_nonfinite_check_positions_values_and_guards(n):
    g = torch.Generator(device="cuda").manual_seed(n)
    guard = 64
    base = torch.randn(n + 2 * guard + 1, generator=g, device="cuda") * 1e3
    base[:guard + 1] = float("nan")             # guards, and the element that makes x start 4 bytes past a 16-byte line
    base[guard + 1 + n:] = float("inf")
    x = base[guard + 1:guard + 1 + n]
    assert x.data_ptr() % 16 != 0
    flagbuf = torch.tensor([7.0, 0.0, 9.0], device="cuda")
    flag = flagbuf[1:2]
    positions = sorted({0, n - 1, min(1, n - 1), min(2, n - 1), max(n - 2, 0), max(n - 3, 0), n // 2 + 1 if n > 2 else 0})
    _check(x, flag)
    assert flag.item() == 0.0, "clean buffer flagged (or the guards were read)"
    for pos in positions:
        for bad in (float("inf"), float("-inf"), float("nan")):
            keep = x[pos].clone()
            x[pos] = bad
            flag.zero_()
            _check(x, flag)
            assert flag.item() == 1.0, (pos, bad)
            x[pos] = keep
        for fine in (1e-45, -1e-45, 3.4028234663852886e38, -3.4028234663852886e38, -0.0):
            keep = x[pos].clone()
            x[pos] = fine
            flag.zero_()
            _check(x, flag)
            assert flag.item() == 0.0, (pos, fine)
            x[pos] = keep
    flag.fill_(1.0)
    snapshot = base.clone()
    _check(x, flag)
    assert flag.item() == 1.0, "the check cleared the flag"
    assert torch.equal(flagbuf[0::2], torch.tensor([7.0, 9.0], device="cuda")), "wrote outside the flag"
    assert torch.equal(_bits(base), _bits(snapshot)), "the check wrote into the buffer"


SCALE_CASES = [
    dict(init=2.0 ** 16, growth=2.0, backoff=0.5, interval=3),
    dict(init=1000.3, growth=1.7, backoff=0.3, interval=2),
    dict(init=2.0e38, growth=2.0, backoff=0.5, interval=1),          # growth to inf is refused
    dict(init=3.0e-3, growth=1.1, backoff=0.9, interval=4),
    dict(init=6.0e37, growth=3.3, backoff=0.77, interval=2),
]
FOUND = [0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0]


@pytest.mark.parametrize("case", range(len(SCALE_CASES)))
def test_scale_update_equals_torch(case):
    c = SCALE_CASES[case]
    s_t = torch.full((), c["init"], dtype=torch.float32, device="cuda")
    g_t = torch.zeros((), dtype=torch.int32, device="cuda")
    s_m, g_m = s_t.clone(), g_t.clone()
    counts = torch.tensor([5, 0, 2], dtype=torch.int64, device="cuda")
    want_counts = counts.clone()
    f = torch.zeros((), dtype=torch.float32, device="cuda")
    grew = 0
    for k, bad in enumerate(FOUND):
        f.fill_(float(bad))
        before = s_t.item()
        torch._amp_update_scale_(s_t, g_t, f, c["growth"], c["backoff"], c["interval"])
        assert _lib().gib_amp_update_scale(_p(s_m), _p(g_m), _p(f), c["growth"], c["backoff"], c["interval"],
                                           _p(counts), counts.numel(), _st()) == 0
        if not bad:
            want_counts += 1
        assert _same(s_m, s_t) and torch.equal(g_m, g_t), (case, k, s_m.item(), s_t.item())
        assert torch.equal(counts, want_counts), (case, k)
        grew += s_t.item() > before
    assert np.isfinite(s_m.item())
    if case != 2:
        assert grew > 0
    else:
        assert s_m.item() < 3.5e38 and s_m.item() != float("inf")


def _adam_pair(seed):
    """two FlatAdams over equal parameters in three groups (one with weight decay)"""
    from graphinvent_b200.optim import FlatAdam
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = [(37,), (64, 33), (5,), (1000, 3), (2,), (129,)]
    ps = [torch.randn(s, generator=g, device="cuda") for s in shapes]
    opts = []
    for _ in range(2):
        q = [torch.nn.Parameter(p.clone()) for p in ps]
        groups = [dict(params=q[0:2]), dict(params=q[2:4], weight_decay=0.01), dict(params=q[4:], lr=3e-3)]
        opts.append((q, FlatAdam(groups, lr=1e-3, betas=(0.9, 0.999))))
    return opts, g


def _grad_bucket(params, values):
    flat = values.clone()
    o = 0
    for p in params:
        p.grad = flat[o:o + p.numel()].view(p.shape)
        o += p.numel()
    return flat


def test_gated_adam_equals_the_host_step_after_unscale():
    opts, g = _adam_pair(3)
    (ref_p, ref), (dev_p, dev) = opts
    total = sum(p.numel() for p in ref_p)
    scaler = torch.amp.GradScaler("cuda", init_scale=3000.7, growth_factor=1.37, backoff_factor=0.61,
                                  growth_interval=2)
    scaler._lazy_init_scale_growth_tracker(torch.device("cuda"))
    schs = [torch.optim.lr_scheduler.OneCycleLR(o, max_lr=1e-2, total_steps=40) for o in (ref, dev)]
    assert ref.param_groups[0]["betas"] != (0.9, 0.999)            # cycle_momentum moves beta1
    found = torch.zeros((), dtype=torch.float32, device="cuda")
    skips = [0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1, 0, 0, 0]
    taken = 0
    for k, skip in enumerate(skips):
        s = scaler._scale.clone()
        raw = torch.randn(total, generator=g, device="cuda") * s
        inv = s.double().reciprocal().float()
        gref = _grad_bucket(ref_p, raw)
        _grad_bucket(dev_p, raw)
        torch._amp_foreach_non_finite_check_and_unscale_([gref], torch.zeros_like(found), inv)
        before = [t.clone() for t in (dev._flat, dev._m, dev._v)]
        found.fill_(float(skip))
        dev.scaled_step(found, scaler)
        assert dev.launches_last_step == 3
        if not skip:
            ref.step()
            taken += 1
        for sch in schs:
            sch.step()
        torch.cuda.synchronize()
        for name, a, b in (("p", dev._flat, ref._flat), ("m", dev._m, ref._m), ("v", dev._v, ref._v)):
            assert _same(a, b), (k, name)
        if skip:
            for a, b in zip((dev._flat, dev._m, dev._v), before):
                assert _same(a, b), k
        assert dev.device_step_counts().tolist() == [taken] * len(dev_p), k
    assert [int(v["step"]) for v in dev.state_dict()["state"].values()] == [taken] * len(dev_p)
    assert ref._steps == [taken] * len(ref_p)


# ---- 2. the whole step -----------------------------------------------------------------------------------------------
SCALER_KW = dict(init_scale=2.0 ** 28, growth_factor=2.0, backoff_factor=0.125, growth_interval=3)


def _stream(fx, int8):
    """batches of the fixture: permutations, a short batch and a repeat"""
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    if int8:
        nodes, edges = nodes.to(torch.int8), edges.to(torch.int8)
    B = nodes.shape[0]
    out = []
    for k in range(9):
        g = torch.Generator(device="cuda").manual_seed(k)
        perm = torch.randperm(B, device="cuda", generator=g)
        if k == 5:
            perm = perm[:B - 3]
        out.append((nodes[perm].contiguous(), edges[perm].contiguous(), target[perm].contiguous()))
    return out


def _scaled_step(fx, cap, int8, scaler, lr=1e-3):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    net = T._net(fx["C"], fx["sd"])
    opt = FlatAdam(net.parameters(), lr=lr)
    with torch.autocast("cuda", dtype=FP16):
        step = TrainStep(net, opt, batch_size=fx["nodes"].shape[0], entry_capacity=cap,
                         input_dtype=torch.int8 if int8 else torch.float32, grad_scaler=scaler)
    assert step.autocast_dtype is FP16 and step.d.tf32 == 3
    return step, net, opt


def _eager(fx, cap, lr=1e-3):
    from graphinvent_b200.optim import FlatAdam
    net = T._net(fx["C"], fx["sd"])
    net.entry_capacity = cap
    return net, FlatAdam(net.parameters(), lr=lr), torch.amp.GradScaler("cuda", **SCALER_KW)


def _eager_step(net, opt, scaler, batch):
    from graphinvent_b200 import functional as Fn
    n_, e_, t_ = batch
    with torch.autocast("cuda", dtype=FP16):
        out = net(n_, e_)
    opt.zero_grad(set_to_none=True)
    scaler.scale(Fn.kl_loss(out, t_)).backward()
    scaler.step(opt)
    scaler.update()
    return out.detach()


def _package_loss(out, target):
    """the captured step's loss arithmetic (the host-argument forms of its _ctl kernels) on given logits"""
    lib = _lib()
    b, apd = out.shape
    rows = torch.empty(b, device="cuda")
    loss = torch.empty(1, device="cuda")
    scale = 1.0 / b
    assert lib.gib_kl_loss_fwd_bwd(_p(out), _p(target), b, apd, ctypes.c_float(scale), _p(rows), None, _st()) == 0
    assert lib.gib_sum_scaled(_p(rows), b, ctypes.c_float(scale), _p(loss), _st()) == 0
    return loss


def _compare(step, opt, scaler, net_e, opt_e, scaler_e, what):
    for p, q in zip(step.params, net_e.parameters()):
        assert _same(p, q), what + ": parameters"
    assert _same(opt._m, opt_e._m) and _same(opt._v, opt_e._v), what + ": moments"
    assert scaler.get_scale() == scaler_e.get_scale(), what + ": scale"
    assert scaler._get_growth_tracker() == scaler_e._get_growth_tracker(), what + ": growth tracker"
    assert opt.device_step_counts().tolist() == opt_e._steps, what + ": step counts"


@pytest.mark.parametrize("int8", [False, True])
@pytest.mark.parametrize("model", MODELS)
def test_fp16_scaled_step_equals_the_eager_scaler_loop(model, int8):
    fx = load_small(model)
    cap = int(fx["edges"].sum().item()) + 64
    batches = _stream(fx, int8)
    scaler = torch.amp.GradScaler("cuda", **SCALER_KW)
    step, net, opt = _scaled_step(fx, cap, int8, scaler)
    net_e, opt_e, scaler_e = _eager(fx, cap)
    skipped, grown = 0, 0
    for k, batch in enumerate(batches):
        s0 = scaler_e.get_scale()
        loss = step(*batch)
        out_e = _eager_step(net_e, opt_e, scaler_e, batch)
        torch.cuda.synchronize()
        b = batch[0].shape[0]
        what = f"{model} int8={int8} step {k}"
        assert _same(step.out[:b], out_e), what + ": logits"
        assert _same(loss.view(1), _package_loss(out_e, batch[2])), what + ": loss"
        _compare(step, opt, scaler, net_e, opt_e, scaler_e, what)
        skipped += step.found_inf.item() == 1.0
        grown += scaler_e.get_scale() > s0
    print(f"{model} int8={int8}: {skipped} of {len(batches)} steps skipped, {grown} growths, "
          f"final scale {scaler.get_scale():.6g}")
    assert skipped >= 2 and grown >= 1, (skipped, grown)
    assert opt.state_dict()["state"][0]["step"] == len(batches) - skipped


def test_checkpoint_resume_continues_bit_for_bit():
    model = "GGNN"
    fx = load_small(model)
    cap = int(fx["edges"].sum().item()) + 64
    batches = _stream(fx, False)
    scaler = torch.amp.GradScaler("cuda", **SCALER_KW)
    step, net, opt = _scaled_step(fx, cap, False, scaler)
    for batch in batches[:5]:
        step(*batch)
    saved = copy.deepcopy((net.state_dict(), opt.state_dict(), scaler.state_dict()))
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    net2 = T._net(fx["C"], fx["sd"])
    net2.load_state_dict(saved[0])
    opt2 = FlatAdam(net2.parameters(), lr=1e-3)
    opt2.load_state_dict(saved[1])
    scaler2 = torch.amp.GradScaler("cuda")
    scaler2.load_state_dict(saved[2])
    with torch.autocast("cuda", dtype=FP16):
        step2 = TrainStep(net2, opt2, batch_size=fx["nodes"].shape[0], entry_capacity=cap, grad_scaler=scaler2)
    for k, batch in enumerate(batches[5:]):
        a, b = step(*batch), step2(*batch)
        torch.cuda.synchronize()
        assert _same(a, b), k
        for p, q in zip(step.params, step2.params):
            assert _same(p, q), k
        assert _same(opt._m, opt2._m) and _same(opt._v, opt2._v), k
        assert scaler.get_scale() == scaler2.get_scale() and scaler._get_growth_tracker() == scaler2._get_growth_tracker()
        assert opt.device_step_counts().tolist() == opt2.device_step_counts().tolist(), k


def test_scaled_steps_do_not_synchronise_but_the_eager_scaler_does():
    fx = load_small("GGNN")
    cap = int(fx["edges"].sum().item()) + 64
    batches = _stream(fx, False)
    scaler = torch.amp.GradScaler("cuda", **SCALER_KW)
    step, net, opt = _scaled_step(fx, cap, False, scaler)
    net_e, opt_e, scaler_e = _eager(fx, cap)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    try:
        torch.cuda.set_sync_debug_mode("error")
        for batch in batches[:4]:
            step(*batch)
        with pytest.raises(RuntimeError):
            _eager_step(net_e, opt_e, scaler_e, batches[0])
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert step.steps == 4


@pytest.mark.parametrize("model", MODELS)
def test_fifty_fp16_scaled_steps_follow_the_reference_loss_curve(model):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    z = np.load(os.path.join(GOLDEN, "loss_curves.npz"))
    fx = load_small(model)
    net = T._net(fx["C"], fx["sd"]).train()
    steps = int(z["steps"])
    opt = FlatAdam(net.parameters(), lr=float(z["lr"]))
    sch = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=float(z["max_lr"]), total_steps=steps)
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    scaler = torch.amp.GradScaler("cuda")
    with torch.autocast("cuda", dtype=FP16):
        step = TrainStep(net, opt, batch_size=nodes.shape[0], entry_capacity=int(edges.sum().item()) + 64,
                         grad_scaler=scaler)
    losses, skipped = [], 0
    for _ in range(steps):
        losses.append(float(step(nodes, edges, target)))
        skipped += step.found_inf.item() != 0.0
        sch.step()
    dev = np.abs(np.array(losses) - z[f"loss/{model}"])
    tol = T.LOSS_TOL_TF32 * 2.0 ** -11 / T.U11      # the TF32 tolerance scaled by the unit roundoff
    print(f"fp16 scaled training {model}: max |loss - reference fp32| {dev.max():.3e} at step {int(dev.argmax())} "
          f"(bound {tol:.2e}), {skipped} skipped, final scale {scaler.get_scale():.6g}")
    assert dev.max() <= tol
    assert losses[-1] < 0.6 * losses[0]


def test_shared_eval_step_gives_the_fp16_step_forward():
    from graphinvent_b200.graphed import EvalStep
    fx = load_small("GGNN")
    cap = int(fx["edges"].sum().item()) + 64
    batches = _stream(fx, False)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    step, net, opt = _scaled_step(fx, cap, False, scaler)
    step(*batches[0])
    B = fx["nodes"].shape[0]
    with torch.autocast("cuda", dtype=FP16):
        ev = EvalStep(net, batch_size=B, entry_capacity=cap, share=step)
    with pytest.raises(ValueError, match="precision"):
        EvalStep(net, batch_size=B, entry_capacity=cap, share=step)          # built outside fp16 autocast
    ev.validation_epoch([batches[1]])
    got = step.out.clone()
    step(*batches[1])                                                          # its forward runs on the same weights
    torch.cuda.synchronize()
    assert _same(got, step.out)


DP_WORKER = r'''
import copy, json, os, sys
import torch, torch.distributed as dist
sys.path.insert(0, os.environ["GIB_ROOT"])
from graphinvent_b200 import parallel, synthetic as S
from graphinvent_b200.config import make_constants, apd_length
from graphinvent_b200.gnn import mpnn
from graphinvent_b200.graphed import TrainStep
from graphinvent_b200.optim import FlatAdam
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl")
C = make_constants("GGNN")
torch.manual_seed(0)
net = mpnn.create(C).cuda()
parallel.broadcast_parameters(net)
ref = copy.deepcopy(net)
G = 256
n, e = S.random_graphs(G, 13, 5, 3, seed=9, min_atoms=1)
t = S.random_targets(G, apd_length(C), seed=9)
nodes, edges, tgt = torch.from_numpy(n).float().cuda(), torch.from_numpy(e).float().cuda(), torch.from_numpy(t).cuda()
bad = nodes.clone()
bad[G - 1, 0, 0] = 1.0e6           # the last molecule (the last rank's shard): an inf fp16 operand in its first layer
cap = int((edges != 0).sum()) + 64
lo, hi = parallel.shard_bounds(G, rank, world)
kw = dict(init_scale=2.0 ** 12, growth_interval=2)
scaler = torch.amp.GradScaler("cuda", **kw)
with torch.autocast("cuda", dtype=torch.float16):
    step = TrainStep(net, FlatAdam(net.parameters(), lr=1e-4), batch_size=hi - lo, entry_capacity=cap,
                     global_batch=G, grad_scaler=scaler)
seq = [bad, nodes, nodes, nodes]
found = []
for x in seq:
    step(x[lo:hi], edges[lo:hi], tgt[lo:hi])
    found.append(step.found_inf.item())
mine = torch.cat([p.detach().reshape(-1) for p in net.parameters()] + [scaler._scale.view(1)])
allp = [torch.empty_like(mine) for _ in range(world)]
dist.all_gather(allp, mine)
if rank == 0:
    s1 = torch.amp.GradScaler("cuda", **kw)
    with torch.autocast("cuda", dtype=torch.float16):
        one = TrainStep(ref, FlatAdam(ref.parameters(), lr=1e-4), batch_size=G, entry_capacity=cap, global_batch=G,
                        group=False, grad_scaler=s1)
    found1 = []
    for x in seq:
        one(x, edges, tgt)
        found1.append(one.found_inf.item())
    worst = max((a - b).abs().max().item() for a, b in zip(net.parameters(), ref.parameters()))
    ranks_equal = all(torch.equal(allp[0], a) for a in allp[1:])
    print(json.dumps({"found": found, "found_single": found1, "ranks_equal": ranks_equal, "param_max_abs_diff": worst,
                      "scale": scaler.get_scale(), "scale_single": s1.get_scale()}))
dist.barrier()
dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_data_parallel_overflow_on_one_rank_skips_every_rank(tmp_path):
    script = tmp_path / "fp16_dp_worker.py"
    script.write_text(DP_WORKER)
    env = dict(os.environ, GIB_ROOT=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29535", str(script)],
                         capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    res = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])
    assert res["found"][0] == 1.0 and res["found"][1:] == [0.0, 0.0, 0.0], res
    assert res["found_single"] == res["found"] and res["ranks_equal"], res
    assert res["scale"] == res["scale_single"], res
    assert res["param_max_abs_diff"] <= 1e-4, res      # the dp_grad_rel_err standard of tests/test_gpu_multi.py
