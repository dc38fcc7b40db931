"""GPU: the TF32, bf16 and fp16 GEMM modes across the reference's hyper-parameter range (tests/test_model_dims_host.py
CONFIGS: one row per branch of csrc/model.cu the default dims never reach), with the modes set the way users set them
(torch.autocast("cuda", dtype=...) for bf16 / fp16, torch's fp32 matmul precision "tf32" for TF32).

1. fp64-anchored forward + backward, every row x mode (exact mode; capacity mode too for the rows whose capacity mode
   runs other kernels).  The yardstick calibrates itself as _fp64_anchored's does, with the oracle's MODE error in place
   of its fp32 error: the fp64 oracle run once more with every GEMM operand rounded the way the package rounds it
   (oracle/mpnn_oracle.py OPERANDS, checked on its own by tests/test_precision_oracle_host.py).  Every case also
   asserts from the launch profile that tensor-core GEMMs ran; one launch never mixes precisions (the dispatcher refuses
   it: tests/test_gpu_tf32.py, tests/test_gpu_autocast.py), so each of them ran in the mode.
2. Every 16-bit plane gib_model_pack writes, every row: bit for bit Wp.to(dtype) / WTp.to(dtype), padding included,
   on an arena poisoned before the pack, with weights scaled into fp16 overflow and subnormals.
3. Bitwise, per mode: the two-part backward == the whole (every row); capacity mode's logits == exact mode's (the
   SAME_KERNELS rows); int8 == float batches (rows A, M).
4. The captured training step over a stream of 3 different batches == eager steps, bit for bit: bf16 TrainStep against
   eager autocast steps, fp16 TrainStep(grad_scaler=) against the eager GradScaler loop (rows A, E, G, I, J).

Worst fraction of the bound in 1., measured on an H100 80GB HBM3 (SXM) at 700 W, per mode (the multipliers 3 and 2
come from the default-mode suite; DESIGN.md section 4):
   tf32  logits 0.535 (row H), gradients 0.821 (row L)
   bf16  logits 0.523 (row C1), gradients 0.503 (row M)
   fp16  logits 0.473 (row H), gradients 0.697 (row I)
Against the fixed bounds of the default-dims tests (LOGIT_C, GRAD_C), printed for information: logits up to 0.99
(row L), gradients up to 4.5 (row J, tf32), 2.4 (row A, bf16) and 3.3 (row L, fp16).  Every case ran 18 (row I) or
more tensor-core launches.  The module runs in about 80 s on one H100.
"""
import ctypes

import pytest
import torch

import tests.test_gpu_tf32 as T
from tests.test_gpu_capacity import _step_grads
from tests.test_gpu_emn_capacity import _run_eagerly
from tests.test_gpu_model_dims import SAME_KERNELS, _batch, _net
from tests.test_model_dims_host import CONFIGS

pytestmark = pytest.mark.gpu

MODES = {"tf32": (None, 1), "bf16": (torch.bfloat16, 2), "fp16": (torch.float16, 3)}   # autocast dtype, precision code
U = {"tf32": 2.0 ** -11, "bf16": 2.0 ** -8, "fp16": 2.0 ** -11}                      # unit roundoff of the operands
TAU = {m: T.KINK_TAU * U[m] / T.U11 for m in MODES}     # the SELU-kink band of each mode (TF32: KINK_TAU itself)
# capacity mode runs other kernels there: A, D, G, I, J as in tests/test_gpu_model_dims.py, and in these modes E too
# (test_capacity_mode_equals_exact_mode below)
CAPACITY_ROWS = ("A", "D", "E", "G", "I", "J")
TC_NT, TC_DW = 0, 1                                     # profile classes (include/gib200.h)
WORST = {}
_ORACLE = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst fraction of the bound per mode:", {k: f"{v[0]:.3f} ({v[1]})" for k, v in sorted(WORST.items())})


def _mode(mode):
    if mode == "tf32":
        return T.precision(matmul="tf32")
    return torch.autocast("cuda", dtype=MODES[mode][0])


def _oracle(cid):
    """fp64, the three mode runs and the kink bands of one row, computed once for every test of the module"""
    if cid not in _ORACLE:
        from oracle import mpnn_oracle as O
        C, nodes, edges, target = _batch(cid)
        sd = O.init_state_dict(C, seed=0)         # the parameters _net(C) loads

        def f64():
            return O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)

        exact = f64()
        runs = {}
        for m in MODES:
            O.OPERANDS = m
            try:
                runs[m] = (f64(), O.train_step_grads(sd, C, nodes, edges, target))    # fp64 and fp32 arithmetic
            finally:
                O.OPERANDS = None
        kink = {}
        for tau in sorted(set(TAU.values())):
            try:
                O.KINK = (tau, "L")
                gL = f64()[2]
                O.KINK = (tau, "R")
                gR = f64()[2]
            finally:
                O.KINK = None
            kink[tau] = {k: (gL[k] - gR[k]).norm().item() for k in gL}
        _ORACLE[cid] = (C, nodes, edges, target, exact, runs, kink)
    return _ORACLE[cid]


def _lib():
    from graphinvent_b200._lib import lib
    return lib


def _profiled_step(net, nodes, edges, target, mode):
    """one eager forward + loss + backward in the mode, and the number of launches of each profile class"""
    lib = _lib()
    torch.cuda.synchronize()
    lib.gib_profile_enable(1)
    try:
        with _mode(mode):
            out, loss, grads = _step_grads(net, nodes, edges, target)
        torch.cuda.synchronize()
        k = 8
        ms, work, cnt = (ctypes.c_double * k)(), (ctypes.c_double * k)(), (ctypes.c_longlong * k)()
        assert lib.gib_profile_collect(ms, work, cnt) == 0
    finally:
        lib.gib_profile_enable(0)
    return out, loss, grads, list(cnt)


def _record(mode, kind, ratio, what):
    key = f"{mode} {kind}"
    if ratio >= WORST.get(key, (0.0, ""))[0]:
        WORST[key] = (ratio, what)


# ---- 1. fp64-anchored ------------------------------------------------------------------------------------------------
# The mode error |x_mode - x64| is taken per molecule / per tensor as the larger of two evaluations of the rounded-operand
# oracle: in fp64 arithmetic (operand rounding alone) and in fp32 arithmetic (what the package's fp32 kernels lose on
# top of it).  The fp64 evaluation alone misses two fp32 effects the package has, measured on the rows (TF32):
#   - molecules without a bond: `energies - 1e6` of the gather attention is quantised to 1/16 in fp32.  Rows F, H, K, L
#     (10, 8, 8 and 34 bond-less molecules of 55): the plain fp32 oracle is 1.5e-3, 3.1e-3, 8.6e-3 and 1.95e-2 off fp64
#     on them, the fp64 mode run at most 1.0e-3, 3.8e-3, 5.2e-3 and 5.2e-3 over all molecules; the package: 1.5e-3,
#     3.6e-3, 8.8e-3, 2.07e-2;
#   - cancelling sums: row I's 1 x 1 msg_nns.2.seq.9.weight has a gradient of 2.0e-5 from terms of either sign; its mode
#     error is 1.4e-7 in fp64 arithmetic, 1.3e-6 in fp32 arithmetic; the package's is 2.2e-6.
# Bounds, with o_mode / g_mode the oracle's rounded-operand runs and u the operand's unit roundoff (2^-11 TF32 and fp16,
# 2^-8 bf16):
#   logits, per molecule:  max|o - o64| <= 3 max|o_mode - o64| + u (1 + max|o64|)
#   gradients, per tensor: |g - g64| <= 2 |g_mode - g64| + kink band(tau_mode) + u |g64| + 1e-7 max|g|   (L2)
#   global L2:             |g - g64| <= 2 |g_mode - g64| + kink band + u |g64|
#   loss:                  |loss - l64| <= 3 |l_mode - l64| + u max(1, |l64|)
#   argmax:                equal to o_mode's wherever o_mode's top-2 gap exceeds 2 (its mode error + the floor)
# The floors are one operand rounding of the quantity's own size.  The oracle rounds every Linear; the package keeps the
# narrow APD output layers and GEMMs below 256 rows on the fp32 SIMT kernel and accumulates in fp32, so its rounding
# events are a subset of the oracle's at other points: a molecule or tensor whose mode error happens to cancel can still
# differ from fp64 by about one rounding of its size.  The multipliers are those of _fp64_anchored.
def _anchored(cid, mode, capacity):
    C, nodes, edges, target, (l64, o64, g64), runs, kink = _oracle(cid)
    (lm, om, gm), (lm32, om32, gm32) = runs[mode]
    kb = kink[TAU[mode]]
    u = U[mode]
    net = _net(C)
    if capacity:
        net.entry_capacity = int((edges > 0).sum()) + 64
    out, loss, grads, cnt = _profiled_step(net, nodes.cuda(), edges.cuda(), target.cuda(), mode)
    tag = f"row {cid} {mode}{' capacity' if capacity else ''}"
    tc = cnt[TC_NT] + cnt[TC_DW]
    assert tc > 0, f"{tag}: no tensor-core launch ({cnt}): the mode was not exercised"
    out = out.cpu().double()
    mag = 1 + o64.abs().max(1).values
    e = (out - o64).abs().max(1).values
    e_mode = torch.maximum((om - o64).abs().max(1).values, (om32.double() - o64).abs().max(1).values)
    floor = u * mag
    ratio_l = (e / (3 * e_mode + floor)).max().item()
    old_l = (e / (T.LOGIT_C * u * mag)).max().item()
    top2 = om.topk(2, dim=1).values
    decided = (top2[:, 0] - top2[:, 1]) > 2 * e_mode + 2 * floor
    same = out.argmax(1) == om.argmax(1)
    gscale = max(g.norm().item() for g in g64.values())
    ratio_g, old_g, worst = 0.0, 0.0, ""
    tot = [0.0, 0.0, 0.0, 0.0]
    for (k, g), got in zip(g64.items(), grads):
        d = (got.cpu().double() - g).norm().item()
        dm = max((gm[k] - g).norm().item(), (gm32[k].double() - g).norm().item())
        gn = g.norm().item()
        r = d / (2 * dm + kb[k] + u * gn + 1e-7 * gscale)
        old_g = max(old_g, d / (T.GRAD_C * u * gn + kb[k] + 1e-7 * gscale))
        for i, v in enumerate((d, dm, kb[k], gn)):
            tot[i] += v * v
        if r > ratio_g:
            ratio_g, worst = r, k
    tot = [t ** 0.5 for t in tot]
    _record(mode, "logits", ratio_l, tag)
    _record(mode, "gradients", ratio_g, tag)
    print(f"{tag}: logits max|o - o64| {e.max().item():.3e}, mode error {e_mode.max().item():.3e}, "
          f"{ratio_l:.3f} of the bound; worst gradient {worst} {ratio_g:.3f} of the bound; global L2 |g - g64| "
          f"{tot[0]:.3e}, mode error {tot[1]:.3e}, kink band (tau {TAU[mode]:g}) {tot[2]:.3e}; decided "
          f"{int(decided.sum())}/{len(decided)}; loss {loss:.7f} vs fp64 {float(l64):.7f} / mode {float(lm):.7f}; "
          f"of the fixed bounds: logits {old_l:.3f} (LOGIT_C), gradients {old_g:.3f} (GRAD_C); "
          f"tensor-core launches {tc} (forward / dX {cnt[TC_NT]}, dW {cnt[TC_DW]})")
    assert ratio_l <= 1.0, f"{tag}: a molecule's logits move beyond 3 x the mode error + floor ({ratio_l:.3f})"
    assert bool(same[decided].all()), f"{tag}: argmax differs on {int((~same & decided).sum())} decided molecules"
    l_mode = max(abs(float(lm) - float(l64)), abs(float(lm32) - float(l64)))
    assert abs(loss - float(l64)) <= 3 * l_mode + u * max(1.0, abs(float(l64))), tag
    assert ratio_g <= 1.0, f"{tag}: gradient {worst} at {ratio_g:.3f} of its bound"
    assert tot[0] <= 2 * tot[1] + tot[2] + u * tot[3], tag


@pytest.mark.parametrize("cid,mode,capacity", [(c, m, False) for c in CONFIGS for m in MODES] +
                         [(c, m, True) for c in CAPACITY_ROWS for m in MODES])
def test_fp64_anchored_in_precision_mode(cid, mode, capacity):
    _anchored(cid, mode, capacity)


# ---- 2. packed 16-bit planes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("cid", list(CONFIGS))
def test_packed_16bit_planes_are_torch_casts(cid, mode):
    """follows tests/test_gpu_autocast.py::test_packed_16bit_planes_are_torch_casts over the rows; the arena starts as
    0x7f bytes, so a plane element the pack does not write (a pad row or column) cannot pass as the +0 of Wp"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import PLAN_LINEAR_FIELDS
    lib = _lib()
    dtype, code = MODES[mode]
    C = _batch(cid)[0]
    net = _net(C)
    # fp16 overflow (x 1e6), subnormals (x 3e-4) and normal values, in turn over the parameters
    scales = (1.0, 1.0e6, 3.0e-4)
    params = [(p.detach() * scales[i % 3]).contiguous() for i, p in enumerate(net.parameters())]
    d = Fn.make_dims(net, 64, tf32=code)
    packed = torch.full((lib.gib_model_packed_bytes(ctypes.byref(d)),), 0x7F, dtype=torch.uint8, device="cuda")
    assert lib.gib_model_pack(ctypes.byref(d), Fn._ptr_table(params), Fn._ptr(packed),
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    out = (ctypes.c_longlong * len(PLAN_LINEAR_FIELDS))()
    n = lib.gib_test_plan_linear(ctypes.byref(d), 0, out)
    f32 = packed.view(torch.float32)
    pads = inf = 0
    for li in range(n):
        lib.gib_test_plan_linear(ctypes.byref(d), li, out)
        f = dict(zip(PLAN_LINEAR_FIELDS, out))
        Rp, Cp, Ctp = f["nblk"] * f["Rbp"], f["Cp"], f["Ctp"]
        pads += Rp * Cp - f["nblk"] * f["Rb"] * f["C"]
        for src, plane, cnt in ((f["ow"], f["ow_lo"], Rp * Cp), (f["owt"], f["owt_lo"], Ctp * Rp)):
            want = f32[src:src + cnt].to(dtype)
            got = packed[plane * 4:plane * 4 + cnt * 2].view(torch.int16)
            assert torch.equal(got, want.view(torch.int16)), (cid, mode, li, "ow" if src == f["ow"] else "owt")
            inf += int(torch.isinf(want).sum())
    assert pads > 0, cid
    assert (inf > 0) == (mode == "fp16"), (cid, mode, inf)


# ---- 3. bitwise equalities -------------------------------------------------------------------------------------------
def _setup(cid):
    C, nodes, edges, target = _batch(cid)
    return C, _net(C), nodes.cuda(), edges.cuda(), target.cuda()


def _train_step(net, B, cap, mode, lr=1e-4, scaler=None, warmup=False):
    """a TrainStep built in the mode; fp16 needs a GradScaler (without one TrainStep keeps the fp32-input precision)"""
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    if mode == "fp16" and scaler is None:
        scaler = torch.amp.GradScaler("cuda", init_scale=256.0)
    with _mode(mode):
        step = TrainStep(net, FlatAdam(net.parameters(), lr=lr), batch_size=B, entry_capacity=cap, warmup=warmup,
                         grad_scaler=scaler)
    assert step.d.tf32 == MODES[mode][1]
    return step


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("cid", list(CONFIGS))
def test_two_part_backward_equals_the_whole(cid, mode):
    C, net, nodes, edges, target = _setup(cid)
    step = _train_step(net, nodes.shape[0], int((edges > 0).sum()) + 64, mode)
    step.load(nodes, edges, target)
    g_whole = _run_eagerly(step)[2]
    step.gflat.zero_()
    step._backward(1)
    step._backward(2)
    torch.cuda.synchronize()
    assert torch.count_nonzero(g_whole) > 0 and torch.isfinite(g_whole).all()
    assert torch.equal(step.gflat, g_whole)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("cid", SAME_KERNELS)
def test_capacity_mode_equals_exact_mode(cid, mode):
    C, net, nodes, edges, target = _setup(cid)
    with _mode(mode):
        out0, loss0, g0 = _step_grads(net, nodes, edges, target)
        net.entry_capacity = int(net.last_stats["entries"] * 1.3) + 64
        out1, loss1, g1 = _step_grads(net, nodes, edges, target)
    assert net.last_stats["capacity"] == net.entry_capacity
    assert torch.equal(out0, out1)
    assert abs(loss0 - loss1) <= 1e-7
    if cid in ("D", "E"):
        # the message MLPs of D (AttGGNN) and E (EMN) run on host-side row counts in exact mode: their weight gradients
        # of fewer than 2048 rows go to the fp32 SIMT kernel there and to the tensor cores, operands rounded, in capacity
        # mode (measured: 5e-5 / 4e-4 / 1.2e-4 of max|g| apart in tf32 / bf16 / fp16); capacity mode is held to fp64
        # by test_fp64_anchored_in_precision_mode instead
        return
    for (name, _), a, b in zip(net.named_parameters(), g0, g1):
        assert (a - b).abs().max().item() <= 2e-6 * max(1e-3, a.abs().max().item()), name


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("cid", ["A", "M"])
def test_int8_batches_equal_float_batches(cid, mode):
    C, net, nodes, edges, target = _setup(cid)
    with _mode(mode):
        out0, loss0, g0 = _step_grads(net, nodes, edges, target)
        out1, loss1, g1 = _step_grads(net, nodes.to(torch.int8), edges.to(torch.int8), target)
    assert torch.equal(out0, out1) and loss0 == loss1
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)


# ---- 4. the captured training step against eager steps ---------------------------------------------------------------
def _stream(cid):
    C, nodes, edges, target = _batch(cid)
    nodes, edges, target = nodes.cuda(), edges.cuda(), target.cuda()
    B = nodes.shape[0]
    out = []
    for k in range(3):
        g = torch.Generator(device="cuda").manual_seed(k)
        perm = torch.randperm(B, device="cuda", generator=g)
        out.append((nodes[perm].contiguous(), edges[perm].contiguous(), target[perm].contiguous()))
    return C, B, int((edges > 0).sum()) + 64, out


@pytest.mark.parametrize("cid", ["A", "E", "G", "I", "J"])
def test_bf16_train_step_equals_eager_autocast_steps(cid):
    """tests/test_gpu_autocast.py::test_bf16_train_step_equals_eager_autocast_steps on the row"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.optim import FlatAdam
    C, B, cap, batches = _stream(cid)
    step = _train_step(_net(C), B, cap, "bf16", lr=1e-3, warmup=True)
    assert step.autocast_dtype is torch.bfloat16
    net = _net(C)
    net.entry_capacity = cap
    opt = FlatAdam(net.parameters(), lr=1e-3)
    p0 = [p.detach().clone() for p in net.parameters()]
    for k, (n_, e_, t_) in enumerate(batches):
        step(n_, e_, t_)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(n_, e_)
        opt.zero_grad(set_to_none=True)
        Fn.kl_loss(out, t_).backward()
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(step.out, out), (cid, k)
        for p, q in zip(step.params, net.parameters()):
            assert torch.equal(p, q), (cid, k)
    assert not all(torch.equal(a, b) for a, b in zip(p0, net.parameters()))


# init 2^20 with backoff 2^-6 and growth every step: large enough that an early step of the stream can overflow, and
# small enough after one backoff for the next steps to be taken
SCALER_KW = dict(init_scale=2.0 ** 20, growth_factor=2.0, backoff_factor=2.0 ** -6, growth_interval=1)


@pytest.mark.parametrize("cid", ["A", "E", "G", "I", "J"])
def test_fp16_scaled_step_equals_the_eager_scaler_loop(cid):
    """tests/test_gpu_fp16_train.py::test_fp16_scaled_step_equals_the_eager_scaler_loop on the row"""
    import tests.test_gpu_fp16_train as H
    from graphinvent_b200.optim import FlatAdam
    C, B, cap, batches = _stream(cid)
    scaler = torch.amp.GradScaler("cuda", **SCALER_KW)
    step = _train_step(_net(C), B, cap, "fp16", lr=1e-3, scaler=scaler, warmup=True)
    assert step.autocast_dtype is torch.float16
    opt = step.optimizer
    net_e = _net(C)
    net_e.entry_capacity = cap
    opt_e, scaler_e = FlatAdam(net_e.parameters(), lr=1e-3), torch.amp.GradScaler("cuda", **SCALER_KW)
    skipped = 0
    for k, batch in enumerate(batches):
        loss = step(*batch)
        out_e = H._eager_step(net_e, opt_e, scaler_e, batch)
        torch.cuda.synchronize()
        what = f"row {cid} step {k}"
        assert H._same(step.out, out_e), what + ": logits"
        assert H._same(loss.view(1), H._package_loss(out_e, batch[2])), what + ": loss"
        H._compare(step, opt, scaler, net_e, opt_e, scaler_e, what)
        skipped += step.found_inf.item() == 1.0
    print(f"row {cid} fp16: {skipped} of {len(batches)} steps skipped, final scale {scaler.get_scale():.6g}")
    assert skipped < len(batches), "every step skipped: the stream compares no update"
