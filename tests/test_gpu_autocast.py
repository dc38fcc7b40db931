"""GPU: bf16 / fp16 tensor-core GEMMs under torch.autocast (precision codes 2 / 3).

1. GEMM call patterns of tests/test_gpu_gemm_patterns.py (epilogues, device-side rows, groups, chains, grouped /
   gate-blocked / device-row weight gradients) with tf32 = 2 / 3 through the test hooks, against float64 evaluated on
   the operands rounded by torch's own `.to(dtype)`: only fp32 accumulation remains, so a wrong rounding mode or an
   operand left unrounded shows up at 2^-9 / 2^-12, far above the bound.
2. The 16-bit planes that gib_model_pack writes equal Wp.to(dtype) / WTp.to(dtype) bit for bit.
3. The four models (float / int8, exact / capacity) against the fp64 oracle within the 16-bit error model.
4. No leakage between modes; a backward after the autocast context uses the forward's mode.
5. bf16 training (captured step == eager steps; 50 steps near the fp32 loss curve); fp16 with GradScaler; the captured
   generator and the RL backward equal their eager paths; EvalStep refuses a TrainStep of another mode.
"""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

import tests.test_gpu_gemm_patterns as P
import tests.test_gpu_tf32 as T
from tests.conftest import GOLDEN, MODELS, load_small

pytestmark = pytest.mark.gpu

DTYPES = {"bf16": (torch.bfloat16, 2), "fp16": (torch.float16, 3)}
U = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}    # unit roundoff of the operand type
EPS_ACC = 3.0e-6                               # fp32-accumulation bound of the TF32 test, relative to |A_r| |W_r|^T
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n16-bit worst error / magnitude:", {k: f"{v[0]:.3g} ({v[1]})" for k, v in sorted(WORST.items())})


def _within(got, ref, mag, what, slack=0.0):
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (mag + 1e-300)).max().item() if err.numel() else 0.0
    if ratio >= WORST.get("acc", (0.0, ""))[0]:
        WORST["acc"] = (ratio, what)
    assert ratio <= EPS_ACC, f"{what}: error / magnitude {ratio:.3g} > {EPS_ACC:.1e}"


# ---- 1. call patterns ------------------------------------------------------------------------------------------------
def _run_nt16(nts, dt, dep=None):
    dtype, code = DTYPES[dt]
    L = P._lib()
    structs = []
    for t in nts:
        s = t.struct()
        t.plane16 = t.W.to(dtype).contiguous()       # ldw = K elements
        s.W_hi, s.W_lo, s.tf32 = P._p(t.plane16), None, code
        structs.append(s)
    arr = (L.GemmProblem * len(nts))(*structs)
    flags = None
    if dep is not None:
        nb = L.lib.gib_test_chain_flag_bytes(arr, len(nts))
        flags = torch.full((max(nb // 4, 1),), 12345, dtype=torch.int32, device="cuda")
        dep = (ctypes.c_int * len(nts))(*dep)
    return P._profiled(lambda: L.lib.gib_test_gemm_nt(arr, len(nts), dep, P._p(flags), P._st()))


def _check_nt16(t, dt, what):
    dtype = DTYPES[dt][0]
    lo, hi, ns, nv = t.lo, t.hi, t.n_store, t.n_valid
    A64 = t.A[lo:hi, :t.K].to(dtype).double()
    Wp = torch.zeros(max(t.N, ns), t.K, dtype=torch.float64, device="cuda")
    Wp[:t.N] = t.W.to(dtype).double()
    pre, mag = A64 @ Wp[:ns].t(), A64.abs() @ Wp[:ns].abs().t()
    slack = 0.0
    if t.mode == P.EPI_ACT:
        if t.bias is not None:
            b = torch.zeros(max(t.N, ns), dtype=torch.float64, device="cuda")
            b[:t.N] = t.bias.double()
            pre, mag = pre + b[:ns], mag + b[:ns].abs()
        ref, mag = P._act64(pre, t.act), mag * P.SLOPE[t.act]
        slack = P.ACT_SLACK if t.act else 0.0
    elif t.mode == P.EPI_MUL_DACT:
        d = P._dact64(t.aux0[lo:hi, :ns].double(), t.act)
        ref, mag, slack = pre * d, mag * d.abs(), mag * P.DACT_SLACK
    else:
        x = t.aux0[lo:hi, :ns].double()
        ref, mag = pre + x, mag + x.abs()
    out = t.C[lo:hi]
    _within(out[:, :nv], ref[:, :nv], mag[:, :nv], f"{dt} {what}", slack)
    assert (out[:, nv:ns] == 0).all() and not torch.signbit(out[:, nv:ns]).any(), f"{what}: pad columns not +0"
    P._same_bits(out[:, ns:], t.C0[lo:hi, ns:], what + " columns >= n_store")
    P._same_bits(t.C[:lo], t.C0[:lo], what + " rows before the range")
    P._same_bits(t.C[hi:], t.C0[hi:], what + " rows after the range")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("M", [1, 129, 4097])
@pytest.mark.parametrize("N", [48, 200, 608])
def test_nt_shapes_and_epilogues_16bit(dt, M, N):
    """every epilogue on the wgmma kernel, through a device-side row count (clipped / ragged tiles, any M) and through
    the dispatcher's own choice"""
    ran = 0
    for K in (16, 48, 160, 688):
        for label, kw in P._epilogues(N):
            kw = dict(kw)
            lda = K + kw.pop("lda_pad", 0)
            for run in ("tc", "dispatch"):
                what = f"M={M} N={N} K={K} {label} [{run}]"
                dyn = dict(cap=M + 5, base=3) if run == "tc" else {}
                t = P.NT(M, N, K, lda=lda, **kw, **dyn)
                if P._expect_single(t, 1, 0) != [P.TC_NT]:
                    continue
                rc, cls = _run_nt16([t], dt)
                assert rc == 0, what + ": " + P._lib().lib.gib_last_error().decode()
                assert cls == [P.TC_NT], f"{what}: kernel classes {cls}"
                _check_nt16(t, dt, what)
                ran += 1
    assert ran > 0


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", list(P._group_cases()))
def test_nt_groups_16bit(dt, case):
    """a group that does not qualify for one grouped launch (k16 member) runs member by member: each member is checked
    against the path the dispatch rule gives it, the fp32 SIMT kernel or the 16-bit tensor-core kernel"""
    nts = P._group_cases()[case]()
    rc, cls = _run_nt16(nts, dt)
    assert rc == 0, P._lib().lib.gib_last_error().decode()
    assert cls == P._expect_group(nts, 1, 0) and P.TC_NT in cls, f"{case}: kernel classes {cls}"
    assert (cls == [P.TC_NT]) == (case != "k16 member"), f"{case}: kernel classes {cls}"
    for i, t in enumerate(nts):
        if cls == [P.TC_NT] or P._expect_single(t, 1, 0) == [P.TC_NT]:
            _check_nt16(t, dt, f"{case} member {i}")
        else:
            t.check("simt", f"{case} member {i} [simt]")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", list(P._chain_cases()))
def test_nt_chains_16bit(dt, case):
    nts, dep = P._chain(**P._chain_cases()[case])
    rc, cls = _run_nt16(nts, dt, dep)
    assert rc == 0, P._lib().lib.gib_last_error().decode()
    assert cls == [P.TC_NT], f"{case}: one chain launch expected, got {cls}"
    for k, t in enumerate(nts):
        _check_nt16(t, dt, f"{case} problem {k}")


def test_16bit_refusals():
    """mixed precisions in one launch, a 16-bit problem without a plane, raw W, debug bit 0 and tensor cores off"""
    L = P._lib()
    nts = [P.NT(1000, 256, 144, act=1), P.NT(1300, 128, 64, act=1)]
    structs = [t.struct() for t in nts]
    structs[0].tf32, structs[1].tf32 = 2, 3
    structs[0].W_hi = structs[1].W_hi = P._p(nts[0].W.to(torch.bfloat16))
    arr = (L.GemmProblem * 2)(*structs)
    rc, cls = P._profiled(lambda: L.lib.gib_test_gemm_nt(arr, 2, None, None, P._st()))
    assert rc < 0 and cls == [] and b"precision" in L.lib.gib_last_error()
    t = P.NT(2000, 256, 144, act=1)
    s = t.struct()
    s.tf32, s.W_hi = 2, None
    rc, cls = P._profiled(lambda: L.lib.gib_test_gemm_nt(ctypes.byref(s), 1, None, None, P._st()))
    assert rc < 0 and cls == [] and b"16-bit plane" in L.lib.gib_last_error()
    plane = t.W.to(torch.bfloat16)
    s.W_hi = P._p(plane)
    for kw in (dict(debug=1), dict(tc=0)):
        with P._mode(**kw):
            rc, cls = P._profiled(lambda: L.lib.gib_test_gemm_nt(ctypes.byref(s), 1, None, None, P._st()))
        assert rc < 0 and cls == [] and b"tensor-core path" in L.lib.gib_last_error(), kw
    t.untouched("refused")


class _RoundedDW:
    def __init__(self, q, dtype):
        self.q, self.dtype = q, dtype

    def contribution(self):
        q = self.q
        idx, _, _, b, bm = q.contribution()
        lo, hi = q.live()
        r = torch.arange(q.R, device="cuda")
        prow = (r // q.Rb) * q.Rbp + r % q.Rb
        G = q.G[lo:hi].to(self.dtype).double()[:, prow]
        X = q.X[lo:hi, :q.C].contiguous().to(self.dtype).double()
        return idx, G.t() @ X, G.abs().t() @ X.abs(), b, bm


def _run_dw16(groups, dt, plan_rows=0):
    dtype, code = DTYPES[dt]
    L = P._lib()
    flat = [q for g in groups for q in g]
    structs = [q.struct() for q in flat]
    for s in structs:
        s.tf32 = code
    arr = (L.DwProblem * len(flat))(*structs)
    sizes = (ctypes.c_int * len(groups))(*[len(g) for g in groups])
    nb = L.lib.gib_test_dw_scratch_bytes(arr, sizes, len(groups), plan_rows)
    scratch = torch.full((nb // 4,), P.NAN, device="cuda")
    dsts = {}
    for q in flat:
        for t in (q.dW, q.dbias):
            if t is not None:
                dsts.setdefault(P._root(t).data_ptr(), (P._root(t), P._root(t).clone()))
    with P._mode(tc=1):
        rc, cls = P._profiled(lambda: L.lib.gib_test_dw_groups(arr, sizes, len(groups), plan_rows, P._p(scratch),
                                                               P._st()))

    def check(what):
        for base_ptr, (t, t0) in dsts.items():
            ref, mag = t0.double().flatten().clone(), t0.double().abs().flatten().clone()
            for q in flat:
                idx, w, wm, b, bm = _RoundedDW(q, dtype).contribution()
                if q.dW is not None and P._root(q.dW).data_ptr() == base_ptr:
                    idx = (idx + (q.dW.data_ptr() - base_ptr) // 4).flatten()
                    ref.index_add_(0, idx, w.flatten())
                    mag.index_add_(0, idx, wm.flatten())
                if q.dbias is not None and P._root(q.dbias).data_ptr() == base_ptr:
                    idx = torch.arange(q.R, device="cuda") + (q.dbias.data_ptr() - base_ptr) // 4
                    ref.index_add_(0, idx, b)
                    mag.index_add_(0, idx, bm)
            _within(t.flatten(), ref, mag, f"{dt} {what}")

    return rc, cls, check


@pytest.mark.parametrize("dt", list(DTYPES))
def test_dw_patterns_16bit(dt):
    """single (ragged chunk rows), gate-blocked, MNN strided slices, a group of 16 and device-side rows"""
    for M in (2048, 4097, 40000):
        G, X = P._operands(M, 112, 144, 100, 136, seed=M)
        rc, cls, check = _run_dw16([[P.DW(G, X, M, torch.randn(100, 136, device="cuda"), 100, 136,
                                          dbias=torch.randn(100, device="cuda"))]], dt)
        assert rc == 0 and cls == [P.TC_DW], cls
        check(f"dW M={M}")
    H, C, M = 100, 136, 4097
    Hp = P.pad16(H)
    G, X = P._operands(M, 3 * Hp, 144, 3 * H, C, seed=7)
    for g in range(3):
        G[:, g * Hp + H:(g + 1) * Hp] = 0
    rc, cls, check = _run_dw16([[P.DW(G, X, M, torch.randn(3 * H, C, device="cuda"), 3 * H, C,
                                      dbias=torch.randn(3 * H, device="cuda"), Rb=H, Rbp=Hp)]], dt)
    assert rc == 0 and cls == [P.TC_DW], cls
    check("gate-blocked")
    R, H2, Ef = 100, 64, 3
    big = torch.randn(R, H2, Ef, device="cuda")
    db = torch.randn(R, device="cuda")
    grp = []
    for t, m in enumerate((2048, 1500, 700)):
        G, X = P._operands(m, P.pad16(R), H2, R, H2, seed=40 + t)
        grp.append(P.DW(G, X, m, P._slice_dst(big, t), R, H2, dbias=db if t == 0 else None, rs=H2 * Ef, cs=Ef))
    rc, cls, check = _run_dw16([grp], dt)
    assert rc == 0 and cls == [P.TC_DW], cls
    check("MNN slices")
    shapes = [(4097, 100, 136), (2047, 256, 48), (33, 608, 144), (5000, 112, 688), (128, 64, 256), (3000, 48, 48),
              (2048, 100, 100), (700, 65, 129), (1500, 300, 64), (4096, 32, 32), (257, 128, 608), (999, 80, 112),
              (129, 96, 96), (1, 48, 32), (31, 256, 256), (0, 64, 64)]
    grp = []
    for k, (m, R, C) in enumerate(shapes):
        G, X = P._operands(m, P.pad16(R), P.pad16(C), R, C, seed=100 + k)
        grp.append(P.DW(G, X, m, torch.randn(R, C, device="cuda"), R, C,
                        dbias=torch.randn(R, device="cuda") if k % 3 else None))
    rc, cls, check = _run_dw16([grp], dt, plan_rows=3 * sum(s[0] for s in shapes))
    assert rc == 0 and cls == [P.TC_DW], cls
    check("group of 16")
    cap = 8192
    grp = P._shared_buffer_group(cap, 112, 144, 100, 136, [(0, 1900), (2048, 0), (4096, 3000), (8064, 500)], seed=9)
    rc, cls, check = _run_dw16([grp], dt, plan_rows=cap)
    assert rc == 0 and cls == [P.TC_DW], cls
    check("device-side rows")


# ---- 2. packed planes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("model", MODELS)
def test_packed_16bit_planes_are_torch_casts(dt, model):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import PLAN_LINEAR_FIELDS, lib
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    dtype, code = DTYPES[dt]
    net = mpnn.create(O.make_constants(model)).cuda()
    params = [(p.detach() * 40.0).contiguous() for p in net.parameters()]   # fp16 overflow of the largest weights
    d = Fn.make_dims(net, 64, tf32=code)
    packed = torch.zeros(lib.gib_model_packed_bytes(ctypes.byref(d)), dtype=torch.uint8, device="cuda")
    assert lib.gib_model_pack(ctypes.byref(d), Fn._ptr_table(params), Fn._ptr(packed), P._st()) == 0
    torch.cuda.synchronize()
    out = (ctypes.c_longlong * len(PLAN_LINEAR_FIELDS))()
    n = lib.gib_test_plan_linear(ctypes.byref(d), 0, out)
    f32 = packed.view(torch.float32)
    for li in range(n):
        lib.gib_test_plan_linear(ctypes.byref(d), li, out)
        f = dict(zip(PLAN_LINEAR_FIELDS, out))
        Rp, Cp, Ctp = f["nblk"] * f["Rbp"], f["Cp"], f["Ctp"]
        for src, plane, cnt in ((f["ow"], f["ow_lo"], Rp * Cp), (f["owt"], f["owt_lo"], Ctp * Rp)):
            want = f32[src:src + cnt].to(dtype).view(torch.int16)
            got = packed[plane * 4:plane * 4 + cnt * 2].view(torch.int16)
            assert torch.equal(got, want), (model, li)


# ---- 3. models against the fp64 oracle -------------------------------------------------------------------------------
LOGIT_C = 16.5
GRAD_C = 22.0
_KINK = {}


def _kink(model, tau):
    """the oracle's SELU-kink band at tau (left minus right derivative at every SELU input within tau of 0)"""
    if (model, tau) not in _KINK:
        from oracle import mpnn_oracle as O
        C, sd, nodes, edges, target, _, _, _ = T._oracle(model)
        try:
            O.KINK = (tau, "L")
            _, _, gL = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
            O.KINK = (tau, "R")
            _, _, gR = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
        finally:
            O.KINK = None
        _KINK[(model, tau)] = {k: (gL[k] - gR[k]).norm().item() for k in gL}
    return _KINK[(model, tau)]


def _oracle_autocast_error(model, dtype):
    """the reference's own error under autocast: the oracle's fp32 restatement (a host-side evaluation) run under
    torch.autocast("cpu") in the same dtype"""
    from oracle import mpnn_oracle as O
    C, sd, nodes, edges, target, o64, _, _ = T._oracle(model)
    with torch.autocast("cpu", dtype=dtype):
        _, o, _ = O.train_step_grads(sd, C, nodes, edges, target)
    return (o.float().double() - o64).abs().max().item()


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("capacity", [False, True])
@pytest.mark.parametrize("int8", [False, True])
@pytest.mark.parametrize("model", MODELS)
def test_models_against_fp64_under_autocast(model, int8, capacity, dt):
    dtype = DTYPES[dt][0]
    u = U[dt]
    C, sd, nodes, edges, target, o64, g64, _ = T._oracle(model)
    kink = _kink(model, T.KINK_TAU * u / T.U11)
    net = T._net(C, sd)
    if capacity:
        net.entry_capacity = int(edges.sum().item()) + 64
    if int8:
        nodes, edges = nodes.to(torch.int8), edges.to(torch.int8)
    with torch.autocast("cuda", dtype=dtype):
        out, grads = T._eager_step(net, nodes, edges, target)
    assert out.dtype == torch.float32
    out3, _ = T._eager_step(net, nodes, edges, target)
    assert not torch.equal(out, out3), "autocast gave the fp32-mode logits"
    e = (out.cpu().double() - o64).abs().max(1).values
    lim = LOGIT_C * u * (1 + o64.abs().max(1).values)
    ratio_l = (e / lim).max().item()
    gscale = max(g.norm().item() for g in g64.values())
    ratio_g, worst = 0.0, ""
    for (k, g), got in zip(g64.items(), grads):
        d = (got.cpu().double() - g).norm().item()
        bound = GRAD_C * u * g.norm().item() + kink[k] + 1e-7 * gscale
        if d / bound > ratio_g:
            ratio_g, worst = d / bound, k
    ref_err = _oracle_autocast_error(model, dtype) if not int8 and not capacity else float("nan")
    print(f"{dt} {model} int8={int8} capacity={capacity}: logits max |o - o64| {e.max().item():.3e} "
          f"({ratio_l:.3f} of bound; the oracle under torch.autocast: {ref_err:.3e}), "
          f"worst gradient {worst} {ratio_g:.3f} of bound")
    assert ratio_l <= 1.0 and ratio_g <= 1.0


# ---- 4. no leakage ---------------------------------------------------------------------------------------------------
def _ctx(mode):
    import contextlib
    if mode in DTYPES:
        return torch.autocast("cuda", dtype=DTYPES[mode][0])
    if mode == "tf32":
        return T.precision(matmul="tf32")
    return contextlib.nullcontext()


def test_modes_do_not_leak_into_each_other_and_backward_keeps_the_forward_mode():
    fx = load_small("GGNN")
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    cap = int(edges.sum().item()) + 64

    def fresh():
        n = T._net(fx["C"], fx["sd"])
        n.entry_capacity = cap          # capacity mode: every message GEMM on the tensor cores, even at this size
        return n

    net = fresh()
    seq = ("fp32", "bf16", "tf32", "fp16", "fp32")
    got = []
    for mode in seq:
        with _ctx(mode):
            got.append(T._eager_step(net, nodes, edges, target))
    for mode, (out, grads) in zip(seq, got):
        with _ctx(mode):
            out2, grads2 = T._eager_step(fresh(), nodes, edges, target)
        assert torch.equal(out, out2), mode
        assert all(torch.equal(a, b) for a, b in zip(grads, grads2)), mode
    outs = dict(zip(seq, (o for o, _ in got)))
    # every mode takes effect (fp16 and TF32 keep the same 10-bit mantissa and may give the same bits)
    for a, b in (("fp32", "bf16"), ("fp32", "tf32"), ("fp32", "fp16"), ("bf16", "tf32"), ("bf16", "fp16")):
        assert not torch.equal(outs[a], outs[b]), (a, b)
    from graphinvent_b200 import functional as Fn
    for mode in DTYPES:
        net2 = fresh()
        with _ctx(mode):
            out = net2(nodes, edges)
        Fn.kl_loss(out, target).backward()                      # outside the context
        want = got[seq.index(mode)][1]
        assert all(torch.equal(p.grad, g) for p, g in zip(net2.parameters(), want)), mode


# ---- 5. training, generation, RL -------------------------------------------------------------------------------------
def test_bf16_train_step_equals_eager_autocast_steps():
    """a bf16 TrainStep over a stream of different batches == eager module-API steps under autocast, bit for bit"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.optim import FlatAdam
    fx = load_small("GGNN")
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    B = nodes.shape[0]
    cap = int(edges.sum().item()) + 64
    batches = []
    for k in range(3):
        g = torch.Generator(device="cuda").manual_seed(k)
        perm = torch.randperm(B, device="cuda", generator=g)
        batches.append((nodes[perm].contiguous(), edges[perm].contiguous(), target[perm].contiguous()))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        step = T._train_step(T._net(fx["C"], fx["sd"]), B, cap)
    assert step.autocast_dtype is torch.bfloat16 and not step.tf32
    net = T._net(fx["C"], fx["sd"])
    net.entry_capacity = cap
    opt = FlatAdam(net.parameters(), lr=1e-3)
    for k, (n_, e_, t_) in enumerate(batches):
        step(n_, e_, t_)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(n_, e_)
        opt.zero_grad(set_to_none=True)
        Fn.kl_loss(out, t_).backward()
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(step.out, out), k
        for p, q in zip(step.params, net.parameters()):
            assert torch.equal(p, q), k


@pytest.mark.parametrize("model", MODELS)
def test_fifty_bf16_training_steps_stay_near_the_reference_loss_curve(model):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    z = np.load(os.path.join(GOLDEN, "loss_curves.npz"))
    fx = load_small(model)
    net = T._net(fx["C"], fx["sd"]).train()
    steps = int(z["steps"])
    opt = FlatAdam(net.parameters(), lr=float(z["lr"]))
    sch = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=float(z["max_lr"]), total_steps=steps)
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        step = TrainStep(net, opt, batch_size=nodes.shape[0], entry_capacity=int(edges.sum().item()) + 64)
    losses = []
    for _ in range(steps):
        losses.append(float(step(nodes, edges, target)))
        sch.step()
    dev = np.abs(np.array(losses) - z[f"loss/{model}"])
    tol = T.LOSS_TOL_TF32 * U["bf16"] / T.U11      # the TF32 tolerance scaled by the unit roundoff
    print(f"bf16 training {model}: max |loss - reference fp32| {dev.max():.3e} at step {int(dev.argmax())} "
          f"(bound {tol:.2e})")
    assert dev.max() <= tol
    assert losses[-1] < 0.6 * losses[0]


def test_fp16_grad_scaler_and_train_step_fallback():
    from graphinvent_b200 import functional as Fn
    C, sd, nodes, edges, target, o64, g64, _ = T._oracle("GGNN")
    net = T._net(C, sd)
    opt = torch.optim.SGD(net.parameters(), lr=0.0)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    with torch.autocast("cuda", dtype=torch.float16):
        loss = Fn.kl_loss(net(nodes.cuda(), edges.cuda()), target.cuda())
    scaler.scale(loss).backward()
    scaler.unscale_(opt)
    grads = [p.grad.detach().clone() for p in net.parameters()]
    scaler.step(opt)
    scaler.update()
    kink = _kink("GGNN", T.KINK_TAU * U["fp16"] / T.U11)
    gscale = max(g.norm().item() for g in g64.values())
    for (k, g), got in zip(g64.items(), grads):
        d = (got.cpu().double() - g).norm().item()
        assert d <= GRAD_C * U["fp16"] * g.norm().item() + kink[k] + 1e-7 * gscale, k
    fx = load_small("GGNN")
    n_, e_, t_ = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    cap = int(e_.sum().item()) + 64
    with torch.autocast("cuda", dtype=torch.float16):
        s16 = T._train_step(T._net(fx["C"], fx["sd"]), n_.shape[0], cap)
    assert s16.autocast_dtype is None and not s16.tf32
    s32 = T._train_step(T._net(fx["C"], fx["sd"]), n_.shape[0], cap)
    a, b = T._run_steps(s16, (n_, e_, t_)), T._run_steps(s32, (n_, e_, t_))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("model", MODELS)
def test_graphed_generator_equals_the_eager_loop_under_autocast(model, dt):
    from tests.test_gpu_generation_graphed import _assert_same, _eager, _graphed_batch, _small, _uniforms
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _small(model)
    B = 96
    Uu = _uniforms(C.max_n_nodes, B, 1)
    with torch.autocast("cuda", dtype=DTYPES[dt][0]):
        gen = GraphedGenerator(net, B, constants=C)
        assert gen.autocast_dtype is DTYPES[dt][0]
        got = _graphed_batch(gen, Uu)
        eager, want = _eager(net, C, B, Uu)
    _assert_same(gen, got, eager, want)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_rl_backward_under_autocast_matches_eager(dt):
    from tests.test_gpu_rl_graphed import _eager_replay, _finished_rollout, _loss
    dtype = DTYPES[dt][0]
    with torch.autocast("cuda", dtype=dtype):
        C, agent, prior, gen, Uu = _finished_rollout("GGNN")
        assert gen.autocast_dtype is dtype
        B = gen.batch_size
        _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=Uu)
    R = gen.rounds
    acts = gen.act_rec[:R].clone()
    _loss(agent_ll, prior_ll).backward()              # outside the context: the rollout's mode
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    with torch.autocast("cuda", dtype=dtype):
        _, (_, ll_a, ll_p, _) = _eager_replay(agent2, prior2, C, B, acts, gen.entry_capacity)
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total


def test_eval_step_refuses_a_train_step_of_another_mode():
    from graphinvent_b200.graphed import EvalStep
    fx = load_small("GGNN")
    net = T._net(fx["C"], fx["sd"])
    B = fx["nodes"].shape[0]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        step = T._train_step(net, B, 4096)
        EvalStep(net, batch_size=B, entry_capacity=4096, share=step)
    for mode in ("fp32", "tf32", "fp16"):
        with _ctx(mode):
            with pytest.raises(ValueError, match="precision"):
                EvalStep(net, batch_size=B, entry_capacity=4096, share=step)
