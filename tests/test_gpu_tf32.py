"""GPU: single-pass TF32 mode (torch's fp32 matmul precision "tf32").

1. Every GEMM call pattern of tests/test_gpu_gemm_patterns.py with tf32 = 1 through the test hooks, against float64
   evaluated on the TF32-ROUNDED operands: what remains is fp32 accumulation, so a wrong rounding or a lo term left in
   shows up at 2^-11, far above the bound.  Sentinels, pad columns and kernel classes are checked as there.
2. `config.tf32_enabled()` agrees with what torch's own CUDA matmul does under every way of setting the flag.
3. The four models, float and int8 inputs, exact and capacity mode: logits and parameter gradients against the fp64
   oracle, within the TF32 error model (one rounding of 2^-11 relative per operand) plus the SELU-kink band.
4. No leakage between modes: eager and captured results of the default mode keep their bits.
5. Training follows the reference's fp32 loss curve; generation and the RL rollout stay bit-identical between the
   captured and the eager path in TF32 mode.
"""
import contextlib
import copy
import os

import numpy as np
import pytest
import torch

import tests.test_gpu_gemm_patterns as P
from tests.conftest import GOLDEN, MODELS, load_small

pytestmark = pytest.mark.gpu

# 4 x (rounded up) the worst |C - C64(rounded operands)| / (|A_r| |W_r|^T) over the sweep, measured on an H100 80GB HBM3
# (SXM): see DESIGN.md section 4
EPS_TF32 = 3.0e-6      # measured worst 7.41e-7 (the group of 16 weight gradients)
WORST = {}


@contextlib.contextmanager
def precision(matmul=None, glob=None, legacy=None):
    """set torch's fp32 matmul precision for the block (new per-backend / global API or the legacy setter) and restore
    both new-API values afterwards"""
    m, g = torch.backends.cuda.matmul.fp32_precision, torch.backends.fp32_precision
    try:
        if legacy is not None:
            torch.set_float32_matmul_precision(legacy)
        if glob is not None:
            torch.backends.fp32_precision = glob
        if matmul is not None:
            torch.backends.cuda.matmul.fp32_precision = matmul
        yield
    finally:
        torch.backends.fp32_precision = g
        torch.backends.cuda.matmul.fp32_precision = m


def rna(x):
    """TF32 round to nearest, ties away (gib_model_pack's cvt.rna and the kernels' integer form)"""
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nTF32 worst error / magnitude:", {k: f"{v[0]:.3g} ({v[1]})" for k, v in sorted(WORST.items())})


def _within(got, ref, mag, what, slack=0.0):
    err = (got.double() - ref).abs()
    ratio = ((err - slack).clamp(min=0) / (mag + 1e-300)).max().item() if err.numel() else 0.0
    if ratio >= WORST.get("tf32", (0.0, ""))[0]:
        WORST["tf32"] = (ratio, what)
    assert ratio <= EPS_TF32, f"{what}: error / magnitude {ratio:.3g} > {EPS_TF32:.1e}"


# ---- 1. call patterns ------------------------------------------------------------------------------------------------
def _run_nt1(nts, dep=None, tf32=1):
    """P._run_nt with the precision field set on every problem"""
    import ctypes
    L = P._lib()
    structs = [t.struct() for t in nts]
    for s in structs:
        s.tf32 = tf32
    arr = (L.GemmProblem * len(nts))(*structs)
    flags = None
    if dep is not None:
        nb = L.lib.gib_test_chain_flag_bytes(arr, len(nts))
        flags = torch.full((max(nb // 4, 1),), 12345, dtype=torch.int32, device="cuda")
        dep = (ctypes.c_int * len(nts))(*dep)
    return P._profiled(lambda: L.lib.gib_test_gemm_nt(arr, len(nts), dep, P._p(flags), P._st()))


def _check_nt1(t, what):
    """P.NT.check on the TF32-rounded A and W, with the fp32-accumulation bound"""
    lo, hi, ns, nv = t.lo, t.hi, t.n_store, t.n_valid
    A64 = rna(t.A[lo:hi, :t.K]).double()
    Wp = torch.zeros(max(t.N, ns), t.K, dtype=torch.float64, device="cuda")
    Wp[:t.N] = rna(t.W).double()
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
    _within(out[:, :nv], ref[:, :nv], mag[:, :nv], what, slack)
    assert (out[:, nv:ns] == 0).all() and not torch.signbit(out[:, nv:ns]).any(), f"{what}: pad columns not +0"
    P._same_bits(out[:, ns:], t.C0[lo:hi, ns:], what + " columns >= n_store")
    P._same_bits(t.C[:lo], t.C0[:lo], what + " rows before the range")
    P._same_bits(t.C[hi:], t.C0[hi:], what + " rows after the range")


@pytest.mark.parametrize("M", [1, 65, 129, 4097])
@pytest.mark.parametrize("N", [48, 129, 200, 608])
def test_nt_shapes_and_epilogues_tf32(M, N):
    """every epilogue: the tensor-core kernel through a device-side row count (any M), and the dispatcher's own choice
    where that is the tensor-core kernel (pre-split W on wgmma, and raw W on the mma.sync kernel)"""
    for K in (16, 48, 160, 688):
        for label, kw in P._epilogues(N):
            kw = dict(kw)
            lda = K + kw.pop("lda_pad", 0)
            for run in ("tc", "dispatch", "raw"):
                what = f"M={M} N={N} K={K} {label} [{run}]"
                dyn = dict(cap=M + 5, base=3) if run == "tc" else {}
                t = P.NT(M, N, K, lda=lda, planes=run != "raw", **kw, **dyn)
                if P._expect_single(t, 1, 0) != [P.TC_NT]:
                    continue
                rc, cls = _run_nt1([t])
                assert rc == 0, what + ": " + P._lib().lib.gib_last_error().decode()
                assert cls == [P.TC_NT], f"{what}: kernel classes {cls}"
                _check_nt1(t, what)


@pytest.mark.parametrize("case", list(P._group_cases()))
def test_nt_groups_tf32(case):
    """a group that does not qualify for one grouped launch (k16 member) runs member by member: each member is checked
    against the path the dispatch rule gives it, the fp32 SIMT kernel or the TF32 tensor-core kernel"""
    nts = P._group_cases()[case]()
    rc, cls = _run_nt1(nts)
    assert rc == 0, P._lib().lib.gib_last_error().decode()
    assert cls == P._expect_group(nts, 1, 0) and P.TC_NT in cls, f"{case}: kernel classes {cls}"
    assert (cls == [P.TC_NT]) == (case != "k16 member"), f"{case}: kernel classes {cls}"
    for i, t in enumerate(nts):
        if cls == [P.TC_NT] or P._expect_single(t, 1, 0) == [P.TC_NT]:
            _check_nt1(t, f"{case} member {i}")
        else:
            t.check("simt", f"{case} member {i} [simt]")


def test_nt_raw_weights_grouped_tf32():
    nts = [P.NT(2000, 256, 144, act=1, planes=False), P.NT(1500, 128, 48, mode=P.EPI_ADD, planes=False)]
    with P._mode(debug=1):
        rc, cls = _run_nt1(nts)
    assert rc == 0 and cls == [P.TC_NT]
    for i, t in enumerate(nts):
        _check_nt1(t, f"raw member {i}")


@pytest.mark.parametrize("case", list(P._chain_cases()))
def test_nt_chains_tf32(case):
    nts, dep = P._chain(**P._chain_cases()[case])
    rc, cls = _run_nt1(nts, dep)
    assert rc == 0, P._lib().lib.gib_last_error().decode()
    assert cls == [P.TC_NT], f"{case}: one chain launch expected, got {cls}"
    for k, t in enumerate(nts):
        _check_nt1(t, f"{case} problem {k}")


def test_mixed_precisions_in_one_launch_are_refused():
    nts = [P.NT(1000, 256, 144, act=1), P.NT(1300, 128, 64, act=1)]
    L = P._lib()
    structs = [t.struct() for t in nts]
    structs[1].tf32 = 1
    arr = (L.GemmProblem * 2)(*structs)
    rc, cls = P._profiled(lambda: L.lib.gib_test_gemm_nt(arr, 2, None, None, P._st()))
    assert rc < 0 and cls == [] and b"precision" in L.lib.gib_last_error()
    for t in nts:
        t.untouched("refused")


def test_tf32_differs_from_3xtf32_and_is_deterministic():
    """the mode takes effect: the same problem gives another result than 3xTF32, and the same bits twice"""
    outs = []
    for tf32 in (0, 1, 1):
        t = P.NT(4097, 256, 688, act=1, seed=3)
        rc, cls = _run_nt1([t], tf32=tf32)
        assert rc == 0 and cls == [P.TC_NT]
        outs.append(t.C.clone())
    assert not torch.equal(outs[0], outs[1])
    assert torch.equal(outs[1], outs[2])
    rel = ((outs[0] - outs[1]).abs().max() / outs[0].abs().max()).item()
    assert 1e-5 < rel < 1e-2, rel


class _RoundedDW:
    """a P.DW problem read through rounded operands: G and X replaced by rna(G), rna(X) for the fp64 check only
    (the bias sums stay sums of the raw G)"""

    def __init__(self, q):
        self.q = q

    def contribution(self):
        q = self.q
        idx, _, _, b, bm = q.contribution()
        lo, hi = q.live()
        r = torch.arange(q.R, device="cuda")
        prow = (r // q.Rb) * q.Rbp + r % q.Rb
        G = rna(q.G[lo:hi]).double()[:, prow]
        X = rna(q.X[lo:hi, :q.C].contiguous()).double()
        return idx, G.t() @ X, G.abs().t() @ X.abs(), b, bm


def _run_dw1(groups, plan_rows=0, debug=0):
    """P._run_dw with tf32 = 1 on every problem; the check compares against the rounded-operand fp64 sums"""
    import ctypes
    L = P._lib()
    flat = [q for g in groups for q in g]
    structs = [q.struct() for q in flat]
    for s in structs:
        s.tf32 = 1
    arr = (L.DwProblem * len(flat))(*structs)
    sizes = (ctypes.c_int * len(groups))(*[len(g) for g in groups])
    nb = L.lib.gib_test_dw_scratch_bytes(arr, sizes, len(groups), plan_rows)
    scratch = torch.full((nb // 4,), P.NAN, device="cuda")
    dsts = {}
    for q in flat:
        for t in (q.dW, q.dbias):
            if t is not None:
                dsts.setdefault(P._root(t).data_ptr(), (P._root(t), P._root(t).clone()))
    with P._mode(tc=1, debug=debug):
        rc, cls = P._profiled(lambda: L.lib.gib_test_dw_groups(arr, sizes, len(groups), plan_rows, P._p(scratch),
                                                               P._st()))

    def check(what):
        for base_ptr, (t, t0) in dsts.items():
            ref, mag = t0.double().flatten().clone(), t0.double().abs().flatten().clone()
            for q in flat:
                idx, w, wm, b, bm = _RoundedDW(q).contribution()
                if q.dW is not None and P._root(q.dW).data_ptr() == base_ptr:
                    idx = (idx + (q.dW.data_ptr() - base_ptr) // 4).flatten()
                    ref.index_add_(0, idx, w.flatten())
                    mag.index_add_(0, idx, wm.flatten())
                if q.dbias is not None and P._root(q.dbias).data_ptr() == base_ptr:
                    idx = torch.arange(q.R, device="cuda") + (q.dbias.data_ptr() - base_ptr) // 4
                    ref.index_add_(0, idx, b)
                    mag.index_add_(0, idx, bm)
            _within(t.flatten(), ref, mag, what)

    return rc, cls, check


@pytest.mark.parametrize("debug", [0, 1])
@pytest.mark.parametrize("M", [2048, 4097, 40000])
def test_dw_single_tf32(M, debug):
    G, X = P._operands(M, 112, 144, 100, 136, seed=M)
    groups = [[P.DW(G, X, M, torch.randn(100, 136, device="cuda"), 100, 136, dbias=torch.randn(100, device="cuda"))]]
    rc, cls, check = _run_dw1(groups, debug=debug)
    assert rc == 0 and cls == [P.TC_DW], cls
    check(f"dW M={M} debug={debug}")


def test_dw_gate_blocked_mnn_slices_and_group_of_16_tf32():
    H, C, M = 100, 136, 4097
    Hp = P.pad16(H)
    G, X = P._operands(M, 3 * Hp, 144, 3 * H, C, seed=7)
    for g in range(3):
        G[:, g * Hp + H:(g + 1) * Hp] = 0
    gate = [[P.DW(G, X, M, torch.randn(3 * H, C, device="cuda"), 3 * H, C, dbias=torch.randn(3 * H, device="cuda"),
                  Rb=H, Rbp=Hp)]]
    rc, cls, check = _run_dw1(gate)
    assert rc == 0 and cls == [P.TC_DW], cls
    check("gate-blocked")
    R, H2, Ef = 100, 64, 3
    big = torch.randn(R, H2, Ef, device="cuda")
    db = torch.randn(R, device="cuda")
    grp = []
    for t, m in enumerate((2048, 1500, 700)):
        G, X = P._operands(m, P.pad16(R), H2, R, H2, seed=40 + t)
        grp.append(P.DW(G, X, m, P._slice_dst(big, t), R, H2, dbias=db if t == 0 else None, rs=H2 * Ef, cs=Ef))
    rc, cls, check = _run_dw1([grp])
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
    rc, cls, check = _run_dw1([grp], plan_rows=3 * sum(s[0] for s in shapes))
    assert rc == 0 and cls == [P.TC_DW], cls
    check("group of 16")


def test_dw_device_side_rows_and_consecutive_groups_tf32():
    cap = 8192
    grp = P._shared_buffer_group(cap, 112, 144, 100, 136, [(0, 1900), (2048, 0), (4096, 3000), (8064, 500)], seed=9)
    rc, cls, check = _run_dw1([grp], plan_rows=cap)
    assert rc == 0 and cls == [P.TC_DW], cls
    check("device-side rows")
    R, C = 100, 136
    dsts = [(torch.randn(R, C, device="cuda"), torch.randn(R, device="cuda")) for _ in range(3)]
    groups, seed = [], 300
    for sizes in ((4097, 2500), (3000, 2048, 2600), (40000,)):
        g = []
        for k, m in enumerate(sizes):
            seed += 1
            G, X = P._operands(m, 112, 144, R, C, seed=seed)
            g.append(P.DW(G, X, m, dsts[k][0], R, C, dbias=dsts[k][1]))
        groups.append(g)
    rc, cls, check = _run_dw1(groups)
    assert rc == 0 and cls == [P.TC_DW] * 3, cls
    check("consecutive groups")


# ---- 2. the switch agrees with torch ---------------------------------------------------------------------------------
SETTINGS = [dict(), dict(legacy="highest"), dict(legacy="high"), dict(legacy="medium"),
            dict(matmul="tf32"), dict(matmul="ieee"), dict(glob="tf32", matmul="none"), dict(glob="ieee", matmul="none"),
            dict(glob="tf32", matmul="ieee"), dict(glob="ieee", matmul="tf32"),
            dict(legacy="high", matmul="ieee"), dict(legacy="highest", matmul="tf32")]


@pytest.mark.parametrize("setting", SETTINGS, ids=[",".join(f"{k}={v}" for k, v in s.items()) or "default"
                                                    for s in SETTINGS])
def test_tf32_enabled_matches_torch_matmul(setting):
    """operands whose fp32 and TF32 products differ visibly: torch's own result says which one it computed"""
    from graphinvent_b200.config import tf32_enabled
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(256, 512, device="cuda", generator=g)
    b = torch.randn(512, 256, device="cuda", generator=g)
    exact = (a.double() @ b.double())
    rounded = (rna(a).double() @ rna(b).double())
    with precision(**setting):
        enabled = tf32_enabled()
        c = (a @ b).double()
    torch_tf32 = (c - rounded).abs().max() < (c - exact).abs().max()
    assert enabled == bool(torch_tf32), (setting, enabled, float((c - exact).abs().max()))


# ---- 3. models against the fp64 oracle -------------------------------------------------------------------------------
# TF32 error model: one rounding of 2^-11 relative per GEMM operand, fp32 accumulation.  Logits: per molecule
# |o - o64| <= LOGIT_C * 2^-11 * (1 + max |o64|); gradients, per tensor (L2): |g - g64| <= GRAD_C * 2^-11 * |g64| + the
# SELU-kink band of the oracle at KINK_TAU (the oracle's gradient with every SELU input within tau of 0 taken on its
# left or its right side) + 1e-7 of the largest tensor's norm.  Constants: 4 x the worst measured ratio, DESIGN.md 4.
U11 = 2.0 ** -11
LOGIT_C = 16.5         # measured worst 4.1 (GGNN)
GRAD_C = 22.0          # measured worst <= 5.5 (EMN fTermNet2 weight, kink band and floor included)
KINK_TAU = 3e-3
_ORACLE = {}


def _oracle(model):
    if model not in _ORACLE:
        from graphinvent_b200 import synthetic as S
        from oracle import mpnn_oracle as O
        C = O.make_constants(model)
        sd = O.init_state_dict(C, seed=11)
        n, e = S.random_graphs(96, 13, 5, 3, seed=12, min_atoms=0)
        n2, e2 = S.corner_case_graphs(13, 8)
        nodes = torch.from_numpy(np.concatenate([n2, n])).float()
        edges = torch.from_numpy(np.concatenate([e2, e])).float()
        target = torch.from_numpy(S.random_targets(nodes.shape[0], 625, seed=3))
        _, o64, g64 = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
        try:
            O.KINK = (KINK_TAU, "L")
            _, _, gL = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
            O.KINK = (KINK_TAU, "R")
            _, _, gR = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
        finally:
            O.KINK = None
        _ORACLE[model] = (C, sd, nodes, edges, target, o64, g64, {k: (gL[k] - gR[k]).norm().item() for k in g64})
    return _ORACLE[model]


def _net(C, sd):
    from graphinvent_b200.gnn import mpnn
    net = mpnn.create(C)
    net.load_state_dict(sd)
    return net.cuda()


def _eager_step(net, nodes, edges, target):
    from graphinvent_b200 import functional as Fn
    net.zero_grad()
    out = net(nodes.cuda(), edges.cuda())
    Fn.kl_loss(out, target.cuda()).backward()
    return out.detach(), [p.grad.detach().clone() for p in net.parameters()]


@pytest.mark.parametrize("capacity", [False, True])
@pytest.mark.parametrize("int8", [False, True])
@pytest.mark.parametrize("model", MODELS)
def test_models_against_fp64_in_tf32_mode(model, int8, capacity):
    C, sd, nodes, edges, target, o64, g64, kink = _oracle(model)
    net = _net(C, sd)
    if capacity:
        net.entry_capacity = int(edges.sum().item()) + 64
    if int8:
        nodes, edges = nodes.to(torch.int8), edges.to(torch.int8)
    with precision(matmul="tf32"):
        out, grads = _eager_step(net, nodes, edges, target)
    with precision(matmul="ieee"):
        out3, _ = _eager_step(net, nodes, edges, target)
    assert not torch.equal(out, out3), "TF32 mode gave the 3xTF32 logits"
    e = (out.cpu().double() - o64).abs().max(1).values
    lim = LOGIT_C * U11 * (1 + o64.abs().max(1).values)
    ratio_l = (e / lim).max().item()
    gscale = max(g.norm().item() for g in g64.values())
    ratio_g, worst = 0.0, ""
    for (k, g), got in zip(g64.items(), grads):
        d = (got.cpu().double() - g).norm().item()
        bound = GRAD_C * U11 * g.norm().item() + kink[k] + 1e-7 * gscale
        if d / bound > ratio_g:
            ratio_g, worst = d / bound, k
    print(f"TF32 {model} int8={int8} capacity={capacity}: logits max |o - o64| {e.max().item():.3e} "
          f"({ratio_l:.3f} of bound), worst gradient {worst} {ratio_g:.3f} of bound")
    assert ratio_l <= 1.0 and ratio_g <= 1.0


# ---- 4. no leakage ---------------------------------------------------------------------------------------------------
def _train_step(net, B, cap):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    opt = FlatAdam(net.parameters(), lr=1e-3)
    return TrainStep(net, opt, batch_size=B, entry_capacity=cap)


def _run_steps(step, batch, n=3):
    nodes, edges, target = batch
    losses = [step(nodes, edges, target).clone() for _ in range(n)]
    return torch.stack(losses), torch.cat([p.detach().reshape(-1) for p in step.params])


def test_modes_do_not_leak_into_each_other():
    fx = load_small("GGNN")
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    cap = int(edges.sum().item()) + 64
    results = []
    for p in ("ieee", "tf32", "ieee"):
        with precision(matmul=p):
            net = _net(fx["C"], fx["sd"])
            net.entry_capacity = cap
            out, grads = _eager_step(net, nodes, edges, target)
            net2 = _net(fx["C"], fx["sd"])
            step = _train_step(net2, nodes.shape[0], cap)
            assert step.tf32 == (p == "tf32")
            losses, params = _run_steps(step, (nodes, edges, target))
        results.append((out, torch.cat([g.reshape(-1) for g in grads]), losses, params))
    for a, b in zip(results[0], results[2]):
        assert torch.equal(a, b)
    assert not torch.equal(results[0][0], results[1][0]) and not torch.equal(results[0][3], results[1][3])
    # a TrainStep keeps the mode of its construction when the global flips
    for p, q in (("tf32", "ieee"), ("ieee", "tf32")):
        with precision(matmul=p):
            s1 = _train_step(_net(fx["C"], fx["sd"]), nodes.shape[0], cap)
            want = _run_steps(s1, (nodes, edges, target))
            s2 = _train_step(_net(fx["C"], fx["sd"]), nodes.shape[0], cap)
        with precision(matmul=q):
            got = _run_steps(s2, (nodes, edges, target))
        assert torch.equal(want[0], got[0]) and torch.equal(want[1], got[1]), (p, q)


def test_eval_step_refuses_a_train_step_of_the_other_mode():
    from graphinvent_b200.graphed import EvalStep
    fx = load_small("GGNN")
    net = _net(fx["C"], fx["sd"])
    B = fx["nodes"].shape[0]
    with precision(matmul="tf32"):
        step = _train_step(net, B, 4096)
        EvalStep(net, batch_size=B, entry_capacity=4096, share=step)
    with precision(matmul="ieee"):
        with pytest.raises(ValueError, match="precision"):
            EvalStep(net, batch_size=B, entry_capacity=4096, share=step)


# ---- 5. training, generation, RL -------------------------------------------------------------------------------------
# max |loss - reference fp32 loss| over the 50 steps in TF32 mode; 4 x the worst measured (DESIGN.md 4)
LOSS_TOL_TF32 = 1.3e-4   # measured worst 3.07e-5 (AttGGNN, step 28)


@pytest.mark.parametrize("model", MODELS)
def test_fifty_tf32_training_steps_follow_the_reference_loss_curve(model):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    z = np.load(os.path.join(GOLDEN, "loss_curves.npz"))
    fx = load_small(model)
    net = _net(fx["C"], fx["sd"]).train()
    steps = int(z["steps"])
    opt = FlatAdam(net.parameters(), lr=float(z["lr"]))
    sch = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=float(z["max_lr"]), total_steps=steps)
    nodes, edges, target = fx["nodes"].cuda(), fx["edges"].cuda(), fx["target"].cuda()
    with precision(matmul="tf32"):
        step = TrainStep(net, opt, batch_size=nodes.shape[0], entry_capacity=int(edges.sum().item()) + 64)
    assert step.tf32
    losses = []
    for _ in range(steps):
        losses.append(float(step(nodes, edges, target)))
        sch.step()
    dev = np.abs(np.array(losses) - z[f"loss/{model}"])
    print(f"TF32 training {model}: max |loss - reference fp32| {dev.max():.3e} at step {int(dev.argmax())}")
    assert dev.max() <= LOSS_TOL_TF32, (model, int(dev.argmax()), float(dev.max()))
    assert losses[-1] < 0.6 * losses[0]


@pytest.mark.parametrize("model", MODELS)
def test_graphed_generator_equals_the_eager_loop_in_tf32_mode(model):
    from tests.test_gpu_generation_graphed import _assert_same, _eager, _graphed_batch, _small, _uniforms
    from graphinvent_b200.graphed import GraphedGenerator
    C, net = _small(model)
    B = 96
    U = _uniforms(C.max_n_nodes, B, 1)
    with precision(matmul="tf32"):
        gen = GraphedGenerator(net, B, constants=C)
        assert gen.tf32
        got = _graphed_batch(gen, U)
        eager, want = _eager(net, C, B, U)
    _assert_same(gen, got, eager, want)


@pytest.mark.parametrize("model", ["GGNN", "EMN"])
def test_rl_backward_in_tf32_mode_matches_eager_and_ignores_a_later_flip(model):
    from tests.test_gpu_rl_graphed import _eager_replay, _finished_rollout, _grads, _loss
    with precision(matmul="tf32"):
        C, agent, prior, gen, U = _finished_rollout(model)
        assert gen.tf32
        B = gen.batch_size
        _, agent_ll, prior_ll, _ = gen.sample(agent, prior, uniforms=U)
    R = gen.rounds
    p_a, p_b, acts = gen.p_a[:R].clone(), gen.p_b[:R].clone(), gen.act_rec[:R].clone()
    with precision(matmul="ieee"):             # flipped between the rollout and its backward
        _loss(agent_ll, prior_ll).backward()
    assert torch.equal(gen.recomputed_p[0][:R], p_a) and torch.equal(gen.recomputed_p[1][:R], p_b)
    agent2, prior2 = copy.deepcopy(agent), copy.deepcopy(prior)
    agent2.zero_grad()
    prior2.zero_grad()
    with precision(matmul="tf32"):
        eager, (_, ll_a, ll_p, _) = _eager_replay(agent2, prior2, C, B, acts, gen.entry_capacity)
    assert torch.allclose(ll_a, agent_ll, rtol=1e-5, atol=1e-6) and torch.allclose(ll_p, prior_ll, rtol=1e-5, atol=1e-6)
    with precision(matmul="ieee"):             # the eager backward runs in its forward's mode too
        _loss(ll_a, ll_p).backward()
    for m, m2 in ((agent, agent2), (prior, prior2)):
        total = sum(p.grad.norm().item() ** 2 for p in m2.parameters()) ** 0.5
        for p, p2 in zip(m.parameters(), m2.parameters()):
            assert (p.grad - p2.grad).norm().item() <= 1e-4 * p2.grad.norm().item() + 1e-5 * total
    assert _grads(agent)[0] is not None
