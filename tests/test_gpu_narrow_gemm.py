"""GPU: the narrow fp32 NT kernel (max(N, n_store) <= 48, several problems per launch) and the dispatch that uses it.

gib_tc_debug bit 4 restores the dispatch before it: narrow problems on sgemm_nt_kernel, mixed groups and the first-layer
input gradients of sibling MLPs problem by problem.  Every output of the new dispatch must equal that one bit for bit,
because each output keeps its accumulation order (one fmaf chain over k = 0 .. K-1) and its epilogue:
- single narrow problems with tensor cores off, across N, K, M and every epilogue, on 0xFF-poisoned outputs inside
  guard bands (the columns past n_store and the bands keep their poison);
- mixed groups with tensor cores on (wgmma members in one launch, narrow members in another), with device-side row
  counts and NaN pad rows around the live range;
- whole training steps of the four models through the module API (exact mode) and the captured TrainStep (capacity
  mode).
"""
import numpy as np
import pytest
import torch

from tests.guarded import Guarded
from tests.test_gpu_gemm_patterns import (EPI_ACT, EPI_ADD, EPI_MUL_DACT, TC_NT, _dev_int, _lib, _p, _planes,
                                          _profiled, _st)

pytestmark = pytest.mark.gpu

OLD = 16          # gib_tc_debug bit 4
SIMT_NT = 3       # profile class of the fp32 SIMT forward / dX launches
EPIS = [("selu", EPI_ACT, 1, True), ("linear", EPI_ACT, 0, False), ("dselu", EPI_MUL_DACT, 1, False),
        ("add", EPI_ADD, 0, False)]


class _mode:
    def __init__(self, tc, debug):
        self.tc, self.debug = tc, debug

    def __enter__(self):
        L = _lib().lib
        L.gib_set_tensor_cores(self.tc)
        L.gib_tc_debug(self.debug)

    def __exit__(self, *exc):
        L = _lib().lib
        L.gib_set_tensor_cores(1)
        L.gib_tc_debug(0)


class Prob:
    """one NT problem; C (and aux) live in poisoned guarded buffers with 4 spare columns; dyn: device-side row range
    [base, base + M) inside buffers of base + M + 5 rows whose A rows outside it are NaN"""

    def __init__(self, M, N, K, n_store, n_valid, epi, seed, dyn=False, base=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        _, self.mode, self.act, with_bias = epi
        self.M, self.N, self.K, self.n_store, self.n_valid, self.dyn = M, N, K, n_store, n_valid, dyn
        self.lo = base if dyn else 0
        self.rows = base + M + 5 if dyn else M
        self.A = torch.full((self.rows, K), float("nan"), device="cuda")
        self.A[self.lo:self.lo + M] = torch.randn(M, K, device="cuda", generator=g)
        self.W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        self.hl = _planes(self.W)
        self.bias = torch.randn(N, device="cuda", generator=g) if with_bias else None
        self.ldc = n_store + 4
        self.aux = None
        if self.mode != EPI_ACT:
            x = torch.randn(self.rows, self.ldc, device="cuda", generator=g) * 2
            self.aux = torch.selu(x) if self.mode == EPI_MUL_DACT else x
        self.m_dev = _dev_int(M) if dyn else None
        self.base_dev = _dev_int(base) if dyn else None

    def struct(self, C):
        s = _lib().GemmProblem()
        s.A, s.lda = _p(self.A), self.K
        s.W, s.ldw = _p(self.W), self.K
        s.W_hi, s.W_lo = _p(self.hl[0]), _p(self.hl[1])
        s.C, s.ldc = C.ptr(), self.ldc
        s.M, s.N, s.K = self.rows, self.N, self.K
        s.bias, s.act, s.mode = _p(self.bias), self.act, self.mode
        s.aux, s.ldaux = _p(self.aux), (self.ldc if self.aux is not None else 0)
        s.n_store, s.n_valid = self.n_store, self.n_valid
        s.m_dev, s.base_dev = _p(self.m_dev), _p(self.base_dev)
        return s


def _launch(ps, tc, debug):
    """run the problems as one gib_test_gemm_nt call: (guarded outputs, classes of the launches)"""
    L = _lib()
    Cs = [Guarded(p.rows * p.ldc * 4) for p in ps]
    arr = (L.GemmProblem * len(ps))(*[p.struct(c) for p, c in zip(ps, Cs)])
    with _mode(tc, debug):
        rc, cls = _profiled(lambda: L.lib.gib_test_gemm_nt(arr, len(ps), None, None, _st()))
    assert rc == 0, L.lib.gib_last_error().decode()
    torch.cuda.synchronize()
    for c in Cs:
        assert c.intact(), "guard band written"
    return Cs, cls


def _same_bits(new, old, ps):
    for i, (a, b, p) in enumerate(zip(new, old, ps)):
        va, vb = a.view(torch.int32, (p.rows, p.ldc)), b.view(torch.int32, (p.rows, p.ldc))
        assert torch.equal(va, vb), f"problem {i}: {int((va != vb).sum())} words differ from the old dispatch"
        assert bool((va[:, p.n_store:] == -1).all()), f"problem {i}: columns past n_store written"
        if p.dyn:
            assert bool((va[:p.lo] == -1).all()) and bool((va[p.lo + p.M:] == -1).all()), "rows outside the range"


@pytest.mark.parametrize("M", [1, 127, 1024, 13312])
@pytest.mark.parametrize("N", [1, 3, 16, 39, 45, 48])
def test_narrow_kernel_bit_identical(N, M):
    """every epilogue, K from 16 to 704, n_store >= N, n_valid < n_store: the narrow kernel against sgemm_nt_kernel"""
    for e, epi in enumerate(EPIS):
        K = [16, 64, 512, 704][(e + N + M) % 4]
        n_store = min(48, N + (e % 3) * 3)
        n_valid = max(1, n_store - 2)
        p = Prob(M, N, K, n_store, n_valid, epi, seed=N * 100 + e + M)
        new, cls_new = _launch([p], tc=0, debug=0)
        old, cls_old = _launch([p], tc=0, debug=OLD)
        assert cls_new == [SIMT_NT] and cls_old == [SIMT_NT]
        _same_bits(new, old, [p])


@pytest.mark.parametrize("M", [127, 1024, 13312])
def test_narrow_group_one_launch(M):
    """up to four narrow problems in one launch, each with its own column tile"""
    ps = [Prob(M, n, 512, n, n, EPIS[i % 4], seed=i) for i, n in enumerate([1, 3, 39, 45])]
    new, cls_new = _launch(ps, tc=0, debug=0)
    old, cls_old = _launch(ps, tc=0, debug=OLD)
    assert cls_new == [SIMT_NT] and cls_old == [SIMT_NT] * 4
    _same_bits(new, old, ps)


def test_mixed_group_host_rows():
    """the tier-2 output layer's shape: a wide member on the wgmma kernel, two narrow ones in one narrow launch, and a
    member too short for the wgmma kernel on its own (M < 256) that stays on sgemm_nt_kernel"""
    ps = [Prob(1024, 592, 512, 592, 585, EPIS[0], seed=1), Prob(1024, 48, 512, 39, 39, EPIS[0], seed=2),
          Prob(1024, 16, 512, 1, 1, EPIS[0], seed=3), Prob(200, 64, 64, 64, 64, EPIS[1], seed=4)]
    new, cls_new = _launch(ps, tc=1, debug=0)
    old, cls_old = _launch(ps, tc=1, debug=OLD)
    assert sorted(cls_old) == [TC_NT, TC_NT, SIMT_NT, SIMT_NT]
    assert sorted(cls_new) == [TC_NT, SIMT_NT, SIMT_NT]
    _same_bits(new, old, ps)


@pytest.mark.parametrize("M", [1, 300, 5000])
def test_mixed_group_device_rows(M):
    """wgmma members on device-side row counts (NaN pad rows around the range) and a narrow host-row member"""
    ps = [Prob(M, 128, 128, 128, 128, EPIS[2], seed=5, dyn=True, base=37),
          Prob(M, 128, 64, 128, 100, EPIS[3], seed=6, dyn=True, base=3),
          Prob(max(M, 1), 16, 512, 3, 3, EPIS[0], seed=7)]
    new, cls_new = _launch(ps, tc=1, debug=0)
    old, cls_old = _launch(ps, tc=1, debug=OLD)
    assert sorted(cls_old) == [TC_NT, TC_NT, SIMT_NT] and sorted(cls_new) == [TC_NT, SIMT_NT]
    _same_bits(new, old, ps)


# ---- whole training steps -------------------------------------------------------------------------------------------
def _batch(model, B, seed):
    from graphinvent_b200 import synthetic as S
    from oracle import mpnn_oracle as O
    C = O.make_constants(model)
    n, e = S.random_graphs(B, C.max_n_nodes, 5, 3, seed=seed)
    apd = C.max_n_nodes * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
    return C, torch.from_numpy(n).float(), torch.from_numpy(e).float(), torch.from_numpy(S.random_targets(B, apd, seed))


def _module_step(model, debug):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C, n, e, t = _batch(model, 300, seed=11)
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=3))
    net = net.cuda()
    with _mode(1, debug):
        out = net(n.cuda(), e.cuda())
        loss = Fn.kl_loss(out, t.cuda())
        loss.backward()
        torch.cuda.synchronize()
    return [out.detach(), loss.detach()] + [p.grad.clone() for p in net.parameters()]


def _captured_steps(model, debug):
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    from oracle import mpnn_oracle as O
    C, n, e, t = _batch(model, 256, seed=12)
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=4))
    net = net.cuda()
    opt = FlatAdam(net.parameters(), lr=1e-3)
    with _mode(1, debug):
        step = TrainStep(net, opt, batch_size=256, entry_capacity=int((e != 0).sum()) + 256, input_dtype=torch.float32)
        losses = []
        for k in range(3):
            C2, n2, e2, t2 = _batch(model, 256 - 40 * k, seed=20 + k)
            step.load(n2, e2, t2)
            losses.append(step().detach().clone())
        torch.cuda.synchronize()
    return losses + [step.out.detach().clone()] + [p.detach().clone() for p in net.parameters()]


def _assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"tensor {i} differs from the old dispatch"


@pytest.mark.parametrize("model", ["GGNN", "MNN", "AttGGNN", "EMN"])
def test_module_step_bit_identical(model):
    _assert_same(_module_step(model, 0), _module_step(model, OLD))


@pytest.mark.parametrize("model", ["GGNN", "MNN", "AttGGNN", "EMN"])
def test_captured_steps_bit_identical(model):
    _assert_same(_captured_steps(model, 0), _captured_steps(model, OLD))


def test_launch_count_drops():
    """the eager GGNN step launches fewer kernels with the new dispatch"""
    L = _lib().lib
    counts = []
    for debug in (0, OLD):
        _module_step("GGNN", debug)
        c0 = L.gib_launch_count()
        _module_step("GGNN", debug)
        counts.append(L.gib_launch_count() - c0)
    assert counts[0] < counts[1], counts
