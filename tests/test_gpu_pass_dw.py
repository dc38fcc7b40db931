"""GPU: the weight gradients of the pass-shared weights (GGNN / MNN message MLPs, GRU) reduced once over all message
passes after the pass loop, all in one grouped launch with a pass extent, against gib_tc_debug bit 5, which launches
them pass by pass as before.

The forward is the same, so logits and loss agree to the bit; so do the gradients of every weight that is not shared
across passes, and the Adam step of those weights.  The shared weights' gradients are the same products summed in
another fp32 order (one fixed-order sum over all passes' k-blocks instead of one sum per pass added into the gradient),
and the tensor cores' fp32 accumulation is not rounded to nearest: each element stays within 2^-15 of the tensor's
largest magnitude (512 units in its last place; a lost or repeated pass would be off by a whole pass's share), and the
deferred result is the same bits run after run.  Every buffer sits in a guarded allocation with poisoned interiors
(tests/test_gpu_buffer_bounds.run_step), in exact mode and in capacity mode, in 3xTF32, TF32 and bf16.
"""
import ctypes

import pytest
import torch

from tests.test_gpu_buffer_bounds import _assert_intact, _bits_equal, run_step

pytestmark = pytest.mark.gpu

PER_PASS = 32          # gib_tc_debug bit 5
SHARED = ("msg_nns.", "message_weights", "gru.")
REL = 2.0 ** -15


def _lib():
    from graphinvent_b200._lib import lib
    return lib


class _mode:
    """gib_tc_debug bits and the matmul precision (0 = 3xTF32, 1 = TF32, 2 = bf16 autocast) of the calls inside"""

    def __init__(self, debug, prec):
        self.debug, self.prec = debug, prec

    def __enter__(self):
        _lib().gib_tc_debug(self.debug)
        self.old = torch.backends.cuda.matmul.fp32_precision
        torch.backends.cuda.matmul.fp32_precision = "tf32" if self.prec == 1 else "ieee"
        self.ac = torch.autocast("cuda", dtype=torch.bfloat16) if self.prec == 2 else None
        if self.ac:
            self.ac.__enter__()

    def __exit__(self, *exc):
        if self.ac:
            self.ac.__exit__(*exc)
        torch.backends.cuda.matmul.fp32_precision = self.old
        _lib().gib_tc_debug(0)


def _case(model, B, seed=7):
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = O.make_constants(model)
    n, e = S.random_graphs(B, C.max_n_nodes, 5, 3, seed=seed)
    apd = C.max_n_nodes * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=seed))
    net = net.cuda()
    return (C, net, torch.from_numpy(n).float().cuda(), torch.from_numpy(e).float().cuda(),
            torch.from_numpy(S.random_targets(B, apd, seed)).float().cuda())


def _slices(net):
    """(name, shared, slice of the flat gradient bucket) per parameter"""
    out, o = [], 0
    for name, p in net.named_parameters():
        out.append((name, name.startswith(SHARED), slice(o, o + p.numel())))
        o += p.numel()
    return out


def _compare(net, new, old, what):
    assert _bits_equal(new["out"], old["out"]), f"{what}: logits differ"
    assert _bits_equal(new["loss"], old["loss"]), f"{what}: loss differs"
    shared, worst = 0, 0.0
    for name, sh, s in _slices(net):
        a, b = new["grads"][s], old["grads"][s]
        if not sh:
            assert _bits_equal(a, b), f"{what}: gradient of {name} (not shared across passes) differs"
            assert _bits_equal(new["params"][s], old["params"][s]), f"{what}: Adam step of {name} differs"
            continue
        shared += 1
        ratio = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
        worst = max(worst, ratio)
        assert ratio <= REL, f"{what}: gradient of {name} off by {ratio:.3e} of its largest magnitude"
    assert shared >= 3
    print(f"{what}: shared-weight gradients within {worst:.3e} of their largest magnitudes")


def _step(net, n, e, t, cap, debug, prec):
    with _mode(debug, prec):
        r = run_step(net, n, e, t, cap, "poison")
    _assert_intact(r["g"], f"debug {debug} prec {prec}")
    return r


@pytest.mark.parametrize("prec", [0, 1, 2])
@pytest.mark.parametrize("mode", ["exact", "capacity"])
@pytest.mark.parametrize("model", ["GGNN", "MNN"])
def test_deferred_matches_per_pass(model, mode, prec):
    C, net, n, e, t = _case(model, 300)
    cap = None if mode == "exact" else int((e != 0).sum()) + 300
    new = _step(net, n, e, t, cap, 0, prec)
    old = _step(net, n, e, t, cap, PER_PASS, prec)
    _compare(net, new, old, f"{model} {mode} prec {prec}")
    again = _step(net, n, e, t, cap, 0, prec)
    assert _bits_equal(again["grads"], new["grads"]), "deferred weight gradients differ run to run"


@pytest.mark.parametrize("model", ["GGNN", "MNN"])
def test_small_batch_exact_mode(model):
    """a batch whose per-pass row counts fall below the tensor-core threshold: the deferred members run pass by pass
    on the fp32 SIMT kernel when all passes together are still short, else as one tensor-core launch"""
    C, net, n, e, t = _case(model, 12, seed=3)
    _compare(net, _step(net, n, e, t, None, 0, 0), _step(net, n, e, t, None, PER_PASS, 0), f"{model} B=12")


def _dw_launches(net, n, e, t, debug):
    """(all kernel launches, tensor-core weight-gradient launches) of one eager forward + backward"""
    from graphinvent_b200 import functional as Fn
    L = _lib()
    with _mode(debug, 0):
        net.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        L.gib_profile_enable(1)
        c0 = L.gib_launch_count()
        Fn.kl_loss(net(n, e), t).backward()
        torch.cuda.synchronize()
        c1 = L.gib_launch_count()
        cap = 4096
        ms, work, cls = (ctypes.c_double * cap)(), (ctypes.c_double * cap)(), (ctypes.c_int * cap)()
        k = L.gib_profile_records(ms, work, cls, cap)
        L.gib_profile_enable(0)
    assert 0 < k <= cap
    return c1 - c0, sum(1 for i in range(k) if cls[i] == 1)


@pytest.mark.parametrize("model", ["GGNN", "MNN"])
def test_launch_count(model):
    """one weight-gradient launch and one reduction per backward for the pass-shared weights instead of two of each per
    pass: 2 T - 1 fewer of each"""
    C, net, n, e, t = _case(model, 300)
    T = C.message_passes
    _dw_launches(net, n, e, t, 0)             # the first call packs the weights
    all_new, dw_new = _dw_launches(net, n, e, t, 0)
    all_old, dw_old = _dw_launches(net, n, e, t, PER_PASS)
    assert dw_old - dw_new == 2 * T - 1, (dw_old, dw_new)
    assert all_old - all_new == 2 * (2 * T - 1), (all_old, all_new)
