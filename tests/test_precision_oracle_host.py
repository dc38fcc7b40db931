"""CPU: the oracle's operand-rounding mode (oracle/mpnn_oracle.py OPERANDS), the yardstick of
tests/test_gpu_precision_dims.py.

1. Unset, the oracle runs its plain ops: outputs and gradients bit for bit, before and after a rounded run.
2. One Linear per mode: the forward, dX and dW are fp64 products of the rounded operands exactly; db is the unrounded
   sum.  The operands are chosen so that every product and every sum is exact in fp64 whatever the summation order
   (short significands in a narrow exponent range), so "exactly" is a bit-for-bit comparison.
3. Rounding edges: TF32 ties go away from zero, fp16 ties to even, an fp16 operand of 7e4 becomes inf.
4. At default dims the bf16 / fp16 mode error is of the order of the oracle's own error under torch.autocast("cpu").
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from tests.conftest import MODELS, load_small

MODES = ("tf32", "bf16", "fp16")
DTYPE16 = {"bf16": torch.bfloat16, "fp16": torch.float16}


@contextlib.contextmanager
def operands(mode):
    from oracle import mpnn_oracle as O
    prev = O.OPERANDS
    O.OPERANDS = mode
    try:
        yield
    finally:
        O.OPERANDS = prev


def _round(t, mode):
    """the test's own statement of the package's rounding: TF32 round to nearest, ties away (cvt.rna) on the fp32 bit
    pattern; bf16 / fp16 torch's .to(dtype)"""
    x = t.detach().float()
    if mode == "tf32":
        b = x.contiguous().view(torch.int32)
        return ((b + 0x1000) & -0x2000).view(torch.float32).double()
    return x.to(DTYPE16[mode]).double()


def _run(fx, dtype):
    from oracle import mpnn_oracle as O
    loss, out, g = O.train_step_grads(fx["sd"], fx["C"], fx["nodes"], fx["edges"], fx["target"], dtype=dtype)
    return [loss, out] + list(g.values())


def _bits_equal(a, b):
    return len(a) == len(b) and all(x.dtype == y.dtype and torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("model", MODELS)
def test_unset_hook_gives_the_plain_oracle_bit_for_bit(model, monkeypatch):
    from oracle import mpnn_oracle as O
    fx = load_small(model)
    assert O.OPERANDS is None
    for dtype in (None, torch.float64):
        got = _run(fx, dtype)
        with operands("bf16"):
            rounded = _run(fx, dtype)
        again = _run(fx, dtype)
        with monkeypatch.context() as m:         # the oracle as written before the hook: plain F.linear / matmul
            m.setattr(O, "linear", F.linear)
            m.setattr(O, "matmul", torch.matmul)
            plain = _run(fx, dtype)
        assert _bits_equal(got, plain) and _bits_equal(again, plain), (model, dtype)
        assert not torch.equal(rounded[1], plain[1]), (model, dtype)


def _exact_case(seed):
    """x, W with 17-bit significands (multiples of 2^-14, |.| <= 4), G with 24-bit ones (multiples of 2^-22, |.| < 2):
    every product of rounded operands is a multiple of 2^-36 below 2^3 and a sum of 37 of them needs < 45 bits, so fp64
    evaluates each of them exactly; x and W are exact in fp32, G too (the package's G is fp32)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-2 ** 16, 2 ** 16, (33, 37), generator=g).double() / 2 ** 14
    w = torch.randint(-2 ** 16, 2 ** 16, (29, 37), generator=g).double() / 2 ** 14
    b = torch.randn(29, generator=g, dtype=torch.float64)
    G = torch.randint(-2 ** 23, 2 ** 23, (33, 29), generator=g).double() / 2 ** 22
    return x, w, b, G


@pytest.mark.parametrize("mode", MODES)
def test_one_linear_rounds_its_operands_forward_and_backward(mode):
    from oracle import mpnn_oracle as O
    x, w, b, G = _exact_case(MODES.index(mode))
    x, w, b = (t.clone().requires_grad_(True) for t in (x, w, b))
    with operands(mode):
        y = O.linear(x, w, b)
        y.backward(G)
    rx, rw, rG = _round(x, mode), _round(w, mode), _round(G, mode)
    assert torch.equal(y.detach(), rx @ rw.t() + b.detach())
    assert torch.equal(x.grad, rG @ rw)
    assert torch.equal(w.grad, rG.t() @ rx)
    assert torch.equal(b.grad, G.sum(0))
    # the case is not vacuous: every operand loses bits in this mode
    for t, r in ((x, rx), (w, rw), (G, rG)):
        assert not torch.equal(t.detach(), r), mode
    assert not torch.equal(y.detach(), x.detach() @ w.detach().t() + b.detach())
    assert not torch.equal(x.grad, G @ w.detach()) and not torch.equal(w.grad, G.t() @ x.detach())
    assert not torch.equal(b.grad, rG.sum(0))


@pytest.mark.parametrize("mode", MODES)
def test_batched_message_product_rounds_its_operands(mode):
    """the MNN message product per_edge @ nghb_rows, [E, M, H] @ [E, H, 1]"""
    from oracle import mpnn_oracle as O
    g = torch.Generator().manual_seed(7)
    a = (torch.randint(-2 ** 16, 2 ** 16, (5, 6, 7), generator=g).double() / 2 ** 14).requires_grad_(True)
    v = (torch.randint(-2 ** 16, 2 ** 16, (5, 7, 1), generator=g).double() / 2 ** 14).requires_grad_(True)
    G = torch.randint(-2 ** 23, 2 ** 23, (5, 6, 1), generator=g).double() / 2 ** 22
    with operands(mode):
        y = O.matmul(a, v)
        y.backward(G)
    ra, rv, rG = _round(a, mode), _round(v, mode), _round(G, mode)
    assert torch.equal(y.detach(), ra @ rv)
    assert torch.equal(a.grad, rG @ rv.transpose(1, 2))
    assert torch.equal(v.grad, ra.transpose(1, 2) @ rG)


def test_rounding_edges():
    from oracle import mpnn_oracle as O
    tie = torch.tensor([1 + 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 3 * 2.0 ** -11], dtype=torch.float64)
    assert O.round_operand(tie, "tf32").tolist() == [1 + 2.0 ** -10, -(1 + 2.0 ** -10), 1 + 2 * 2.0 ** -10]   # away
    assert O.round_operand(tie, "fp16").tolist() == [1.0, -1.0, 1 + 2 * 2.0 ** -10]                          # even
    big = torch.tensor([7e4, -7e4, 65504.0, 3.0e38], dtype=torch.float64)
    assert O.round_operand(big, "fp16").tolist() == [float("inf"), float("-inf"), 65504.0, float("inf")]
    assert O.round_operand(big, "bf16")[:2].abs().min().item() == 70144.0          # bf16 keeps the range
    # through a Linear: an fp16 input of 7e4 makes its output row infinite, the other rows stay finite
    x = torch.ones(3, 4, dtype=torch.float64)
    x[1, 2] = 7e4
    with operands("fp16"):
        y = O.linear(x, torch.full((2, 4), 0.5, dtype=torch.float64), torch.zeros(2, dtype=torch.float64))
    assert torch.isinf(y[1]).all() and torch.isfinite(y[[0, 2]]).all()


@pytest.mark.parametrize("model", MODELS)
def test_16bit_mode_error_is_of_the_order_of_the_oracle_under_cpu_autocast(model):
    """at default dims (tests/test_gpu_tf32.py::_oracle, 101 molecules): |o_mode - o64| against the oracle's fp32
    restatement run under torch.autocast("cpu").  Autocast also keeps the Linear outputs in 16 bits, the package keeps
    its activations in fp32, so the mode error may be the smaller one"""
    import tests.test_gpu_tf32 as T
    from oracle import mpnn_oracle as O
    from tests.test_gpu_autocast import _oracle_autocast_error
    C, sd, nodes, edges, target, o64, _, _ = T._oracle(model)
    for dt, dtype in DTYPE16.items():
        with operands(dt):
            _, o, _ = O.train_step_grads(sd, C, nodes, edges, target, dtype=torch.float64)
        mode_err = (o - o64).abs().max().item()
        ref_err = _oracle_autocast_error(model, dtype)
        print(f"{model} {dt}: mode error {mode_err:.3e}, oracle under CPU autocast {ref_err:.3e} "
              f"(ratio {mode_err / ref_err:.3f})")
        # measured: 0.68 - 0.89 of the autocast error over the four models and both dtypes
        assert ref_err / 4 <= mode_err <= 1.5 * ref_err, (model, dt, mode_err, ref_err)
