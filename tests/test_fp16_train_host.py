"""CPU: the dynamic-loss-scaling pieces of the captured training step that need no GPU -- the new C-ABI entry points
and their argument refusals, `TrainStep(grad_scaler=)`'s refusals, a disabled scaler meaning no scaler, and the matmul
precision a TrainStep picks with and without a scaler under each autocast / TF32 state."""
import ctypes

import pytest
import torch

from tests.test_autocast_host import autocast_state

NEW = ("gib_kl_loss_fwd_bwd_ctl_scaled", "gib_nonfinite_check", "gib_adam_step_scaled", "gib_amp_update_scale")


def _host_ptr():
    buf = ctypes.create_string_buffer(256)       # never dereferenced: every call below returns before a launch
    return buf, ctypes.c_void_p(ctypes.addressof(buf))


def _enabled_scaler(monkeypatch, **kw):
    """a GradScaler("cuda") as it is built on a CUDA machine (torch disables it when no CUDA device is present)"""
    monkeypatch.setattr(torch.cuda.amp.common, "amp_definitely_not_available", lambda: False)
    s = torch.amp.GradScaler("cuda", **kw)
    assert s.is_enabled()
    return s


def test_new_symbols_are_declared_and_bound():
    from graphinvent_b200 import _lib
    for name in NEW:
        assert name in _lib.exported_symbols()
        assert callable(getattr(_lib.lib, name))
    assert _lib.lib.gib_version() == 206


def test_argument_refusals():
    from graphinvent_b200._lib import lib
    keep, p = _host_ptr()
    # non-finite check: n < 0, null flag, null data with n > 0; n == 0 is a no-op
    assert lib.gib_nonfinite_check(p, -1, p, None) < 0 and b"n >= 0" in lib.gib_last_error()
    assert lib.gib_nonfinite_check(p, 4, None, None) < 0 and b"null" in lib.gib_last_error()
    assert lib.gib_nonfinite_check(None, 4, p, None) < 0 and b"null" in lib.gib_last_error()
    assert lib.gib_nonfinite_check(None, 0, p, None) == 0
    # gated Adam: n < 0, each device scalar null, a null buffer with n > 0, misaligned buffers; n == 0 is a no-op
    args = [p, p, p, p, 8, p, p, p, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0, None]
    assert lib.gib_adam_step_scaled(*args[:4], -1, *args[5:]) < 0 and b"n >= 0" in lib.gib_last_error()
    for k in (5, 6, 7):
        a = list(args)
        a[k] = None
        assert lib.gib_adam_step_scaled(*a) < 0 and b"null device scalar" in lib.gib_last_error(), k
    for k in range(4):
        a = list(args)
        a[k] = None
        assert lib.gib_adam_step_scaled(*a) < 0 and b"null buffer" in lib.gib_last_error(), k
    a = list(args)
    a[1] = ctypes.c_void_p(p.value + 4)
    assert lib.gib_adam_step_scaled(*a) < 0 and b"alignment" in lib.gib_last_error()
    assert lib.gib_adam_step_scaled(*args[:4], 0, *args[5:]) == 0
    # scale update: each pointer null, n_counts < 0, growth_interval < 1
    args = [p, p, p, 2.0, 0.5, 3, p, 2, None]
    for k in (0, 1, 2, 6):
        a = list(args)
        a[k] = None
        assert lib.gib_amp_update_scale(*a) < 0 and b"null" in lib.gib_last_error(), k
    a = list(args)
    a[7] = -1
    assert lib.gib_amp_update_scale(*a) < 0 and b"n_counts" in lib.gib_last_error()
    a = list(args)
    a[5] = 0
    assert lib.gib_amp_update_scale(*a) < 0 and b"growth_interval" in lib.gib_last_error()
    # scaled loss: null ctl, null scale; an empty batch is a no-op
    assert lib.gib_kl_loss_fwd_bwd_ctl_scaled(p, p, 4, 8, None, p, p, p, None) < 0
    assert lib.gib_kl_loss_fwd_bwd_ctl_scaled(p, p, 4, 8, p, None, p, p, None) < 0
    assert b"loss_scale" in lib.gib_last_error()
    assert lib.gib_kl_loss_fwd_bwd_ctl_scaled(p, p, 0, 8, p, p, p, p, None) == 0
    del keep


def _net():
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    return mpnn.create(O.make_constants("GGNN"))


def test_train_step_refuses_what_it_cannot_scale(monkeypatch):
    from graphinvent_b200.graphed import TrainStep
    net = _net()
    scaler = _enabled_scaler(monkeypatch)
    sgd = torch.optim.SGD(net.parameters(), lr=0.1)
    with pytest.raises(ValueError, match="FlatAdam"):
        TrainStep(net, sgd, batch_size=4, entry_capacity=64, grad_scaler=scaler)
    for bad in (object(), 2.0 ** 16, torch.ones(())):
        with pytest.raises(TypeError, match="GradScaler"):
            TrainStep(net, sgd, batch_size=4, entry_capacity=64, grad_scaler=bad)
    cpu = torch.amp.GradScaler("cpu")
    with pytest.raises(ValueError, match="CUDA GradScaler"):
        TrainStep(net, sgd, batch_size=4, entry_capacity=64, grad_scaler=cpu)


def test_train_step_refuses_a_scaler_without_the_device_state(monkeypatch):
    from graphinvent_b200.graphed import _grad_scaler
    from graphinvent_b200.optim import FlatAdam
    scaler = _enabled_scaler(monkeypatch)
    del scaler._growth_tracker
    with pytest.raises(RuntimeError, match="_growth_tracker"):
        _grad_scaler(scaler, object.__new__(FlatAdam))     # a FlatAdam needs CUDA parameters: only its type matters


def test_a_disabled_scaler_is_no_scaler():
    from graphinvent_b200.graphed import TrainStep, _grad_scaler
    off = torch.amp.GradScaler("cuda", enabled=False)
    assert _grad_scaler(off, torch.optim.SGD(_net().parameters(), lr=0.1)) is None     # no FlatAdam needed either
    assert _grad_scaler(None, None) is None
    with autocast_state(True, torch.float16):
        assert TrainStep.precision_code(off) == TrainStep.precision_code(None) == 0
    # without CUDA the constructor then stops where a scaler-less one does: at the CPU parameters
    with pytest.raises(RuntimeError, match="CUDA"):
        TrainStep(_net(), torch.optim.SGD(_net().parameters(), lr=0.1), batch_size=4, entry_capacity=64,
                  grad_scaler=off)


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("dtype", [None, torch.bfloat16, torch.float16, torch.float32])
def test_precision_with_and_without_a_scaler(dtype, tf32, monkeypatch):
    from graphinvent_b200.graphed import TrainStep
    scaler = _enabled_scaler(monkeypatch)
    with autocast_state(dtype is not None, dtype or torch.float16, tf32):
        without, with_ = TrainStep.precision_code(None), TrainStep.precision_code(scaler)
    fp32_input = int(tf32)
    assert with_ == {torch.bfloat16: 2, torch.float16: 3}.get(dtype, fp32_input)
    assert without == {torch.bfloat16: 2}.get(dtype, fp32_input)     # fp16 only with a scaler
