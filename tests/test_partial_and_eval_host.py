"""Partial batches and the captured validation pass on CPU: the C-ABI symbols, struct mirrors and argument refusals,
the batch-size refusal of TrainStep / EvalStep, and the reference restatements the GPU tests compare against
(tests/test_gpu_partial_and_eval.py) on hand-computed cases with the reference's quirks."""
import ctypes
import math
import types

import pytest
import torch

SYMBOLS = ("gib_kl_loss_fwd_bwd_ctl", "gib_sum_scaled_ctl", "gib_validation_nll_ctl", "gib_eval_collect")


def test_ctl_symbols_are_exported_and_bound():
    from graphinvent_b200 import _lib
    for name in SYMBOLS:
        assert name in _lib.exported_symbols(), name
        assert getattr(_lib.lib, name).restype is not None, name


def test_struct_mirrors_match_the_header_layout():
    from graphinvent_b200._lib import BatchCtl, EvalPass
    assert ctypes.sizeof(BatchCtl) == 8 and BatchCtl.scale.offset == 4
    assert ctypes.sizeof(EvalPass) == 48
    assert [getattr(EvalPass, f).offset for f in ("lik", "lik_len", "n_slots", "idx", "n_structures", "flags",
                                                  "clipped")] == [8, 16, 24, 28, 32, 36, 40]


def test_ctl_entry_points_refuse_null_arguments_before_any_launch():
    from graphinvent_b200._lib import lib
    assert lib.gib_kl_loss_fwd_bwd_ctl(1, 1, 4, 85, None, 1, None, None) == -1
    assert b"gib_kl_loss_fwd_bwd_ctl" in lib.gib_last_error()
    assert lib.gib_sum_scaled_ctl(1, 4, None, 1, None) == -1
    assert lib.gib_validation_nll_ctl(1, 1, 4, 85, None, 1, None) == -1
    ok = dict(kl=1, nll=1, t=1, B=4, apd=85, ctl=1, cws=1, p=1)
    for bad in (dict(B=0), dict(apd=0), dict(kl=None), dict(nll=None), dict(t=None), dict(ctl=None), dict(cws=None),
                dict(p=None)):
        a = {**ok, **bad}
        assert lib.gib_eval_collect(a["kl"], a["nll"], a["t"], a["B"], a["apd"], a["ctl"], a["cws"], a["p"], None) == -1
        assert b"gib_eval_collect" in lib.gib_last_error()


def test_batches_larger_than_the_static_buffers_are_refused():
    from graphinvent_b200.graphed import _batch_rows
    step = types.SimpleNamespace(B=4)
    n, e, t = torch.zeros(5, 3, 2), torch.zeros(5, 3, 3, 1), torch.zeros(5, 7)
    with pytest.raises(ValueError, match="up to 4 molecules, got 5"):
        _batch_rows(step, "TrainStep", n, e, t)
    with pytest.raises(ValueError, match="hold 3, 5 and 5"):
        _batch_rows(step, "EvalStep", n[:3], e, t)
    assert _batch_rows(step, "TrainStep", n[:0], e[:0], t[:0]) == 0
    assert _batch_rows(step, "TrainStep", n[:4], e[:4], t[:4]) == 4


# ---- the reference's list logic, restated on per-row values (the GPU tests take them from the kernels) ----------
def validation_likelihood(batches, n_samples, batch_size, N):
    """Analyzer.py:734-778 with the per-batch NLL rows given: batches = [(nll_rows, target_last_column)]"""
    n = min(100000, n_samples)
    lik = torch.zeros(n * (N + 5))
    n_structures = torch.zeros(1)
    for idx, (v, last) in enumerate(batches):
        if idx * batch_size > n:
            break
        v = v[~torch.isnan(v)]
        lik[idx * batch_size: idx * batch_size + len(v)] = v
        n_structures += torch.sum(last).unsqueeze(dim=0)
    return lik, torch.sum(lik, dim=0) / n_structures[0]


def validation_epoch(batch_losses, n_slots):
    """Workflow.py:813-831 with each batch's KLDivLoss(batchmean) given"""
    t = torch.zeros(n_slots)
    for i, x in enumerate(batch_losses):
        t[i] = x
    return torch.mean(t)


def test_validation_likelihood_restatement_by_hand():
    nan = float("nan")
    b0 = (torch.tensor([nan, 1.0, 2.0, nan]), torch.tensor([1.0, 0.0, 1.0, 1.0]))
    b1 = (torch.tensor([nan, nan, nan, nan]), torch.tensor([0.0, 0.0, 0.0, 0.0]))      # all NaN: writes nothing
    b2 = (torch.tensor([3.0, nan]), torch.tensor([1.0, 1.0]))                          # short
    b3 = (torch.tensor([5.0, 5.0, 5.0, 5.0]), torch.tensor([1.0, 1.0, 1.0, 1.0]))
    # n_samples = 8, B = 4: idx 2 (2 * 4 = 8) still runs -- the break is `>` -- idx 3 does not
    lik, avg = validation_likelihood([b0, b1, b2, b3], 8, 4, N=1)
    assert lik.tolist() == [1.0, 2.0, 0, 0, 0, 0, 0, 0, 3.0, 0, 0, 0] + [0.0] * 36
    assert math.isclose(float(avg), 6.0 / 5.0, rel_tol=1e-6)
    # n_samples = 7: idx 2 breaks (8 > 7)
    lik, avg = validation_likelihood([b0, b1, b2, b3], 7, 4, N=1)
    assert float(lik.sum()) == 3.0 and math.isclose(float(avg), 3.0 / 3.0, rel_tol=1e-6)
    # a write past the buffer raises in the reference (the captured pass clips, flags, and raises after the pass)
    with pytest.raises(RuntimeError):
        validation_likelihood([b3], 0, 4, N=0)


def test_validation_epoch_restatement_by_hand():
    assert float(validation_epoch([1.0, 3.0], 2)) == 2.0
    assert float(validation_epoch([1.0, 3.0], 4)) == 1.0          # len(loader) > batches yielded: zero slots count
    assert math.isnan(float(validation_epoch([1.0, float("nan")], 3)))   # a NaN row's batch makes the mean NaN
    with pytest.raises(IndexError):
        validation_epoch([1.0, 2.0, 3.0], 2)                     # more batches than slots
