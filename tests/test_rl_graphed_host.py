"""The captured RL rollout (graphinvent_b200.graphed.GraphedGeneratorRL) on CPU: its C-ABI symbols and argument
checks, the rollout-record arithmetic, and the autograd bookkeeping of `_RolloutLikelihoods` (which model gets a
backward, the in-place check) with the device work played by a numpy restatement of the owner map."""
import types

import numpy as np
import pytest
import torch

RL_SYMBOLS = ("gib_rl_sample_round", "gib_rl_snapshot", "gib_rl_restore", "gib_rl_gather", "gib_rl_scatter_grad",
              "gib_rl_dlogits", "gib_rl_next_round")


def test_rl_symbols_are_exported_and_bound():
    from graphinvent_b200 import _lib
    for name in RL_SYMBOLS:
        assert name in _lib.exported_symbols(), name
        assert getattr(_lib.lib, name).restype is not None, name


def test_rl_entry_points_refuse_bad_arguments_before_any_launch():
    """every refusal is a -1 with a message, decided on the host: the null device pointers are never touched"""
    from graphinvent_b200._lib import lib
    N, A, CH, Ef = 13, 5, 3, 3
    apd = N * (A * CH * Ef + Ef) + 1

    def sample_round(B=8, apd=apd, la=1, lb=1, u=1, acts=None, rec=1):
        v = lambda x: None if x is None else x                         # noqa: E731  (fake non-null host values)
        return lib.gib_rl_sample_round(B, N, A + CH, Ef, A, CH, 0, 0, v(la), v(lb), apd, v(u), acts, None, v(rec),
                                       v(rec), v(rec), *([None] * 11), 16, None, None, None)
    for kw in (dict(apd=apd + 1), dict(B=0), dict(B=1 << 24), dict(la=None), dict(lb=None), dict(u=None),
               dict(rec=None)):
        assert sample_round(**kw) == -1, kw
        assert b"gib_rl_sample_round" in lib.gib_last_error() or b"gib_generation_round" in lib.gib_last_error()
    assert lib.gib_rl_snapshot(8, 0, 8, 3, 0, *([None] * 9)) == -1
    assert lib.gib_rl_snapshot(8, 13, 8, 3, 0, *([None] * 9)) == -1
    assert lib.gib_rl_restore(8, 13, 8, 3, *([None] * 6)) == -1
    assert lib.gib_rl_gather(0, 16, 26, *([None] * 6)) == -1
    assert lib.gib_rl_scatter_grad(8, 16, 26, None, None, None, None, None, None) == -1
    assert lib.gib_rl_scatter_grad(8, 16, 26, 1, 1, None, None, None, None) == -1      # d_a without dp_a
    assert lib.gib_rl_dlogits(0, 625, *([None] * 7)) == -1
    assert lib.gib_rl_dlogits(8, 625, None, 1, 1, None, 1, None, None) == -1
    assert lib.gib_rl_next_round(None, None) == -1
    assert b"gib_rl_next_round" in lib.gib_last_error()


def test_rollout_record_arithmetic():
    from graphinvent_b200.graphed import rl_record_bytes
    # reference defaults (gdb13: 5 atom types + 3 charges, 3 bond types, 13 atoms): 2N * B * (N*F + N^2*Ef) bytes of
    # int8 snapshots = 15.9 MB, plus 12 bytes per (round, slot) and the fp32 owner map [2B, 2N]
    B, N, F, Ef = 1000, 13, 8, 3
    snap = 2 * N * B * (N * F + N * N * Ef)
    assert snap == 15_886_000
    assert rl_record_bytes(B, N, F, Ef) == snap + 2 * N * B * 12 + 2 * B * 2 * N * 4 == 16_406_000
    assert rl_record_bytes(1, 1, 1, 1) == 2 * (1 + 1 + 12) + 2 * 2 * 4
    # linear in the batch, one record per waiting rollout
    assert rl_record_bytes(2 * B, N, F, Ef) == 2 * rl_record_bytes(B, N, F, Ef)


class _FakeGen:
    """stands in for GraphedGeneratorRL: the owner-map gather / inversion in numpy, and one "model" per slot whose
    probability of every (round, slot) is a fixed linear function of its parameters, p[r, b] = w . x[r, b]"""

    def __init__(self, rec, x):
        self.rec, self.x, self.calls = rec, x, []
        self.batch_size = rec.p_a.shape[1]

    def _gather(self, rec):
        owner = rec.owner.numpy().astype(int)
        out = []
        for p in (rec.p_a, rec.p_b):
            o = np.zeros(owner.shape, np.float32)
            g, t = np.nonzero(owner)
            o[g, t] = p.numpy()[t, owner[g, t] - 1]
            out.append(torch.from_numpy(o))
        return tuple(out)

    def _backward(self, rec, d_a, d_b, pa, pb):
        self.calls.append((pa is not None, pb is not None))
        owner = rec.owner.numpy().astype(int)
        g, t = np.nonzero(owner)
        out = []
        for d, ps in ((d_a, pa), (d_b, pb)):
            if ps is None:
                out.append(None)
                continue
            dp = np.zeros(rec.p_a.shape, np.float32)
            dp[t, owner[g, t] - 1] = d.numpy()[g, t]
            out.append([torch.from_numpy(np.einsum("rb,rbk->k", dp, self.x).astype(np.float32))])
        return out


def _fake(seed=0, B=6, R=4):
    rng = np.random.default_rng(seed)
    x = rng.random((R, B, 3)).astype(np.float32)
    wa, wb = (torch.nn.Parameter(torch.from_numpy(rng.random(3).astype(np.float32))) for _ in range(2))
    owner = np.zeros((2 * B, 2 * R), np.float32)
    for r in range(R):
        slots = rng.permutation(np.arange(1, B))[:3]
        owner[rng.choice(2 * B, 3, replace=False), r] = slots + 1
    with torch.no_grad():
        pa = torch.einsum("rbk,k->rb", torch.from_numpy(x), wa)
        pb = torch.einsum("rbk,k->rb", torch.from_numpy(x), wb)
    rec = types.SimpleNamespace(owner=torch.from_numpy(owner), p_a=pa, p_b=pb, rounds=R)
    return _FakeGen(rec, x), rec, wa, wb, torch.from_numpy(x), torch.from_numpy(owner)


def _explicit(x, owner, w):
    """per-(molecule, round) bookkeeping: table[g, t] = w . x[t, owner[g, t] - 1]"""
    rows = []
    for g in range(owner.shape[0]):
        row = []
        for t in range(owner.shape[1]):
            s = int(owner[g, t])
            row.append(x[t, s - 1] @ w if s else torch.zeros(()))
        rows.append(torch.stack(row))
    return torch.stack(rows)


def test_rollout_function_routes_gradients_like_explicit_bookkeeping():
    from graphinvent_b200.graphed import _RolloutLikelihoods
    gen, rec, wa, wb, x, owner = _fake()
    la, lb = _RolloutLikelihoods.apply(gen, rec, 1, wa, wb)
    ea, eb = _explicit(x, owner, wa), _explicit(x, owner, wb)
    assert torch.allclose(la, ea.detach()) and torch.allclose(lb, eb.detach())
    B = gen.batch_size
    loss = torch.log(la.sum(1)[:B] + 1).sum() + 2 * lb.sum()
    loss.backward()
    ga, gb = wa.grad.clone(), wb.grad.clone()
    wa.grad = wb.grad = None
    (torch.log(ea.sum(1)[:B] + 1).sum() + 2 * eb.sum()).backward()
    assert torch.allclose(ga, wa.grad, rtol=1e-5) and torch.allclose(gb, wb.grad, rtol=1e-5)
    assert gen.calls == [(True, True)]


def test_rollout_function_skips_frozen_models_and_sums_shared_ones():
    from graphinvent_b200.graphed import _RolloutLikelihoods
    gen, rec, wa, wb, x, owner = _fake(1)
    wb.requires_grad_(False)
    la, lb = _RolloutLikelihoods.apply(gen, rec, 1, wa, wb)
    (la.sum() + lb.sum()).backward()
    assert gen.calls == [(True, False)] and wb.grad is None and wa.grad is not None
    # the same model as agent and prior (one parameter twice): autograd sums both streams
    gen2, rec2, wa2, _, x2, owner2 = _fake(2)
    rec2.p_b = rec2.p_a.clone()
    la, lb = _RolloutLikelihoods.apply(gen2, rec2, 1, wa2, wa2)
    (la.sum() + 3 * lb.sum()).backward()
    want = 4 * sum(x2[t, int(owner2[g, t]) - 1] for g, t in zip(*np.nonzero(owner2.numpy())))
    assert torch.allclose(wa2.grad, want, rtol=1e-5)


def test_rollout_function_refuses_parameters_changed_before_its_backward():
    from graphinvent_b200.graphed import _RolloutLikelihoods
    gen, rec, wa, wb, _, _ = _fake(3)
    la, lb = _RolloutLikelihoods.apply(gen, rec, 1, wa, wb)
    with torch.no_grad():
        wb.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (la.sum() + lb.sum()).backward()
    assert gen.calls == []
    gen, rec, wa, wb, _, _ = _fake(4)
    la, lb = _RolloutLikelihoods.apply(gen, rec, 1, wa, wb)
    wa.data = wa.data.clone()                          # a new storage (e.g. an optimizer re-flattening the weights)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (la.sum() + lb.sum()).backward()
