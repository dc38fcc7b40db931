"""CPU: the route-likelihood backward's C-ABI (symbols, argument refusals) and a numpy restatement of its per-state
coefficient, dL/d log p, against torch.autograd through tests/route_nll_reference.reduce."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import route_nll_reference as R
from tests.conftest import GOLDEN

NEW_SYMBOLS = ("gib_route_grad_coef", "gib_route_dlogits")


def coef_restated(p, offsets, g_lik=None, g_nll=None, g_final=None):
    """dL/d log p_s = g_lik[s] p_s - g_nll[m] + g_final[m] p_s / sum_m p, per state of fp32 `p`, as
    gib_route_grad_coef computes it: sum p in fp64 in build order, each coefficient in fp64, rounded once; a missing
    gradient is zero and a zero g_final drops its term"""
    p = np.asarray(p, np.float32)
    out = np.zeros(p.shape, np.float32)
    for m, (a, e) in enumerate(zip(offsets[:-1], offsets[1:])):
        q = p[a:e].astype(np.float64)
        c = np.full(e - a, -float(g_nll[m]) if g_nll is not None else 0.0)
        if g_lik is not None:
            c += np.asarray(g_lik[a:e], np.float64) * q
        gf = float(g_final[m]) if g_final is not None else 0.0
        if gf != 0.0:
            s = 0.0
            for v in q:
                s += v
            c += gf * q / s
        out[a:e] = c.astype(np.float32)
    return out


def test_symbols_are_declared_and_bound():
    from graphinvent_b200 import _lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "gib200.h")).read()
    for name in NEW_SYMBOLS:
        assert getattr(_lib.lib, name).argtypes is not None and f"{name}(" in header


def test_entry_points_refuse_bad_arguments():
    from graphinvent_b200._lib import lib
    p = ctypes.c_void_p(64)
    coef = lambda *a: lib.gib_route_grad_coef(*a, None)
    assert coef(0, p, p, p, p, p, p) < 0 and b"gib_route_grad_coef" in lib.gib_last_error()
    assert coef(-1, p, p, None, None, None, p) < 0 and b"n_molecules" in lib.gib_last_error()
    for args in ((3, None, p, p, p, p, p), (3, p, None, p, p, p, p), (3, p, p, p, p, p, None)):
        assert coef(*args) < 0 and b"gib_route_grad_coef" in lib.gib_last_error()
    dl = lambda *a: lib.gib_route_dlogits(*a, None)
    assert dl(0, 625, p, p, p, p, p) < 0 and b"gib_route_dlogits" in lib.gib_last_error()
    assert dl(4, 0, p, p, p, p, p) < 0 and b"apd=0" in lib.gib_last_error()
    for args in ((4, 625, None, p, p, p, p), (4, 625, p, None, p, p, p), (4, 625, p, p, None, p, p),
                 (4, 625, p, p, p, None, p)):
        assert dl(*args) < 0 and b"must be given" in lib.gib_last_error()


def _random_case(seed):
    """fp32 probabilities of molecules of 1 to 9 states, some exactly 0, some one-state molecules"""
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 10, 40)
    lengths[:4] = 1
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    S, M = int(offsets[-1]), len(lengths)
    p = (rng.random(S) ** 4).astype(np.float32)
    p[rng.random(S) < 0.1] = 0.0
    p[offsets[1]] = 0.0                                   # a one-state molecule with p = 0
    p[offsets[5]:offsets[6]] = 0.0                        # a molecule whose every p is 0 but for its last
    p[offsets[6] - 1] = 0.25
    return p, offsets, rng.standard_normal(S), rng.standard_normal(M), rng.standard_normal(M)


@pytest.mark.parametrize("which", ["lik", "nll", "final", "all"])
def test_coefficient_against_autograd_through_reduce(which):
    """autograd of sum(g_lik * p) + sum(g_nll * nll) + sum(g_final * final) w.r.t. x = log p, in fp64; an fp32 p = 0 is
    taken there as 1e-300, where the coefficient's limit -g_nll (+ g_final on a molecule of p = 0 states only) is
    already reached.  The restatement's one fp32 rounding bounds the difference."""
    p, offsets, g_lik, g_nll, g_final = _random_case(7)
    use = {"lik": (g_lik, None, None), "nll": (None, g_nll, None), "final": (None, None, g_final),
           "all": (g_lik, g_nll, g_final)}[which]
    ok_final = np.array([p[a:e].sum() > 0 for a, e in zip(offsets[:-1], offsets[1:])])
    if use[2] is not None:                   # log(sum p) of an all-zero molecule has no gradient: leave it out
        use = (use[0], use[1], np.where(ok_final, use[2], 0.0))
    x = torch.tensor(np.log(np.where(p > 0, p.astype(np.float64), 1e-300)), requires_grad=True)
    q = torch.exp(x)
    nll, final = R.reduce(q, offsets)
    loss = sum((torch.from_numpy(np.asarray(g)) * t).sum() for g, t in zip(use, (q, nll, final)) if g is not None)
    want, = torch.autograd.grad(loss, x)
    got = coef_restated(p, offsets, *use)
    # the size of the terms: |g_lik| + |g_nll| + |g_final| per state
    scale = np.zeros(len(p))
    for m, (a, e) in enumerate(zip(offsets[:-1], offsets[1:])):
        if use[0] is not None:
            scale[a:e] += np.abs(use[0][a:e])
        scale[a:e] += sum(abs(g[m]) for g in use[1:] if g is not None)
    assert np.all(np.isfinite(got))
    assert np.all(np.abs(got - want.numpy()) <= 2e-7 * scale + 1e-290), np.abs(got - want.numpy()).max()


def test_zero_probabilities_keep_a_finite_coefficient():
    """p = 0 has nll = inf but the coefficient -g_nll (the kernel never divides by p); no gradient, no term"""
    p = np.array([0.0, 0.5, 0.0], np.float32)
    offsets = np.array([0, 1, 3])
    got = coef_restated(p, offsets, g_nll=np.array([2.0, -1.0]))
    assert np.array_equal(got, np.array([-2.0, 1.0, 1.0], np.float32))
    assert np.array_equal(coef_restated(p, offsets), np.zeros(3, np.float32))
    nll, _ = R.reduce(torch.from_numpy(p).double(), offsets)
    assert torch.isinf(nll[0])
