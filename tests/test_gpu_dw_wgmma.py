"""GPU: edges of the weight-gradient kernel (csrc/gemm_tc3.cu: tc3_wgmma_dw_kernel) that the sweep of
tests/test_gpu_gemm_patterns.py does not reach, against float64 with the same bound and kernel-class check:
128 x 128 output tiles with a ragged last column tile, several row tiles whose bias partials come from the first
column tile only, last reduction chunks that end 1 or 31 rows into a k-block, and NaN rows past a device-side live
count, which the consumers (G) and the in-kernel transpose (X) must both turn into zeros."""
import pytest
import torch

from tests.test_gpu_gemm_patterns import (DW, NAN, TC_DW, _dev_int, _dw_expect, _lib, _operands, _path, _run_dw,
                                          pad16)

pytestmark = pytest.mark.gpu

MODES = [(1, 0), (1, 1)]   # the grouped launch, and the per-problem one (gib_tc_debug bit 0)


def _check(groups, tc, debug, what, plan_rows=0):
    rc, cls, check, _ = _run_dw(groups, plan_rows=plan_rows, tc=tc, debug=debug)
    assert rc == 0, _lib().lib.gib_last_error().decode()
    assert cls == _dw_expect(groups, tc, debug), f"{what}: kernel classes {cls}"
    assert TC_DW in cls, f"{what}: no tensor-core weight-gradient launch"
    check(_path(cls), what)


@pytest.mark.parametrize("M", [2049, 4127])        # every chunk but the last is a multiple of 32: M % 32 = 1, 31
@pytest.mark.parametrize("C", [140, 600])          # Kk = 144 (128 + 16), 608 (4 x 128 + 96)
@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_ragged_tiles_and_chunk_tails(M, C, tc, debug):
    R = 100                                        # Nn = 112: one row tile, 16 rows of it past Nn
    G, X = _operands(M, pad16(R), pad16(C), R, C, seed=M + C)
    dW = torch.randn(R, C, device="cuda")
    db = torch.randn(R, device="cuda")
    _check([[DW(G, X, M, dW, R, C, dbias=db)]], tc, debug, f"M={M} Kk={pad16(C)}")


@pytest.mark.parametrize("M", [3073, 4095])
@pytest.mark.parametrize("tc,debug", MODES)
def test_dw_gate_blocked_three_row_tiles(M, tc, debug):
    """GRU weights with H = 120: Nn = 3 x 128, five column tiles (Kk = 608); the bias partials of each row tile come
    from its first column tile"""
    H, C = 120, 600
    Hp = pad16(H) + 8                              # gate blocks 128 columns apart
    G, X = _operands(M, 3 * Hp, pad16(C), 3 * Hp, C, seed=M + 7)
    for g in range(3):
        G[:, g * Hp + H:(g + 1) * Hp] = 0
    dW = torch.randn(3 * H, C, device="cuda")
    db = torch.randn(3 * H, device="cuda")
    _check([[DW(G, X, M, dW, 3 * H, C, dbias=db, Rb=H, Rbp=Hp)]], tc, debug, f"gate-blocked Nn=384 M={M}")


@pytest.mark.parametrize("R,C", [(100, 136), (120, 600)])
def test_dw_nan_rows_past_the_live_count(R, C):
    """capacity mode: G and X are NaN in every row outside the live ranges; the ranges end 1 and 31 rows into a
    k-block, so the last stage of each holds NaN rows that must not reach dW or db"""
    cap, Nn, Kk = 8192, pad16(R), pad16(C)
    torch.manual_seed(R + C)
    G = torch.full((cap, Nn), NAN, device="cuda")
    X = torch.full((cap, Kk), NAN, device="cuda")
    grp = []
    for base, m in ((0, 2081), (4096, 3999)):
        G[base:base + m] = 0
        G[base:base + m, :R] = torch.randn(m, R, device="cuda")
        X[base:base + m] = 0
        X[base:base + m, :C] = torch.randn(m, C, device="cuda")
        dW = torch.randn(R, C, device="cuda")
        db = torch.randn(R, device="cuda")
        grp.append(DW(G, X, cap, dW, R, C, dbias=db, rows=(_dev_int(m), _dev_int(base), base, base + m)))
    _check([grp], 1, 0, f"NaN past the live count Nn={Nn} Kk={Kk}", plan_rows=cap)
