"""GPU: the even k-block split of the grouped tensor-core weight-gradient launch (csrc/gemm_tc3.cu: dw_plan) against
float64 with test_gpu_gemm_patterns' bound: segments that cross tile and member boundaries, 1-tile and 16-tile
members in one launch, device-side row counts of 0 / 1 / 33 / the capacity with NaN rows past the live count, and
two launches of the same group that must agree bit for bit (the reduction sums each tile's partials in a fixed order)."""
import pytest
import torch

from tests.test_gpu_gemm_patterns import (DW, TC_DW, _dev_int, _lib, _operands, _path, _run_dw,
                                          _shared_buffer_group)

pytestmark = pytest.mark.gpu


def _ok(rc, cls, n=1):
    assert rc == 0, _lib().lib.gib_last_error().decode()
    assert cls == [TC_DW] * n, cls


def _mixed_group(rows, seed):
    """a 1-tile member (128 x 128), a 16-tile one (512 x 512), a ragged one and a narrow one"""
    shapes = [(128, 128), (512, 512), (100, 136), (48, 600)]
    grp = []
    for k, ((R, C), M) in enumerate(zip(shapes, rows)):
        G, X = _operands(M, -(-R // 16) * 16, -(-C // 16) * 16, R, C, seed=seed + k)
        dW = torch.randn(R, C, device="cuda")
        db = torch.randn(R, device="cuda") if k != 2 else None
        grp.append(DW(G, X, M, dW, R, C, dbias=db))
    return grp


@pytest.mark.parametrize("rows", [(4097, 33, 2048, 3000), (40000, 2049, 1, 700), (257, 9000, 31, 4096)])
def test_dw_mixed_tiles_across_boundaries(rows):
    """ragged row counts put segment ends inside tiles and ranges across member boundaries"""
    grp = _mixed_group(rows, seed=sum(rows))
    rc, cls, check, _ = _run_dw([grp])
    _ok(rc, cls)
    check(_path(cls), f"mixed tiles rows={rows}")


@pytest.mark.parametrize("live", [0, 1, 33, "cap"])
def test_dw_device_rows_nan_past_live(live):
    """device-side counts inside a capacity of 4224 rows; rows past each live range are NaN / Inf"""
    cap = 4224
    m = cap - 2048 if live == "cap" else live
    grp = _shared_buffer_group(cap, 128, 512, 128, 500, [(0, 2048), (2048, m)], seed=7 + (m or 0))
    rc, cls, check, _ = _run_dw([grp])
    _ok(rc, cls)
    check("tc", f"device rows live={live}")


def test_dw_two_launches_bit_identical():
    """the same group twice (host counts) and once more on device-side counts: the same bits in dW and dbias"""
    rows = (13312, 4097, 33, 2048)
    outs = []
    for dev in (False, False, True):
        grp = _mixed_group(rows, seed=11)
        for q in grp:
            q.dW.zero_()
            if q.dbias is not None:
                q.dbias.zero_()
            if dev:
                q.rows = (_dev_int(q.M), _dev_int(0), 0, q.M)
        rc, cls, _, _ = _run_dw([grp])
        _ok(rc, cls)
        torch.cuda.synchronize()
        outs.append([t.clone() for q in grp for t in (q.dW, q.dbias) if t is not None])
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not any(torch.isnan(t).any().item() for t in outs[0])
