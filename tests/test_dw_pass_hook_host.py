"""CPU: the argument checks of the pass-extent weight-gradient test hook (gib_test_dw_groups_passes /
gib_test_dw_scratch_bytes_passes) and of the operands the fp32 SIMT weight-gradient kernel reads as float4
(gib_linear_bwd_dw).  Every refusal returns -2 with a message naming the argument and comes before any CUDA call: the
pointers below are host addresses that are never dereferenced, and no kernel is launched.  The scratch size query counts
a pass extent as csrc/gemm_tc3.cu: tc3_dw_layout does."""
import ctypes

import pytest

from graphinvent_b200 import _lib

L = _lib.lib
BKF, TILE, SIMT_BK = 32, 128, 16
_BUF = ctypes.create_string_buffer(256)
BASE = (ctypes.addressof(_BUF) + 15) & ~15        # a 16-byte aligned host address, never dereferenced


def cdiv(a, b):
    return -(-a // b)


def _problem(M=4096, Nn=128, Kk=256, G=BASE, X=BASE):
    q = _lib.DwProblem()
    q.G, q.ldg, q.Nn, q.X, q.ldx, q.Kk, q.M = G, Nn, Nn, X, Kk, Kk, M
    q.dW, q.R, q.C, q.Rb, q.Rbp, q.rs, q.cs = BASE, Nn, Kk, Nn, Nn, Kk, 1
    return q


def _extent(passes, pass_g=None, pass_x=None, M=4096, Nn=128, Kk=256):
    M = max(M, 1)      # an empty member still has a stride
    return _lib.DwExtent(passes, M * Nn if pass_g is None else pass_g, M * Kk if pass_x is None else pass_x)


def _arrays(problems, extents, sizes):
    qs = (_lib.DwProblem * len(problems))(*problems)
    ext = None if extents is None else (_lib.DwExtent * len(extents))(*extents)
    return qs, ext, (ctypes.c_int * len(sizes))(*sizes)


def _refused(problems, extents, sizes, names):
    """both hooks refuse before any launch, with a message that names the argument"""
    qs, ext, gs = _arrays(problems, extents, sizes)
    launches = L.gib_launch_count()
    assert L.gib_test_dw_scratch_bytes_passes(qs, ext, gs, len(sizes)) == 0
    rc = L.gib_test_dw_groups_passes(qs, ext, gs, len(sizes), ctypes.c_void_p(BASE), None)
    msg = L.gib_last_error().decode()
    assert rc == -2, (rc, msg)
    assert "gib_test_dw_groups_passes" in msg and all(n in msg for n in names), msg
    assert L.gib_launch_count() == launches


@pytest.mark.parametrize("sizes", [[0], [33], [2, 0], [1, 33], [-1]])
def test_group_sizes_outside_1_to_32(sizes):
    n = max(1, sum(s for s in sizes if s > 0))
    _refused([_problem()] * n, None, sizes, ["group_sizes"])


def test_no_groups():
    _refused([_problem()], None, [], ["n_groups"])


@pytest.mark.parametrize("passes", [0, -3, 17, 64])
def test_pass_counts_outside_1_to_16(passes):
    _refused([_problem(), _problem()], [_extent(1), _extent(passes)], [2], ["problem 1", "passes"])


@pytest.mark.parametrize("field,value", [("pass_g", 0), ("pass_g", -4 * 4096), ("pass_x", 0), ("pass_x", -8)])
def test_pass_strides_that_are_not_positive(field, value):
    e = _extent(3)
    setattr(e, field, value)
    _refused([_problem()], [e], [1], [field])


@pytest.mark.parametrize("field,value", [("pass_g", 128 * 4096 + 2), ("pass_x", 256 * 4096 + 6), ("pass_g", 1)])
def test_pass_strides_that_are_not_multiples_of_4(field, value):
    e = _extent(2)
    setattr(e, field, value)
    _refused([_problem()], [e], [1], [field])


def test_a_stride_is_not_checked_without_a_pass_extent():
    """passes = 1 reads one slice: its strides mean nothing and are not refused (the query then sizes the scratch)"""
    qs, ext, gs = _arrays([_problem()], [_lib.DwExtent(1, -3, 5)], [1])
    assert L.gib_test_dw_scratch_bytes_passes(qs, ext, gs, 1) > 0


@pytest.mark.parametrize("operand", ["G", "X"])
@pytest.mark.parametrize("offset", [4, 8, 12])
def test_unaligned_operand_bases(operand, offset):
    """a base 4, 8 or 12 bytes past a 16-byte boundary: refused in any member of any group, with or without a pass
    extent"""
    bad = _problem(**{operand: BASE + offset})
    _refused([bad], None, [1], [operand, "16-byte"])
    _refused([_problem(), _problem(), bad], [_extent(1), _extent(1), _extent(4)], [1, 2], [operand, "16-byte"])


@pytest.mark.parametrize("operand", ["G", "X"])
def test_linear_bwd_dw_refuses_unaligned_operands_before_any_cuda_call(operand):
    """the fp32 SIMT kernel loads G and X as float4: gib_linear_bwd_dw refuses a base that is not 16-byte aligned
    before it touches the device (on a machine without one, any CUDA call would fail with a CUDA error instead)"""
    g, x = (BASE + 4, BASE) if operand == "G" else (BASE, BASE + 4)
    launches = L.gib_launch_count()
    rc = L.gib_linear_bwd_dw(g, 128, 128, x, 256, 256, 100, BASE, BASE, 100, 200, BASE, None, None, None)
    msg = L.gib_last_error().decode()
    assert rc == -2, (rc, msg)
    assert "gib_linear_bwd_dw" in msg and f"{operand} is not 16-byte aligned" in msg, msg
    assert L.gib_launch_count() == launches


# ---- scratch size ------------------------------------------------------------------------------------------------------
def _layout_floats(members, sms):
    """tc3_dw_layout: one partial tile and one bias partial per slot, slots = min(SMs, ceil(units / 8)) + tiles"""
    tiles = sum(cdiv(nn, TILE) * cdiv(kk, TILE) for _, nn, kk, _ in members)
    units = sum(cdiv(nn, TILE) * cdiv(kk, TILE) * cdiv(max(m, 0), BKF) * p for m, nn, kk, p in members)
    return (min(sms, cdiv(units, 8)) + tiles) * (TILE * TILE + TILE)


def _r64(f):
    return (f + 63) // 64 * 64


def _simt_half(m, nn, kk, sms):
    """gemm_dw_half_floats: the split-K partials of one pass of one member, or its one-pass tensor-core layout"""
    s = min(cdiv(2 * sms, cdiv(nn, TILE) * cdiv(kk, TILE)), max(cdiv(m, 64), 1))
    s = max(s, 1)
    c = max(cdiv(cdiv(m, s), SIMT_BK) * SIMT_BK, SIMT_BK)
    s = max(cdiv(m, c), 1)
    return max(_r64(s * nn * kk + s * nn), _r64(_layout_floats([(m, nn, kk, 1)], sms)))


def _expected_bytes(groups, sms):
    half = max(max(max(_simt_half(m, nn, kk, sms) for m, nn, kk, _ in g), _r64(_layout_floats(g, sms)))
               for g in groups)
    return 4 * 2 * half


def _query(groups):
    flat = [q for g in groups for q in g]
    problems = [_problem(M=m, Nn=nn, Kk=kk) for m, nn, kk, _ in flat]
    extents = [_extent(p, M=m, Nn=nn, Kk=kk) for m, nn, kk, p in flat]
    qs, ext, gs = _arrays(problems, extents, [len(g) for g in groups])
    return L.gib_test_dw_scratch_bytes_passes(qs, ext, gs, len(groups))


@pytest.mark.parametrize("m", [1, 100, 683, 13452])
def test_scratch_grows_with_the_pass_count_as_the_layout_predicts(m):
    sms = L.gib_device_sm_count()
    last = 0
    for passes in (1, 2, 3, 4, 16):
        groups = [[(m, 128, 128, passes)], [(m, 256, 128, passes), (m, 384, 128, passes)]]
        got = _query(groups)
        assert got == _expected_bytes(groups, sms), (m, passes)
        assert got >= last
        last = got
    if m == 100:      # 4 units per pass: the layout, not the split-K partials, sizes the scratch from 3 passes on
        assert _query([[(100, 128, 128, 16)]]) > _query([[(100, 128, 128, 1)]])


def test_scratch_of_groups_of_17_and_32():
    """the C2 deferred launch (15 message-MLP layers over three bond types and the GRU pair, 4 passes) and a group of
    32 with mixed pass counts and an empty member; ext = NULL is one pass each"""
    sms = L.gib_device_sm_count()
    msg = [(256, 128), (256, 256), (256, 256), (256, 256), (128, 256)]
    c2 = [(m, nn, kk, 4) for m in (13452, 2242, 320) for nn, kk in msg] + [(5000, 384, 128, 4)] * 2
    assert _query([c2]) == _expected_bytes([c2], sms)
    g32 = [(0 if k % 7 == 3 else 100 + 61 * k, 144 if k % 2 else 128, 128 if k % 3 else 144, (1, 3, 16, 2)[k % 4])
           for k in range(32)]
    assert _query([g32]) == _expected_bytes([g32], sms)
    qs, _, gs = _arrays([_problem(M=m, Nn=nn, Kk=kk) for m, nn, kk, _ in g32], None, [32])
    one = [(m, nn, kk, 1) for m, nn, kk, _ in g32]
    assert L.gib_test_dw_scratch_bytes_passes(qs, None, gs, 1) == _expected_bytes([one], sms)
