"""CPU: the schedule of a grouped tensor-core weight-gradient launch whose members carry a pass extent (csrc/gemm_tc3.cu:
dw_plan / dw_segment / dw_owner with GemmDW::passes), through gib_test_dw_schedule_passes, against a numpy
restatement: units numbered member, tile, pass, k-block; CTA b of G = min(SMs, ceil(U / 8)) takes units
[U b / G, U (b + 1) / G) cut at tile boundaries only, so a segment may run from one pass into the next; slot b + tile;
the reduction sums each tile's slots over the CTAs that cover it in ascending order.  Empty members (no live rows, an
absent bond type) have no units.  With one pass the schedule is the one gib_test_dw_schedule reports."""
import ctypes

import numpy as np
import pytest

from graphinvent_b200 import _lib

BKF, TILE = 32, 128


def cdiv(a, b):
    return -(-a // b)


def _hook(rows, passes, shapes, sms):
    n = len(rows)
    tiles = sum(cdiv(nn, TILE) * cdiv(kk, TILE) for nn, kk in shapes)
    max_segs = sms + tiles + 1
    segs = (ctypes.c_int * (7 * max_segs))()
    tile_ctas = (ctypes.c_int * (2 * tiles))()
    G = ctypes.c_int(-7)
    arr = lambda v: (ctypes.c_int * n)(*v)   # noqa: E731
    ns = _lib.lib.gib_test_dw_schedule_passes(arr(rows), arr(passes), arr([s[0] for s in shapes]),
                                              arr([s[1] for s in shapes]), n, sms, segs, max_segs, tile_ctas,
                                              ctypes.byref(G))
    assert ns >= 0, _lib.lib.gib_last_error().decode()
    return G.value, [tuple(segs[7 * i:7 * i + 7]) for i in range(ns)], \
        [(tile_ctas[2 * t], tile_ctas[2 * t + 1]) for t in range(tiles)]


def _numpy_plan(rows, passes, shapes, sms):
    """the restatement: (G, segments (CTA, member, tile, first pass, first row, k-blocks, slot), per tile first / last
    CTA)"""
    mt_nt = np.array([(cdiv(nn, TILE), cdiv(kk, TILE)) for nn, kk in shapes], dtype=np.int64)
    tiles = mt_nt[:, 0] * mt_nt[:, 1]
    kb = np.array([cdiv(m, BKF) for m in rows], dtype=np.int64)
    per_tile = kb * np.array(passes, dtype=np.int64)              # units of one tile
    ubegin = np.concatenate([[0], np.cumsum(tiles * per_tile)])
    tbegin = np.concatenate([[0], np.cumsum(tiles)])
    U = int(ubegin[-1])
    G = min(sms, cdiv(U, 8))
    segs = []
    for b in range(G):
        u, u1 = U * b // G, U * (b + 1) // G
        while u < u1:
            p = int(np.searchsorted(ubegin, u, side="right") - 1)
            local = u - int(ubegin[p])
            t, k = divmod(local, int(per_tile[p]))
            nk = min(u1 - u, int(per_tile[p]) - k)
            ps, kk = divmod(k, int(kb[p]))
            segs.append((b, p, t, ps, kk * BKF, nk, b + int(tbegin[p]) + t))
            u += nk
    owner = lambda u: ((u + 1) * G - 1) // U    # noqa: E731
    tile_ctas = []
    for p in range(len(rows)):
        for t in range(int(tiles[p])):
            if per_tile[p] == 0:
                tile_ctas.append((-1, -1))
            else:
                u = int(ubegin[p]) + t * int(per_tile[p])
                tile_ctas.append((owner(u), owner(u + int(per_tile[p]) - 1)))
    return G, segs, tile_ctas


def _check(rows, passes, shapes, sms):
    got = _hook(rows, passes, shapes, sms)
    assert got == _numpy_plan(rows, passes, shapes, sms), (rows, passes, sms)
    G, segs, tile_ctas = got
    # every (member, tile, pass, k-block) once; the slots unique and inside SMs + tiles
    seen = set()
    for b, p, t, ps, r0, nk, slot in segs:
        kb = cdiv(rows[p], BKF)
        k = ps * kb + r0 // BKF
        for j in range(k, k + nk):
            key = (p, t, j // kb, j % kb)
            assert key not in seen and key[2] < passes[p]
            seen.add(key)
    assert len(seen) == sum(cdiv(nn, TILE) * cdiv(kk, TILE) * cdiv(m, BKF) * np_
                            for (nn, kk), m, np_ in zip(shapes, rows, passes))
    assert len({s[6] for s in segs}) == len(segs)
    assert all(s[6] < sms + len(tile_ctas) for s in segs)
    return G, segs


# C2's message-MLP layers (3 bond types x 5 Linears, the third type empty in one case) and its GRU pair
MSG = [(256, 128), (256, 256), (256, 256), (256, 256), (128, 256)]
GRU = [(384, 128), (384, 128)]


@pytest.mark.parametrize("passes", [1, 2, 4, 6])
@pytest.mark.parametrize("live", [(0, 0, 0), (1, 31, 0), (33, 1000, 0), (13452, 2242, 320), (4133, 4133, 4133)])
def test_message_mlps_against_numpy(live, passes):
    shapes = [s for _ in live for s in MSG]
    rows = [m for m in live for _ in MSG]
    for sms in (1, 2, 7, 66, 132):
        _check(rows, [passes] * len(rows), shapes, sms)


@pytest.mark.parametrize("rows", [1, 32, 33, 13312, 155648])
def test_gru_pair_against_numpy(rows):
    for sms in range(1, 133, 13):
        _check([rows, rows], [4, 4], GRU, sms)


def test_segments_cross_pass_boundaries():
    """few CTAs: a segment runs from the last k-block of one pass into the next pass's first"""
    G, segs = _check([100, 100], [4, 4], GRU, 3)
    crossing = [s for s in segs if cdiv(100, BKF) * s[3] + s[4] // BKF + s[5] > cdiv(100, BKF) * (s[3] + 1)]
    assert crossing, "no segment crosses a pass boundary"


def test_one_pass_is_the_former_schedule():
    """passes = 1 everywhere: the segments and the reduction order gib_test_dw_schedule reports"""
    shapes = MSG + GRU
    rows = [4097, 33, 0, 2048, 31, 13312, 7]
    n = len(rows)
    for sms in (1, 5, 132):
        G, segs, tiles = _hook(rows, [1] * n, shapes, sms)
        max_segs = sms + len(tiles) + 1
        s6 = (ctypes.c_int * (6 * max_segs))()
        tc = (ctypes.c_int * (2 * len(tiles)))()
        G6 = ctypes.c_int()
        arr = lambda v: (ctypes.c_int * n)(*v)   # noqa: E731
        ns = _lib.lib.gib_test_dw_schedule(arr(rows), arr([s[0] for s in shapes]), arr([s[1] for s in shapes]), n,
                                           sms, s6, max_segs, tc, ctypes.byref(G6))
        assert ns == len(segs) and G6.value == G
        for i, (b, p, t, ps, r0, nk, slot) in enumerate(segs):
            assert ps == 0
            assert tuple(s6[6 * i:6 * i + 6]) == (b, p, t, r0, min(rows[p] - r0, nk * BKF), slot)
        assert [(tc[2 * i], tc[2 * i + 1]) for i in range(len(tiles))] == tiles
