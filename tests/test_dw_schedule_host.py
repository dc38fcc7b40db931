"""CPU: the schedule of the grouped tensor-core weight-gradient launch (csrc/gemm_tc3.cu: dw_plan / dw_segment /
dw_owner, the same host / device arithmetic the kernel and the reduction run), through gib_test_dw_schedule.  For live
row counts around the k-block of 32 rows and SM counts 1..132: every (member, tile, k-block) unit is covered by
exactly one segment, a CTA's segments are its even share of the units, there are at most G + T segments, every slot
fits the SMs + T scratch slots, and the reduction reads each tile's slots in ascending CTA order."""
import ctypes

import pytest

from graphinvent_b200 import _lib

BKF, TILE = 32, 128


def cdiv(a, b):
    return -(-a // b)


def _schedule(rows, shapes, sms):
    n = len(rows)
    tiles = sum(cdiv(nn, TILE) * cdiv(kk, TILE) for nn, kk in shapes)
    max_segs = sms + tiles + 1
    segs = (ctypes.c_int * (6 * max_segs))()
    tile_ctas = (ctypes.c_int * (2 * tiles))()
    G = ctypes.c_int(-7)
    arr = lambda v: (ctypes.c_int * n)(*v)   # noqa: E731
    ns = _lib.lib.gib_test_dw_schedule(arr(rows), arr([s[0] for s in shapes]), arr([s[1] for s in shapes]), n, sms,
                                       segs, max_segs, tile_ctas, ctypes.byref(G))
    assert ns >= 0, _lib.lib.gib_last_error().decode()
    return G.value, [tuple(segs[6 * i:6 * i + 6]) for i in range(ns)], \
        [(tile_ctas[2 * t], tile_ctas[2 * t + 1]) for t in range(tiles)]


def _check(rows, shapes, sms):
    G, segs, tile_ctas = _schedule(rows, shapes, sms)
    mt_nt = [(cdiv(nn, TILE), cdiv(kk, TILE)) for nn, kk in shapes]
    tbegin = [0]
    for mt, nt in mt_nt:
        tbegin.append(tbegin[-1] + mt * nt)
    T = tbegin[-1]
    units = [mt * nt * cdiv(m, BKF) for m, (mt, nt) in zip(rows, mt_nt)]
    U = sum(units)
    assert G == min(sms, cdiv(U, 8)), (G, U, sms)
    assert len(segs) <= G + T

    # every unit exactly once, in the order of the CTAs and of the units
    covered = {}
    order = []
    for b, p, t, r0, nr, slot in segs:
        assert 0 <= b < G and 0 <= p < len(rows) and 0 <= t < mt_nt[p][0] * mt_nt[p][1]
        assert r0 % BKF == 0 and nr > 0 and r0 + nr <= rows[p], (p, r0, nr, rows[p])
        for k in range(r0 // BKF, cdiv(r0 + nr, BKF)):
            key = (p, t, k)
            assert key not in covered, f"unit {key} covered twice"
            covered[key] = b
            order.append((b, p, t, k))
    assert len(covered) == U
    assert order == sorted(order), "a CTA's units are not one ascending range"
    # the even split: CTA b holds units [floor(U b / G), floor(U (b + 1) / G))
    per_cta = [0] * max(G, 1)
    for b in covered.values():
        per_cta[b] += 1
    for b in range(G):
        assert per_cta[b] == U * (b + 1) // G - U * b // G

    # slots: unique, b + global tile, inside the scratch of SMs + T slots
    slots = [s[5] for s in segs]
    assert len(set(slots)) == len(slots)
    for b, p, t, _, _, slot in segs:
        assert slot == b + tbegin[p] + t and slot < G + T <= sms + T

    # the reduction: per tile the CTAs first .. last, each with exactly one segment there, summed in ascending order
    by_tile = {}
    for b, p, t, _, _, _ in segs:
        by_tile.setdefault(tbegin[p] + t, []).append(b)
    for gt, (first, last) in enumerate(tile_ctas):
        ctas = by_tile.get(gt, [])
        if first < 0:
            assert ctas == [] and last == -1
        else:
            assert ctas == list(range(first, last + 1)), (gt, ctas, first, last)
    return G, segs


# member shapes (padded Nn, Kk): one tile, 16 tiles, ragged tiles, and C2's gather MLP group
SHAPES = {
    "one_and_sixteen": [(128, 128), (512, 512), (112, 144), (48, 608)],
    "gather_mlps": [(256, 128), (256, 256), (256, 256), (256, 256), (112, 256),
                    (256, 144), (256, 256), (256, 256), (256, 256), (112, 256)],
}
CAP = 4133


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("live", [0, 1, 31, 32, 33, 1000, CAP])
def test_every_unit_once_for_each_sm_count(name, live):
    shapes = SHAPES[name]
    rows = [live if i % 2 == 0 else max(live - 7, 0) for i in range(len(shapes))]
    for sms in range(1, 133):
        _check(rows, shapes, sms)


def test_segments_cross_tile_and_member_boundaries():
    """few CTAs: each range spans several tiles and members; many: tiles are shared by consecutive CTAs"""
    shapes = SHAPES["one_and_sixteen"]
    G, segs = _check([4097, 33, 0, 2048], shapes, 5)
    assert G == 5 and len({s[1] for s in segs if s[0] == 0}) >= 1
    assert any(len({s[1] for s in segs if s[0] == b}) > 1 for b in range(G)), "no CTA crosses a member boundary"
    G, segs = _check([4097, 33, 0, 2048], shapes, 132)
    per_tile = {}
    for b, p, t, *_ in segs:
        per_tile.setdefault((p, t), set()).add(b)
    assert max(len(v) for v in per_tile.values()) > 1, "no tile split between CTAs"

