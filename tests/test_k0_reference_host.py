"""CPU: the numpy restatement of K0 (tests/k0_reference.py) against torch.nonzero, its truncation rule on hand-made
batches, and the guard-band helper (tests/guarded.py) that the GPU memory-discipline tests rely on."""
import numpy as np
import pytest
import torch

from tests.guarded import MIB, Guarded
from tests.k0_reference import FLAG_MULTITYPE, FLAG_NONBINARY, FLAG_OVERFLOW, capacity_rows, k0_reference


def _random_edges(B, N, Ef, seed, p=0.15):
    rng = np.random.default_rng(seed)
    e = np.zeros((B, N, N, Ef), np.float32)
    b, i, j = np.nonzero(rng.random((B, N, N)) < p)
    e[b, i, j, rng.integers(0, Ef, b.size)] = 1.0
    return e


@pytest.mark.parametrize("by_type", [True, False], ids=["typed", "EMN"])
@pytest.mark.parametrize("B,N,Ef", [(1, 1, 1), (7, 5, 3), (40, 13, 4), (3, 9, 2)])
def test_exact_mode_matches_nonzero(by_type, B, N, Ef):
    e = _random_edges(B, N, Ef, seed=B * N + Ef)
    e[B - 1, N - 1, 0, :] = [0.5, 2.0, 1.0, 1.0][:Ef]          # multi-type, non-binary cell
    r = k0_reference(e, by_type)
    et = torch.from_numpy(e)
    G = Ef if by_type else 1
    nz = (et != 0) if by_type else (et != 0).any(-1, keepdim=True)
    assert r.E == int(nz.sum()) and r.G == G
    base = 0
    for t in range(G):
        b, i, j = nz[..., t].nonzero(as_tuple=True)               # row-major (b, i, j): the reference's order
        cnt = b.numel()
        assert r.hdr[2 + t] == cnt and r.hdr[6 + t] == base
        sl = slice(base, base + cnt)
        assert np.array_equal(r.ent_dst[sl], (b * N + i).numpy()) and np.array_equal(r.ent_src[sl], (b * N + j).numpy())
        want_w = et[b, i, j, t] if by_type else torch.ones(cnt)
        assert np.array_equal(r.ent_w[sl], want_w.numpy())
        pad_to = base + (cnt + 127) // 128 * 128
        assert (r.ent_src[base + cnt: pad_to] == -1).all() and (r.ent_w[base + cnt: pad_to] == 0).all()
        base = pad_to
    assert r.P == base and r.hdr[1] == base and r.hdr[6 + G] == base
    # CSR by destination: (b, i, j, t) order; by source: (b, j, i, t) order
    cells = nz.nonzero()
    for order, ptr, ent in (((0, 1, 2, 3), r.dst_ptr, r.dst_ent), ((0, 2, 1, 3), r.src_ptr, r.src_ent)):
        key = cells[:, list(order)]
        idx = np.lexsort(key.numpy().T[::-1])
        got_cells = r.ent_dst[ent] // N, r.ent_dst[ent] % N, r.ent_src[ent] % N
        want = cells[idx].numpy()
        assert np.array_equal(got_cells[0], want[:, 0]) and np.array_equal(got_cells[1], want[:, 1])
        assert np.array_equal(got_cells[2], want[:, 2])
        slot = want[:, 0] * N + (want[:, 1] if order[1] == 1 else want[:, 2])
        assert np.array_equal(ptr, np.concatenate([[0], np.cumsum(np.bincount(slot, minlength=B * N))]))
    assert not r.overflow and r.survivors.all()


def test_flags():
    e = np.zeros((2, 3, 3, 3), np.float32)
    assert k0_reference(e, True).flags == 0 and k0_reference(e, True).E == 0
    e[0, 1, 2, 0] = 1.0
    assert k0_reference(e, True).flags == 0
    e[0, 1, 2, 1] = 1.0
    assert k0_reference(e, True).flags == FLAG_MULTITYPE
    e[1, 0, 0, 2] = np.nan                                     # NaN is a bond (nonzero) and not 1
    assert k0_reference(e, True).flags == FLAG_MULTITYPE | FLAG_NONBINARY
    z = np.zeros((1, 2, 2, 1), np.float32)
    z[0, 1, 1, 0] = -0.0                                       # -0.0 is no bond
    assert k0_reference(z, False).E == 0
    i8 = np.zeros((1, 2, 2, 2), np.int8)
    i8[0, 0, 1] = [-128, 127]
    r = k0_reference(i8, True)
    assert r.E == 2 and r.flags == FLAG_MULTITYPE | FLAG_NONBINARY
    assert sorted(r.ent_w[r.ent_src >= 0].tolist()) == [-128.0, 127.0]


def _groups_batch():
    """3 bond types with 700, 200 and 100 entries in 10 molecules of 100 cells: group bases 0, 768, 1024, P = 1152"""
    e = np.zeros((10, 10, 10, 3), np.float32)
    c = np.arange(1000)
    t = np.where(c % 10 < 7, 0, np.where(c % 10 < 9, 1, 2))
    e.reshape(1000, 3)[c, t] = 1.0
    return e


# capacity -> P_cap = ceil128(capacity) + 3 * 128, and the molecules that survive
CUTS = {
    "above_E": (1001, 1408, "all"),
    "at_E": (1000, 1408, "all"),
    "below_E": (999, 1408, "all_but_last"),        # every row kept, the last CSR slot dropped
    "inside_group1": (450, 896, "none"),           # group 1 cut at row 896, group 2 dropped
    "at_group1": (300, 768, "none"),               # P_cap == base of group 1: groups 1 and 2 dropped
    "inside_group0": (100, 512, "none"),
    "one": (1, 512, "none"),
}


@pytest.mark.parametrize("cut", list(CUTS))
def test_truncation_rule(cut):
    e = _groups_batch()
    full = k0_reference(e, True)
    assert list(full.type_base) == [0, 768, 1024, 1152] and full.E == 1000
    cap, cap_P, surv = CUTS[cut]
    r = k0_reference(e, True, capacity=cap)
    assert r.cap_P == cap_P == capacity_rows(cap, 3)
    assert r.ent_src.size == cap_P and r.dst_ent.size == min(1000, cap)
    assert r.overflow == (1000 > cap) and bool(r.hdr[11] & FLAG_OVERFLOW) == (1000 > cap)
    assert r.hdr[0] == 1000 and r.hdr[1] == 1152              # the header keeps the true counts
    # rows below P_cap are exact mode's rows; rows [P, P_cap) are pad rows
    n = min(cap_P, full.P)
    assert np.array_equal(r.ent_src[:n], full.ent_src[:n]) and np.array_equal(r.ent_dst[:n], full.ent_dst[:n])
    assert np.array_equal(r.ent_w[:n], full.ent_w[:n])
    assert (r.ent_src[full.P:] == -1).all() and (r.ent_dst[full.P:] == -1).all() and (r.ent_w[full.P:] == 0).all()
    # kept CSR slots name exact mode's row, or row 0 when that row was dropped; pointers are clamped to the capacity
    k = r.dst_ent.size
    assert np.array_equal(r.dst_ent, np.where(full.dst_ent[:k] < cap_P, full.dst_ent[:k], 0))
    assert np.array_equal(r.src_ent, np.where(full.src_ent[:k] < cap_P, full.src_ent[:k], 0))
    assert np.array_equal(r.dst_ptr, np.minimum(full.dst_ptr, cap))
    assert np.array_equal(r.src_ptr, np.minimum(full.src_ptr, cap))
    # survivors, restated from the CSR: every row of the molecule below P_cap, its last slot below the capacity
    for b in range(10):
        rows = full.dst_ent[full.dst_ptr[b * 10]: full.dst_ptr[b * 10 + 10]]
        assert r.survivors[b] == (rows.max() < cap_P and full.dst_ptr[b * 10 + 10] <= cap), b
    want = {"all": [True] * 10, "all_but_last": [True] * 9 + [False], "none": [False] * 10}[surv]
    assert list(r.survivors) == want
    # the graph buffer holds E_cap slots and P_cap rows: nothing is laid out past them
    assert r.expected_buf.size == r.layout["src_ent"] + (cap + 31) // 32 * 32


def test_capacity_survivors_of_a_cut_inside_the_last_group():
    """molecules whose entries all lie below the cut survive, the others do not"""
    e = np.zeros((4, 4, 4, 2), np.float32)
    e[:, :, :, 1] = 1.0                                      # 64 entries of type 1 (rows 128..191)
    e[0, 0, 1, 0] = 1.0                                      # one of type 0 (row 0)
    full = k0_reference(e, True)
    assert list(full.type_base) == [0, 128, 256] and full.E == 65
    r = k0_reference(e, True, capacity=20)                   # P_cap = 128 + 256 = 384: every row kept, 20 CSR slots
    assert r.cap_P == 384 and r.overflow
    assert list(r.survivors) == [True, False, False, False]  # molecule 0 holds 17 entries, its CSR ends at slot 17


@pytest.mark.parametrize("device", ["cpu"] + (["cuda"] if torch.cuda.is_available() else []))
@pytest.mark.parametrize("where", ["front_first", "front_last", "back_first", "back_last"])
def test_guard_detects_a_one_byte_write(device, where):
    g = Guarded(1000, device=device)
    assert g.start >= MIB and g.raw.numel() - g.start - 1000 >= MIB
    assert g.t.data_ptr() % 512 == 0 and g.t.numel() == 1000
    assert g.intact() and bool((g.t == 0xFF).all())
    g.t.fill_(0)                                             # the interior is the caller's
    assert g.intact() and g.damage() is None
    pos = {"front_first": 0, "front_last": g.start - 1, "back_first": g.start + 1000,
           "back_last": g.raw.numel() - 1}[where]
    g.raw[pos] = 0xFE
    assert not g.intact()
    assert g.damage() == (pos - g.start, pos - g.start)


def test_guarded_copy_and_zero_fill():
    src = torch.arange(12, dtype=torch.float32).view(3, 4)
    g = Guarded.like(src, device="cpu")
    assert torch.equal(g.view(), src) and g.intact()
    z = Guarded(64, device="cpu", fill="zero")
    assert bool((z.t == 0).all()) and z.intact()
    assert torch.isnan(Guarded(16, device="cpu").view(torch.float32)).all()
    assert (Guarded(16, device="cpu").view(torch.int32) == -1).all()
