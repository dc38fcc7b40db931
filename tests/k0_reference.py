"""K0 (csrc/graph_build.cu) restated in numpy: from a dense bond tensor to the count workspace and the graph buffer,
byte for byte, in exact mode and in capacity mode.

Vocabulary as in graph_build.cu: a bond entry is one non-zero element edges[b, i, j, t] (NaN counts, -0.0 does not);
with typed groups (every model but the EMN) group t holds the entries of bond type t, the EMN has one group whose entry
is the cell (b, i, j) when any of its types is non-zero, with weight 1.  Each group starts on a 128-row boundary; pad
rows hold src = dst = -1, w = 0.  dst_ent lists the entry rows in (b, i, j, t) order, src_ent in (b, j, i, t) order.

Capacity mode (`capacity` = entry capacity E_cap): the arrays hold E_cap CSR slots and P_cap = ceil128(E_cap) +
128 G entry rows (gib_graph_header_capacity).  An entry row p >= P_cap is dropped, a CSR slot q >= E_cap is dropped, a
kept slot that names a dropped row names row 0, pointers are clamped to E_cap, the rows [P, P_cap) are pad rows, and
the overflow flag is raised when E > E_cap.  Bytes no kernel writes keep whatever the buffer held: `expected_*` arrays
hold `unwritten` there (the poison of tests/guarded.py by default).
"""
import numpy as np

TILE = 128
HDR_INTS = 16
HDR_E, HDR_P, HDR_TYPE_COUNT, HDR_TYPE_BASE, HDR_FLAGS = 0, 1, 2, 6, 11
FLAG_MULTITYPE, FLAG_NONBINARY, FLAG_OVERFLOW = 1, 2, 4


def ceil_tile(n):
    return -(-int(n) // TILE) * TILE


def _al(n):
    """array starts inside the graph buffer are 128-byte aligned (csrc/model.cu graph_arrays)"""
    return (int(n) + 31) & ~31


def graph_layout(S, E, P):
    """int32 offsets of the seven arrays inside the graph buffer, and its length in int32"""
    off = {}
    o = 0
    for name, n in (("ent_src", P), ("ent_dst", P), ("ent_w", P), ("dst_ptr", S + 1), ("dst_ent", E),
                    ("src_ptr", S + 1), ("src_ent", E)):
        off[name] = o
        o += _al(n)
    return off, o


def capacity_rows(capacity, G):
    """P_cap of gib_graph_header_capacity: every group padded to 128 rows adds at most 127 rows per group"""
    return ceil_tile(capacity) + G * TILE


class K0Result:
    pass


def k0_reference(edges, by_type, capacity=None, unwritten=-1):
    """edges: numpy [B, N, N, Ef] float32 or int8.  by_type: typed groups (GGNN / MNN / AttGGNN) or one group (EMN).
    Returns a K0Result with the header, the per-array contents, the full expected count workspace and graph buffer
    (int32 views) and, in capacity mode, the molecules that survive the truncation."""
    e = np.asarray(edges)
    assert e.ndim == 4 and e.dtype in (np.float32, np.int8), (e.shape, e.dtype)
    B, N, _, Ef = e.shape
    S = B * N
    v = e.astype(np.float32)
    nz = v != 0
    flags = 0
    if (nz.sum(-1) > 1).any():
        flags |= FLAG_MULTITYPE
    if (nz & (v != 1)).any():
        flags |= FLAG_NONBINARY
    G = Ef if by_type else 1
    if by_type:
        f, w = nz, v
    else:
        f, w = nz.any(-1, keepdims=True), np.ones((B, N, N, 1), np.float32)

    cnt = f.reshape(B, N * N, G).sum(1).T.astype(np.int64)          # [G, B]
    tc = cnt.sum(1)
    base = [0]
    for g in range(G):
        base.append(base[-1] + ceil_tile(tc[g]))
    E, P = int(tc.sum()), base[G]
    tot = cnt.sum(0)                                                 # entries per molecule
    ent_off = np.concatenate([[0], np.cumsum(tot)[:-1]]).astype(np.int64)
    off = np.concatenate([np.zeros((G, 1), np.int64), np.cumsum(cnt, 1)[:, :-1]], 1)

    # entry row of every non-zero cell: group base + rank in row-major (b, i, j) order inside the group
    prow = np.full(f.shape, -1, np.int64)
    for g in range(G):
        b, i, j = np.nonzero(f[..., g])
        prow[b, i, j, g] = base[g] + np.arange(b.size)
    dst_order = prow.ravel()[np.flatnonzero(f)]
    src_order = np.ascontiguousarray(prow.transpose(0, 2, 1, 3)).ravel()[
        np.flatnonzero(np.ascontiguousarray(f.transpose(0, 2, 1, 3)))]
    dst_ptr = np.concatenate([[0], np.cumsum(f.sum((2, 3)).reshape(S))])
    src_ptr = np.concatenate([[0], np.cumsum(f.sum((1, 3)).reshape(S))])

    cap = capacity is not None
    cap_E = int(capacity) if cap else E
    cap_P = capacity_rows(cap_E, G) if cap else P
    if cap and E > cap_E:
        flags |= FLAG_OVERFLOW

    # entry arrays over [0, cap_P): entries, group pads, tail pads
    ent_src = np.full(cap_P, -1, np.int64)
    ent_dst = np.full(cap_P, -1, np.int64)
    ent_w = np.zeros(cap_P, np.float32)
    for g in range(G):
        b, i, j = np.nonzero(f[..., g])
        p = base[g] + np.arange(b.size)
        keep = p < cap_P
        ent_src[p[keep]] = (b * N + j)[keep]
        ent_dst[p[keep]] = (b * N + i)[keep]
        ent_w[p[keep]] = w[b, i, j, g][keep]
    n_slots = min(E, cap_E)
    dst_ent = np.where(dst_order < cap_P, dst_order, 0)[:n_slots]
    src_ent = np.where(src_order < cap_P, src_order, 0)[:n_slots]

    hdr = np.zeros(HDR_INTS, np.int64)
    hdr[HDR_E], hdr[HDR_P] = E, P
    hdr[HDR_TYPE_COUNT:HDR_TYPE_COUNT + G] = tc
    hdr[HDR_TYPE_BASE:HDR_TYPE_BASE + G + 1] = base
    hdr[HDR_FLAGS] = flags

    r = K0Result()
    r.B, r.N, r.Ef, r.G, r.S = B, N, Ef, G, S
    r.E, r.P, r.cap_E, r.cap_P, r.capacity = E, P, cap_E, cap_P, capacity
    r.hdr = hdr.astype(np.int32)
    r.type_count, r.type_base, r.flags = tc, np.array(base), flags
    r.ent_src, r.ent_dst, r.ent_w = ent_src.astype(np.int32), ent_dst.astype(np.int32), ent_w
    r.dst_ptr = np.minimum(dst_ptr, cap_E).astype(np.int32)
    r.src_ptr = np.minimum(src_ptr, cap_E).astype(np.int32)
    r.dst_ent, r.src_ent = dst_ent.astype(np.int32), src_ent.astype(np.int32)
    r.overflow = bool(flags & FLAG_OVERFLOW)

    # the count workspace: header, per-group counts [G, B], their exclusive scans over molecules, entry offsets [B]
    r.expected_cws = np.concatenate([r.hdr, cnt.ravel(), off.ravel(), ent_off]).astype(np.int32)

    # the graph buffer, sized as gib_graph_bytes sizes it for the header the caller passes (E / P, or E_cap / P_cap)
    lay, total = graph_layout(S, cap_E, cap_P)
    buf = np.full(total, unwritten, np.int32)
    for name, arr in (("ent_src", r.ent_src), ("ent_dst", r.ent_dst), ("ent_w", r.ent_w.view(np.int32)),
                      ("dst_ptr", r.dst_ptr), ("dst_ent", r.dst_ent), ("src_ptr", r.src_ptr), ("src_ent", r.src_ent)):
        buf[lay[name]: lay[name] + arr.size] = arr
    r.layout, r.expected_buf = lay, buf

    # molecules whose every entry row is below P_cap and whose CSR slots are all below E_cap: their message passing
    # sees exactly the bonds of exact mode
    maxrow = prow.reshape(B, -1).max(1)
    r.survivors = (maxrow < cap_P) & (ent_off + tot <= cap_E)
    return r
