"""numpy restatement of the GGNN / MNN message-row table (graphinvent_b200/csrc/graph.cuh: MsgRows) from K0's arrays.

The entries with value 1 that share (molecule, source slot, bond type) share one message row, every other entry has a
row of its own.  Type group t starts at the entry group's first row tb[t]; inside it rows ascend by source slot, and for
one (slot, type) the shared row comes first, then one row per other entry in source-CSR order.  A source-CSR position
whose entry has another source slot (capacity mode: K0 lists row 0 for an entry it dropped) is not an entry of the slot.
"""
import numpy as np

MR_COUNT, MR_BASE, MR_EOFF, MR_TOTAL, MR_META_INTS = 0, 4, 9, 14, 16


def msg_rows_reference(ent_src, ent_dst, ent_w, dst_ptr, dst_ent, src_ptr, src_ent, tb, G, E):
    """K0's arrays (P and S from their lengths), the type bases tb[0..G] and the entry capacity E of the E-sized arrays
    (the header's E) -> dict of the table's arrays"""
    P, S = len(ent_src), len(src_ptr) - 1
    tb = [int(x) for x in tb[:G + 1]]

    def type_of(p):
        t = G - 1
        while t > 0 and p < tb[t]:
            t -= 1
        return t

    # rows of each type in order: (slot, w, entries)
    rows = [[] for _ in range(G)]
    for s in range(S):
        shared = [[] for _ in range(G)]
        own = [[] for _ in range(G)]
        for q in range(src_ptr[s], src_ptr[s + 1]):
            e = int(src_ent[q])
            if ent_src[e] != s:
                continue
            (shared if ent_w[e] == 1.0 else own)[type_of(e)].append(e)
        for t in range(G):
            if shared[t]:
                rows[t].append((s, np.float32(1.0), shared[t]))
            rows[t].extend((s, ent_w[e], [e]) for e in own[t])
    count = [max(0, min(len(rows[t]), tb[t + 1] - tb[t])) for t in range(G)]
    eoff = np.concatenate([[0], np.cumsum([sum(len(r[2]) for r in rows[t]) for t in range(G)])]).astype(np.int64)

    u_src = np.full(P, -1, np.int32)
    u_w = np.zeros(P, np.float32)
    u_ptr = np.zeros(P + 1, np.int32)
    u_dst = np.full(E, -1, np.int32)
    ent_u = np.full(P, -1, np.int32)
    row_of = {}                                    # (type, index in the group) -> row, for the slot CSR
    for t in range(G):
        pos = eoff[t]
        for k, (s, w, ents) in enumerate(rows[t]):
            row = tb[t] + k if k < count[t] and tb[t] + k < P else -1
            row_of[(t, k)] = row
            if row >= 0:
                u_src[row], u_w[row], u_ptr[row] = s, w, min(E, pos)
                ent_u[ents] = row
            for e in ents:
                if pos < E:
                    u_dst[pos] = ent_dst[e]
                pos += 1
    for p in range(P):
        t = type_of(p)
        if p >= tb[t] + count[t] or p >= tb[G]:
            u_src[p], u_w[p], u_ptr[p] = -1, 0.0, min(E, eoff[t + 1])
    u_ptr[P] = min(E, eoff[G])

    # source slot -> its message rows, by type
    s_ptr = np.zeros(S + 1, np.int32)
    s_u = np.full(E, -1, np.int32)
    by_slot = [[[] for _ in range(G)] for _ in range(S)]
    for t in range(G):
        for k, (s, _, _) in enumerate(rows[t]):
            by_slot[s][t].append(row_of[(t, k)])
    n = 0
    for s in range(S):
        s_ptr[s] = min(E, n)
        for t in range(G):
            for row in by_slot[s][t]:
                if n < E:
                    s_u[n] = row
                n += 1
    s_ptr[S] = min(E, n)
    total = n

    live = int(dst_ptr[S])
    dst_u = np.full(E, -1, np.int32)
    dst_u[:live] = ent_u[dst_ent[:live]]

    meta = np.zeros(MR_META_INTS, np.int32)
    meta[MR_COUNT:MR_COUNT + G] = count
    meta[MR_BASE:MR_BASE + G + 1] = tb
    meta[MR_EOFF:MR_EOFF + G + 1] = eoff
    meta[MR_TOTAL] = total
    return dict(u_src=u_src, u_w=u_w, u_ptr=u_ptr, u_dst=u_dst, ent_u=ent_u, dst_u=dst_u, s_ptr=s_ptr, s_u=s_u,
                meta=meta)


TABLE_ARRAYS = ("u_src", "u_w", "u_ptr", "u_dst", "ent_u", "dst_u", "s_ptr", "s_u", "meta")   # gib_model_msg_rows order
