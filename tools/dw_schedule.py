"""Host model of the tensor-core weight-gradient launches of one C2 training step (bench.py --config C2: GGNN, hidden
128, message 128, 4 passes, batch 1024 of 13-atom graphs): the makespan of each grouped dW launch under the former
schedule (one chunk length per launch from rows x the largest member's tiles, chunks dealt to CTAs round-robin) and
under the even k-block split of csrc/gemm_tc3.cu (dw_plan), both from the plan's shapes; and for the pass-shared
weights (GRU, message rows) the even split of one launch over all 4 passes (GemmDW::passes) against 4 per-pass
launches.  CPU only, no library:

    python tools/dw_schedule.py [--sms 132]

Assumptions (a model, not a measurement): 1536 clocks per 128 x 128 x 32 k-block (the 3xTF32 tensor rate), 2.5 k
clocks to drain a work item / segment, no overlap between CTAs' drains and the next item.  Members narrower than 32
(the SIMT kernel's) are left out of the launches and of the split."""
import argparse

BKF, KB_CLK, DRAIN, MAX_CHUNK = 32, 1536, 2500, 4096


def cdiv(a, b):
    return -(-a // b)


def tiles(nn, kk):
    return cdiv(nn, 128) * cdiv(kk, 128)


def former(members, sms, plan_rows=0):
    """per-CTA clocks of the chunk-and-round-robin rule; members: (Nn, Kk, M, live); plan_rows: capacity mode"""
    mt = max(tiles(nn, kk) for nn, kk, _, _ in members)
    rows = plan_rows or sum(m for _, _, m, _ in members)
    c = 8 * BKF
    for r in range(1, 65):
        c = cdiv(cdiv(rows * mt, r * sms), BKF) * BKF
        if c <= MAX_CHUNK:
            break
    c = max(min(c, MAX_CHUNK), 8 * BKF)
    items = []
    for nn, kk, _, live in members:
        for z in range(cdiv(live, c)):
            rows_z = min(live, (z + 1) * c) - z * c
            items += [cdiv(rows_z, BKF)] * tiles(nn, kk)
    grid = min(len(items), sms)
    per = [0] * grid
    for i, k in enumerate(items):
        per[i % grid] += k * KB_CLK + DRAIN
    return c, len(items), max(per)


def even(members, sms, passes=1):
    """per-CTA clocks of the even split: CTA b takes units [U b / G, U (b + 1) / G), one drain per tile it touches;
    passes: every member reduces over that many slices (a tile holds kb * passes units)"""
    bounds, u = [], 0
    for nn, kk, _, live in members:
        kb = cdiv(live, BKF) * passes
        for _ in range(tiles(nn, kk)):
            if kb:
                bounds.append((u, u + kb))
            u += kb
    U = u
    G = min(sms, cdiv(U, 8))
    worst, segs = 0, 0
    for b in range(G):
        u0, u1 = U * b // G, U * (b + 1) // G
        n = sum(1 for a, e in bounds if a < u1 and e > u0)
        segs += n
        worst = max(worst, (u1 - u0) * KB_CLK + n * DRAIN)
    return G, segs, worst


def c2_launches():
    """(name, members, plan rows of the former rule, launches per step) of one C2 step"""
    S, B = 1024 * 13, 1024
    out = []
    fadd2 = [(512, 688), (512, 512), (512, 512), (512, 512), (592, 512)]
    fconn2 = [(512, 144), (512, 512), (512, 512), (512, 512), (48, 512)]
    fterm2 = [(512, 112), (512, 512), (512, 512), (512, 512)]          # last layer (Nn = 16): SIMT kernel
    out.append(("tier-2 APD heads (M = 1024)", [(a, b, B, B) for a, b in fadd2 + fconn2 + fterm2], 0, 1))
    fadd1 = [(512, 128), (512, 512), (512, 512), (512, 512), (48, 512)]
    fconn1 = [(512, 128), (512, 512), (512, 512), (512, 512)]          # last layer (Nn = 16): SIMT kernel
    out.append(("tier-1 APD heads (M = 13312)", [(a, b, S, S) for a, b in fadd1 + fconn1], 0, 1))
    gemb = [(256, 128), (256, 256), (256, 256), (256, 256), (112, 256)]
    gatt = [(256, 144), (256, 256), (256, 256), (256, 256), (112, 256)]
    out.append(("gather MLPs (M = 13312)", [(a, b, S, S) for a, b in gemb + gatt], 0, 1))
    out.append(("GRU projections", [(384, 128, S, S), (384, 128, S, S)], 0, 4))
    msg = [(256, 128), (256, 256), (256, 256), (256, 256), (128, 256)]
    live, cap = [13452, 2242, 320], 30336                            # bond-type groups of the benchmark batch
    out.append(("message rows, capacity mode", [(a, b, cap, m) for m in live for a, b in msg], cap * 5, 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--ghz", type=float, default=1.55)
    args = ap.parse_args()
    print(f"{'dW launch (C2)':34s} {'chunk':>6s} {'items':>6s} {'former kclk':>12s} {'G':>4s} {'segs':>5s} "
          f"{'even kclk':>10s} {'former/even':>12s} {'x/step':>6s}")
    tot_f = tot_e = 0
    for name, members, plan, n in c2_launches():
        c, items, mf = former(members, args.sms, plan)
        G, segs, me = even(members, args.sms)
        tot_f += mf * n
        tot_e += me * n
        print(f"{name:34s} {c:6d} {items:6d} {mf / 1e3:12.1f} {G:4d} {segs:5d} {me / 1e3:10.1f} {mf / me:12.2f} {n:6d}")
    print(f"step: former {tot_f / 1e3:.0f} k clk, even {tot_e / 1e3:.0f} k clk: "
          f"{(tot_f - tot_e) / (args.ghz * 1e9) * 1e3:.3f} ms at {args.ghz} GHz")
    tot_p = tot_a = 0
    for name, members, _, n in c2_launches():
        if n == 1:
            continue
        _, _, per = even(members, args.sms)
        G, segs, once = even(members, args.sms, passes=n)
        tot_p += per * n
        tot_a += once
        print(f"{name:34s} per pass {n} x {per / 1e3:.1f} k clk, all passes in one launch {once / 1e3:.1f} k clk "
              f"(G {G}, {segs} segments)")
    print(f"pass-shared weights: {(tot_p - tot_a) / (args.ghz * 1e9) * 1e3:.3f} ms at {args.ghz} GHz, plus "
          f"{2 * (4 - 1)} launch ramps and tails")


if __name__ == "__main__":
    main()
