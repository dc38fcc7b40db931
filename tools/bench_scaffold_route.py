"""Conditional route likelihoods p(molecule | scaffold): `graphed.RouteScorer.score(..., scaffold_ids=)` against the
unconditional scorer on the same molecules and against the eager way of computing them.

    python tools/bench_scaffold_route.py [--repeats 5] [--batch 1000] [--ks 1,3,5,8]

Workload: gdb13_1K/train (979 molecules, tests/golden/preprocess_gdb13.npz) with the reference's pretrained GGNN
(oracle/_ref/pretrained_model.pth).  For each k of --ks, molecule m's scaffold is its own min(k, n_m)-atom prefix (one
table row per molecule), scored without attachment points ("free") and with the atoms each decoration bonds to as
attachment points ("attachment").  Arms, all from the same host int8 stacks, timed end to end by the host clock
around work that ends in a device synchronise, one warm-up call each, then the median of --repeats calls, the arms
alternating:
  conditional   RouteScorer(model, batch, scaffolds=..., attachment=...).score(nodes, edges, scaffold_ids=ids)
  conditional+backward   the same with requires_grad=True and nll.sum().backward()
  unconditional RouteScorer(model, batch).score(nodes, edges) (every state of every route)
  eager         numpy conditional states (tests/scaffold_route_reference.py), `model(nodes, edges)` in float32, the
                mask as -inf, softmax gather, per-molecule sums
Reported per arm as molecules/s and states/s, with the fraction of route states the conditional routes skip (the
1 + m_k states before each scaffold), the largest |d log p| between the conditional and eager arms, and the card's
name and power limit.  One JSON line per (k, attachment) configuration.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # no nvidia-smi: the record says so
        return f"unknown ({e})"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def eager(net, X, E, acts, masks, offsets, B):
    import torch
    lik = []
    with torch.no_grad():
        for s in range(0, X.shape[0], B):
            x = torch.from_numpy(X[s:s + B]).cuda().float()
            e = torch.from_numpy(E[s:s + B]).cuda().float()
            o = net(x, e).masked_fill(torch.from_numpy(masks[s:s + B]).cuda(), float("-inf"))
            a = torch.from_numpy(acts[s:s + B]).cuda().view(-1, 1)
            lik.append(torch.softmax(o, dim=1).gather(1, a).view(-1))
        lik = torch.cat(lik).double()
        off = torch.from_numpy(offsets).cuda()
        idx = torch.repeat_interleave(torch.arange(len(offsets) - 1, device="cuda"), off[1:] - off[:-1])
        nll = torch.zeros(len(offsets) - 1, dtype=torch.float64, device="cuda").index_add_(0, idx, -torch.log(lik))
        return lik.float().cpu(), nll.float().cpu()


def eager_arm(net, nodes, edges, ids, sn, protect, B):
    """the eager way end to end: the numpy conditional states and masks are part of the work"""
    from tests import scaffold_route_reference as SR
    X, E, acts, offsets, sid, n_at = SR.conditional_states(nodes, edges, ids, sn, [5, 3])
    masks = SR.state_masks(sid, n_at, sn, protect, nodes.shape[1], edges.shape[3], 45)
    return eager(net, X, E, acts, masks, offsets, B)


def configuration(net, nodes, edges, k, masked, B, repeats, gpu, whole_scorer):
    import torch
    from graphinvent_b200.graphed import RouteScorer
    from tests import preprocess_reference as P
    from tests import scaffold_route_reference as SR
    M = nodes.shape[0]
    ks = np.array([min(k, P.n_atoms(nodes[m])) for m in range(M)])
    sn, se = SR.prefix_scaffolds(nodes, edges, ks)
    ids = np.arange(M)
    attach = [SR.decoration_points(nodes[m], edges[m], int(ks[m])) for m in range(M)] if masked else None
    protect = SR.protect_of(sn, attach) if masked else None
    scorer = RouteScorer(net, B, n_atom_types=5, n_formal_charge=3, scaffolds=(sn, se), attachment=attach)

    def cond():
        out = scorer.score(nodes, edges, scaffold_ids=ids)
        return out.likelihoods.cpu(), out.nll.cpu()

    def cond_bwd():
        out = scorer.score(nodes, edges, scaffold_ids=ids, requires_grad=True)
        out.nll.sum().backward()
        net.zero_grad(set_to_none=True)

    def whole():
        return whole_scorer.score(nodes, edges).likelihoods.cpu()

    arms = {"conditional": cond, "conditional+backward": cond_bwd, "unconditional": whole,
            "eager": lambda: eager_arm(net, nodes, edges, ids, sn, protect, B)}
    res = {name: fn() for name, fn in arms.items()}                     # warm-up
    S_c, S_u = res["conditional"][0].numel(), res["unconditional"].numel()
    assert res["eager"][0].numel() == S_c
    dlogp = (torch.log(res["eager"][0].double()) - torch.log(res["conditional"][0].double())).abs().max().item()
    times = {name: [] for name in arms}
    for _ in range(repeats):
        for name, fn in arms.items():
            times[name].append(timed(fn)[0])
    rec = dict(workload="gdb13_1K/train, pretrained GGNN", k=k, attachment=masked, molecules=M,
               conditional_states=S_c, route_states=S_u, skipped_fraction=1 - S_c / S_u, batch=B, repeats=repeats,
               gpu=gpu, max_abs_dlogp=dlogp)
    for name, ts in times.items():
        t = statistics.median(ts)
        S = S_u if name == "unconditional" else S_c
        rec[name] = dict(seconds=t, molecules_per_s=M / t, states_per_s=S / t)
    rec["speedup_vs_eager"] = rec["eager"]["seconds"] / rec["conditional"]["seconds"]
    rec["time_vs_unconditional"] = rec["conditional"]["seconds"] / rec["unconditional"]["seconds"]
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--ks", default="1,3,5,8")
    ap.add_argument("--out", help="also write the JSON lines here")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_scaffold_route.py needs a CUDA device")
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import RouteScorer
    from tests.conftest import pretrained_path
    gpu = card()
    path = pretrained_path()
    if path is None:
        raise SystemExit("oracle/_ref/pretrained_model.pth is missing: run __graft_entry__.build() first")
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]
    net = mpnn.create(make_constants("GGNN"))
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    net = net.cuda().eval()
    whole = RouteScorer(net, a.batch, n_atom_types=5, n_formal_charge=3)
    recs = [configuration(net, nodes, edges, int(k), masked, a.batch, a.repeats, gpu, whole)
            for k in a.ks.split(",") for masked in (False, True)]
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in recs)


if __name__ == "__main__":
    main()
