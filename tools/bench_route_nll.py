"""Decoding-route likelihoods of molecules: `graphed.RouteScorer.score` against the eager way of computing them
without it.

    python tools/bench_route_nll.py [--repeats 5] [--synthetic 1000] [--batch 1000]

Eager arm: each molecule's route states built with numpy (tests/preprocess_reference.route, reversed into build
order), batched through `model(nodes, edges)` in float32 and `softmax(...).gather(action)`, then the per-molecule
sums.  Scorer arm: `RouteScorer(model, batch).score(nodes, edges)` from the same host int8 stacks.  Both are timed
end to end -- state construction, uploads, kernels, the copies back -- by the host clock around work that ends in
a device synchronise; one warm-up call each, then the median of --repeats calls, the two arms alternating.

Workloads: gdb13_1K/train (979 molecules, tests/golden/preprocess_gdb13.npz) with the reference's pretrained GGNN
(oracle/_ref/pretrained_model.pth), and --synthetic molecules of up to 38 atoms (graphinvent_b200.synthetic) with a
seeded GGNN of max_n_nodes 38.  Reported per arm as molecules/s and states/s, with the largest |d log p| between the
arms, and the card's name and power limit.  One JSON line per workload.
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


def eager(net, nodes, edges, segs, B):
    import torch
    from tests import route_nll_reference as R
    X, E, acts, offsets = R.build_order_states(nodes, edges, segs)
    lik = []
    with torch.no_grad():
        for s in range(0, X.shape[0], B):
            x = torch.from_numpy(X[s:s + B]).cuda().float()
            e = torch.from_numpy(E[s:s + B]).cuda().float()
            a = torch.from_numpy(acts[s:s + B]).cuda().view(-1, 1)
            lik.append(torch.softmax(net(x, e), dim=1).gather(1, a).view(-1))
        lik = torch.cat(lik).double()
        off = torch.from_numpy(offsets).cuda()
        idx = torch.repeat_interleave(torch.arange(len(offsets) - 1, device="cuda"), off[1:] - off[:-1])
        nll = torch.zeros(len(offsets) - 1, dtype=torch.float64, device="cuda").index_add_(0, idx, -torch.log(lik))
        out = lik.float().cpu(), nll.float().cpu()
    return out


def scorer_arm(scorer, nodes, edges):
    out = scorer.score(nodes, edges)
    return out.likelihoods.cpu(), out.nll.cpu()


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def workload(name, net, nodes, edges, B, repeats, gpu):
    import torch
    from graphinvent_b200.graphed import RouteScorer
    scorer = RouteScorer(net, B, n_atom_types=5, n_formal_charge=3)
    arms = {"eager": lambda: eager(net, nodes, edges, [5, 3], B), "scorer": lambda: scorer_arm(scorer, nodes, edges)}
    res = {k: fn() for k, fn in arms.items()}                          # warm-up
    S = res["scorer"][0].numel()
    assert res["eager"][0].numel() == S
    dlogp = (torch.log(res["eager"][0].double()) - torch.log(res["scorer"][0].double())).abs().max().item()
    times = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            times[k].append(timed(fn)[0])
    rec = dict(workload=name, molecules=int(nodes.shape[0]), states=S, batch=B, repeats=repeats, gpu=gpu,
               max_abs_dlogp=dlogp)
    for k, ts in times.items():
        t = statistics.median(ts)
        rec[k] = dict(seconds=t, molecules_per_s=nodes.shape[0] / t, states_per_s=S / t)
    rec["speedup"] = rec["eager"]["seconds"] / rec["scorer"]["seconds"]
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", help="also write the JSON lines here")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_route_nll.py needs a CUDA device")
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    from tests.conftest import pretrained_path
    gpu = card()
    recs = []
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    path = pretrained_path()
    if path is None:
        raise SystemExit("oracle/_ref/pretrained_model.pth is missing: run __graft_entry__.build() first")
    net = mpnn.create(make_constants("GGNN"))
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    recs.append(workload("gdb13_1K/train, pretrained GGNN", net.cuda().eval(), z["gdb13_1K_train/nodes"],
                         z["gdb13_1K_train/edges"], a.batch, a.repeats, gpu))
    C = make_constants("GGNN", max_n_nodes=38)
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(O.make_constants("GGNN", max_n_nodes=38), seed=0))
    nodes, edges = S.random_graphs(a.synthetic, 38, 5, 3, seed=38, min_atoms=1)
    recs.append(workload(f"synthetic N=38 x {a.synthetic}, seeded GGNN", net.cuda().eval(), nodes, edges, a.batch,
                         a.repeats, gpu))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in recs)


if __name__ == "__main__":
    main()
