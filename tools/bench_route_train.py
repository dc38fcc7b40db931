"""Fine-tuning on decoding-route likelihoods: one step of `graphed.RouteScorer.score(..., requires_grad=True)` +
backward + FlatAdam against the eager way of computing it without the scorer.

    python tools/bench_route_train.py [--repeats 5] [--synthetic 250] [--batch 1000]

One step is the loss mean(nll) over the molecules, its backward into the model's parameters and one FlatAdam step.
Eager arm: each molecule's route states built with numpy (tests/preprocess_reference.route, reversed into build
order), batched through `model(nodes, edges)` in float32 with autograd, log-softmax gathered at the route actions,
the per-molecule sums, backward, FlatAdam.  Scorer arm: score from the same host int8 stacks, backward (one
recomputed forward per batch of states), FlatAdam.  Each arm trains its own copy of the model from the same weights
with a zero learning rate, so every step sees the same parameters.  Both are timed end to end by the host clock around
work that ends in a device synchronise; one warm-up step each, then the median of --repeats steps, the arms
alternating.  Peak allocated memory is taken per arm over one step, from the state after the warm-up.

Workloads: gdb13_1K/train (979 molecules, tests/golden/preprocess_gdb13.npz) with the reference's pretrained GGNN
(oracle/_ref/pretrained_model.pth), and --synthetic molecules of up to 38 atoms (graphinvent_b200.synthetic) with a
seeded GGNN of max_n_nodes 38.  Reported per arm: ms per step, route states per second and peak allocated GiB (the
step's peak above what was allocated before it, plus the scorer's resident buffers), with the largest gradient
difference between the arms over the largest gradient element, and the card's name and power limit.  An eager arm
that runs out of memory is reported as such.  One JSON line per workload.
"""
import argparse
import copy
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_route_nll import card, timed  # noqa: E402


def eager_step(net, opt, states, B):
    import torch
    X, E, acts, offsets = states
    opt.zero_grad()
    M = len(offsets) - 1
    off = torch.from_numpy(offsets).cuda()
    idx = torch.repeat_interleave(torch.arange(M, device="cuda"), off[1:] - off[:-1])
    logp = []
    for s in range(0, X.shape[0], B):
        x = torch.from_numpy(X[s:s + B]).cuda().float()
        e = torch.from_numpy(E[s:s + B]).cuda().float()
        a = torch.from_numpy(acts[s:s + B]).cuda().view(-1, 1)
        logp.append(torch.log_softmax(net(x, e), dim=1).gather(1, a).view(-1))
    nll = torch.zeros(M, device="cuda").index_add(0, idx, -torch.cat(logp))
    loss = nll.mean()
    loss.backward()
    opt.step()
    return loss.detach()


def scorer_step(scorer, opt, nodes, edges):
    opt.zero_grad()
    loss = scorer.score(nodes, edges, requires_grad=True).nll.mean()
    loss.backward()
    opt.step()
    return loss.detach()


def peak_of(fn, resident=0):
    """GiB: the peak allocated during one step above what was allocated before it, plus `resident` bytes the arm
    keeps between steps (the scorer's static and backward buffers)"""
    import torch
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base + resident) / 2**30


def resident_bytes(scorer):
    import torch
    return sum(t.numel() * t.element_size() for o in (scorer, scorer._bwd) for t in vars(o).values()
               if isinstance(t, torch.Tensor) and t.is_cuda and t._base is None)


def workload(name, net, nodes, edges, B, repeats, gpu):
    import torch
    from graphinvent_b200.graphed import RouteScorer
    from graphinvent_b200.optim import FlatAdam
    from tests import route_nll_reference as R
    nets = {"eager": copy.deepcopy(net), "scorer": copy.deepcopy(net)}
    opts = {k: FlatAdam(m.parameters(), lr=0.0) for k, m in nets.items()}
    scorer = RouteScorer(nets["scorer"], B, n_atom_types=5, n_formal_charge=3)

    def eager():
        states = R.build_order_states(nodes, edges, [5, 3])       # the route states are part of the eager step
        return eager_step(nets["eager"], opts["eager"], states, B)

    arms = {"scorer": lambda: scorer_step(scorer, opts["scorer"], nodes, edges), "eager": eager}
    rec = dict(workload=name, molecules=int(nodes.shape[0]), batch=B, repeats=repeats, gpu=gpu, loss={})
    for k in list(arms):                                              # warm-up
        try:
            rec["loss"][k] = float(arms[k]())
        except torch.cuda.OutOfMemoryError as e:                      # the eager arm's activations did not fit
            rec[k] = dict(error=f"out of memory: {str(e).splitlines()[0]}")
            nets[k].zero_grad(set_to_none=True)
            del arms[k]
            torch.cuda.empty_cache()
    rec["states"] = S = int(scorer.score(nodes, edges).likelihoods.numel())
    if "eager" in arms:
        grads = {k: torch.cat([p.grad.reshape(-1) for p in m.parameters()]) for k, m in nets.items()}
        rec["max_grad_diff_over_max_grad"] = ((grads["eager"] - grads["scorer"]).abs().max()
                                              / grads["eager"].abs().max()).item()
    peaks = {k: peak_of(fn, resident_bytes(scorer) if k == "scorer" else 0) for k, fn in arms.items()}
    times = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            times[k].append(timed(fn)[0])
    for k, ts in times.items():
        t = statistics.median(ts)
        rec[k] = dict(ms_per_step=1e3 * t, states_per_s=S / t, peak_allocated_gib=peaks[k])
    if "eager" in arms:
        rec["speedup"] = rec["eager"]["ms_per_step"] / rec["scorer"]["ms_per_step"]
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=250)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", help="also write the JSON lines here")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_route_train.py needs a CUDA device")
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
