"""The validation pass of a training run (`Workflow.validation_epoch`, Workflow.py:800-831, and
`Analyzer.get_validation_likelihood`, Analyzer.py:708-778) -- the eager loop against captured replays
(`graphed.EvalStep` sharing a `graphed.TrainStep`) -- and one TrainStep replay on a short batch against a full one.

    python tools/bench_eval.py [--models GGNN,EMN] [--batch 1000] [--batches 50] [--repeats 3]

Eager: the module API in exact mode on each batch, `functional.kl_loss` into the epoch's slot tensor, then
`functional.validation_nll` with the reference's list logic (NaN removal, writes at idx * batch_size, n_structures).
Captured: `EvalStep.validation_epoch` and `EvalStep.validation_likelihood` with `share=` a TrainStep of the same dims,
as a training run would hold one.  Both run on the same seeded synthetic batches (gdb13 dims, `--batches` batches of
`--batch` molecules, already on the device), `n_samples` large enough that every batch is evaluated.  The two
implementations alternate, `--repeats` times after one warm-up pass each.

Reported per model: ms per batch of each pass (CUDA events around the whole pass, host loop included),
torch.cuda.max_memory_allocated during the pass and what was allocated when it started, the largest difference of the
two implementations' results, and ms per TrainStep replay (FlatAdam step included) on a full batch and on a batch of
batch / 2 molecules.  One JSON line, with the card's name, power limit and SM clock read from nvidia-smi in the same
call.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def make_batches(C, B, n_batches, dev):
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    out = []
    for k in range(n_batches):
        n, e = S.random_graphs(B, C.max_n_nodes, 5, 3, n_edge_features=C.n_edge_features, seed=1000 + k, min_atoms=0)
        t = S.random_targets(B, apd_length(C), seed=2000 + k)
        out.append(tuple(torch.from_numpy(x).float().to(dev) for x in (n, e, t)))
    return out


def eager_validation_epoch(net, loader):
    """Workflow.py:813-831 on the module API"""
    from graphinvent_b200 import functional as Fn
    slots = torch.zeros(len(loader), device=loader[0][0].device)
    with torch.no_grad():
        for i, (n, e, t) in enumerate(loader):
            slots[i] = Fn.kl_loss(net(n, e), t)
    return torch.mean(slots)


def eager_validation_likelihood(net, loader, n_samples, B, N):
    """Analyzer.py:734-778 on the module API"""
    from graphinvent_b200 import functional as Fn
    n = min(100000, n_samples)
    dev = loader[0][0].device
    lik = torch.zeros(n * (N + 5), device=dev)
    n_structures = torch.zeros(1, device=dev)
    with torch.no_grad():
        for idx, (nodes, edges, t) in enumerate(loader):
            if idx * B > n:
                break
            v = Fn.validation_nll(net(nodes, edges), t)
            v = v[~torch.isnan(v)]
            lik[idx * B: idx * B + len(v)] = v
            n_structures += torch.sum(t[:, -1]).unsqueeze(dim=0)
    return lik, torch.sum(lik, dim=0) / n_structures[0]


def timed(fn, dev):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    return res, e0.elapsed_time(e1), torch.cuda.max_memory_allocated(dev), base


def run(model_name, B, n_batches, repeats, dev):
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import EvalStep, TrainStep
    from graphinvent_b200.optim import FlatAdam
    from oracle import mpnn_oracle as O
    C = O.make_constants(model_name)
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=0))
    net = net.to(dev)
    loader = make_batches(C, B, n_batches, dev)
    by_type = model_name != "EMN"
    entries = max(int((e != 0).sum()) if by_type else int((e != 0).any(-1).sum()) for _, e, _ in loader)
    cap = int(entries * 1.05) + 256
    opt = FlatAdam(net.parameters(), lr=1e-5)
    step = TrainStep(net, opt, batch_size=B, entry_capacity=cap)
    ev = EvalStep(net, batch_size=B, entry_capacity=cap, share=step)
    n_samples = n_batches * B
    N = C.max_n_nodes
    net.eval()
    passes = {
        "eager": (lambda: eager_validation_epoch(net, loader),
                  lambda: eager_validation_likelihood(net, loader, n_samples, B, N)),
        "graphed": (lambda: ev.validation_epoch(loader), lambda: ev.validation_likelihood(loader, n_samples)),
    }
    rec = {name: {"epoch_ms": [], "likelihood_ms": [], "epoch_peak": 0, "likelihood_peak": 0, "epoch_base": 0,
                  "likelihood_base": 0} for name in passes}
    results = {}
    for i in range(1 + repeats):
        for name, (epoch, likelihood) in passes.items():
            for which, fn in (("epoch", epoch), ("likelihood", likelihood)):
                res, ms, peak, base = timed(fn, dev)
                results[(name, which)] = res
                if i > 0:
                    r = rec[name]
                    r[f"{which}_ms"].append(ms)
                    if peak > r[f"{which}_peak"]:
                        r[f"{which}_peak"], r[f"{which}_base"] = peak, base
    ev.check()
    out = {}
    for name, r in rec.items():
        out[name] = {f"{w}_ms_per_batch": float(np.mean(r[f"{w}_ms"])) / n_batches for w in ("epoch", "likelihood")}
        for w in ("epoch", "likelihood"):
            out[name][f"{w}_ms_each_pass"] = [round(x, 2) for x in r[f"{w}_ms"]]
            out[name][f"{w}_max_memory_allocated_GiB"] = r[f"{w}_peak"] / 2**30
            out[name][f"{w}_allocated_at_start_GiB"] = r[f"{w}_base"] / 2**30
    for w in ("epoch", "likelihood"):
        out[f"{w}_graphed_over_eager"] = out["eager"][f"{w}_ms_per_batch"] / out["graphed"][f"{w}_ms_per_batch"]
    ve, vg = results[("eager", "epoch")], results[("graphed", "epoch")]
    (le, ae), (lg, ag) = results[("eager", "likelihood")], results[("graphed", "likelihood")]
    out["max_diff"] = {"validation_loss": abs(float(ve) - float(vg)), "likelihoods": float((le - lg).abs().max()),
                       "avg_final_likelihood": abs(float(ae) - float(ag))}
    out["train_step_workspace_GiB"] = step.workspace_bytes / 2**30
    # one TrainStep replay on a short batch against a full one (the graph runs all B rows either way)
    net.train()
    half = tuple(x[:B // 2] for x in loader[0])
    ms = {"full": [], "half": []}
    for i in range(2 + 5):
        for name, batch in (("full", loader[1]), ("half", half)):
            _, t, _, _ = timed(lambda: step(*batch), dev)
            if i >= 2:
                ms[name].append(t)
    step.check()
    out["train_step_ms"] = {"full_batch": float(np.mean(ms["full"])), f"batch_of_{B // 2}": float(np.mean(ms["half"]))}
    return out


def main():
    from bench_generation import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="GGNN,EMN")
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--batches", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a CUDA device; none found")
    dev = torch.device("cuda", 0)
    results = {m: run(m, args.batch, args.batches, args.repeats, dev) for m in args.models.split(",")}
    print(json.dumps({"metric": "validation pass (validation_epoch + get_validation_likelihood), eager vs captured",
                      "results": results, "gpu": gpu_info(0), "batch": args.batch, "batches": args.batches,
                      "repeats": args.repeats}), flush=True)


if __name__ == "__main__":
    main()
