"""One RL fine-tuning step (`Workflow.learning_step`, Workflow.py:569-612): rollout (agent, prior), rollout (BASF,
agent), the reference's loss on both, one backward, one FlatAdam step -- eager `generation.GraphGeneratorRL` against
captured rounds with a recomputing backward (`graphed.GraphedGeneratorRL`).

    python tools/bench_rl.py [--models GGNN,EMN] [--batches 1000,100] [--steps 3] [--warmup 1]

The RDKit scoring between the rollouts and the loss stays on the host in the reference; here the scores are a fixed
seeded vector (sigma 20, the reference default), so the step is the device work only.  Weights: the seeded recipe of
tools/bench_generation.py (a random-init EMN ends every rollout in round 1); the prior and the BASF model are copies
of the agent, and none is frozen (the reference freezes neither), so the backward runs for all three.

Per (model, batch, implementation): mean ms per learning step over `--steps` timed steps (CUDA events around each
whole step), molecules/s (2 x batch finished molecules per step), rounds per rollout, and
torch.cuda.max_memory_allocated over the timed steps (with what was allocated when that step started: both
implementations' models and static buffers live in the process).  Eager and captured steps alternate in one process.  An eager
step that runs out of device memory is recorded as {"oom": ...}, not retried.  One JSON line, with the card's name,
power limit and SM clock read from nvidia-smi in the same call.
"""
import argparse
import copy
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SIGMA = 20.0


def learning_step(gen, agent, prior, basf, opt, scores, **kw):
    """Workflow.learning_step's device part: two rollouts, compute_loss_component on each (Workflow.py:889-896)"""
    _, agent_ll, prior_ll, _ = gen.sample(agent, prior, **kw)
    _, basf_ll, agent_ll2, _ = gen.sample(basf, agent, **kw)
    loss = torch.mean((agent_ll - (prior_ll + SIGMA * scores)) ** 2)
    loss = loss + torch.mean((agent_ll2 - (basf_ll + SIGMA * scores)) ** 2)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
    return gen.rounds


def run(model_name, B, steps, warmup, train_steps, dev):
    from bench_generation import train_weights
    from graphinvent_b200.generation import GraphGeneratorRL
    from graphinvent_b200.graphed import GraphedGeneratorRL
    from graphinvent_b200.optim import FlatAdam
    gc.collect()                                   # the previous configuration's generators and graphs
    torch.cuda.empty_cache()
    C, net, _ = train_weights(model_name, train_steps, dev)
    g = torch.Generator(device=dev).manual_seed(5)
    scores = torch.rand(B, generator=g, device=dev)
    out = {}
    state = {}
    for name, cls in (("eager", GraphGeneratorRL), ("graphed", GraphedGeneratorRL)):
        agent = copy.deepcopy(net).train()
        prior, basf = copy.deepcopy(net), copy.deepcopy(net)
        opt = FlatAdam(agent.parameters(), lr=1e-5)
        gen = cls(agent, B, n_atom_types=5, n_formal_charge=3, device=dev)
        state[name] = dict(gen=gen, agent=agent, prior=prior, basf=basf, opt=opt,
                           rng=torch.Generator(device=dev).manual_seed(11), ms=[], rounds=[], peak=0, base=0, oom=None)
    order = list(state)
    for i in range(warmup + steps):
        for name in order:
            s = state[name]
            if s["oom"]:
                continue
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            try:
                e0.record()
                r = learning_step(s["gen"], s["agent"], s["prior"], s["basf"], s["opt"], scores, generator=s["rng"])
                e1.record()
                torch.cuda.synchronize()
            except torch.cuda.OutOfMemoryError as ex:
                s["oom"] = str(ex).splitlines()[0][:200]
                torch.cuda.empty_cache()
                continue
            except RuntimeError as ex:             # e.g. a rollout past the 2N-round limit: recorded, not retried
                s["oom"] = "error: " + str(ex)[:200]
                continue
            if i >= warmup:
                s["ms"].append(e0.elapsed_time(e1))
                s["rounds"].append(r)
                if torch.cuda.max_memory_allocated(dev) > s["peak"]:
                    s["peak"], s["base"] = torch.cuda.max_memory_allocated(dev), base
    for name in order:
        s = state[name]
        if s["oom"] and not s["ms"]:
            out[name] = {"oom" if "memory" in s["oom"] else "failed": s["oom"]}
            continue
        ms = sum(s["ms"]) / len(s["ms"])
        out[name] = {"ms_per_step": ms, "ms_each": [round(x, 2) for x in s["ms"]], "molecules_per_s": 2 * B / (ms / 1e3),
                     "rounds_last_rollout": s["rounds"], "max_memory_allocated_GiB": s["peak"] / 2**30,
                     "allocated_at_step_start_GiB": s["base"] / 2**30}
        if s["oom"]:
            out[name]["stopped_by"] = s["oom"]
        if name == "graphed":
            out[name]["workspace_GiB"] = s["gen"].workspace_bytes / 2**30
        del s["gen"]
        torch.cuda.empty_cache()
    if "ms_per_step" in out.get("eager", {}) and "ms_per_step" in out.get("graphed", {}):
        out["graphed_over_eager"] = out["eager"]["ms_per_step"] / out["graphed"]["ms_per_step"]
    return out


def main():
    from bench_generation import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="GGNN,EMN")
    ap.add_argument("--batches", default="1000,100")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--train-steps", type=int, default=300)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rl.py measures on a CUDA device; none found")
    dev = torch.device("cuda", 0)
    results = {}
    for m in args.models.split(","):
        for B in (int(x) for x in args.batches.split(",")):
            results[f"{m}/B={B}"] = run(m, B, args.steps, args.warmup, args.train_steps, dev)
    print(json.dumps({"metric": "RL learning step (two rollouts + loss + backward + FlatAdam)", "results": results,
                      "gpu": gpu_info(0), "steps": args.steps, "warmup": args.warmup}), flush=True)


if __name__ == "__main__":
    main()
