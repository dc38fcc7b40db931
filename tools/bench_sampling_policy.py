"""Temperature / top-k / top-p sampling: the policy sampler's launch time and captured generation under a grid of
policies.

    python tools/bench_sampling_policy.py [--batches 3] [--repeats 3] [--launches 500]

Kernel: `gib_sample_actions` (today's sampler) and `gib_sample_actions_policy` under five policies -- off (1, 0, 1), T
only (0.7, 0, 1), top-k (1, 10, 1), top-p (1, 0, 0.9) and all three (0.7, 10, 0.9) -- on seeded N(0, 2) logits with
20 % -inf at batch 1000, apd 625 (gdb13) and 16411 (a long row, read from L2): CUDA events around `--launches`
back-to-back launches, ms per launch.

Generation: `GraphedGenerator` at batch 1000 with the reference's pretrained gdb13 GGNN (oracle/_ref/pretrained_model.pth,
installed by `__graft_entry__.build()`) and an EMN with seeded initial weights (`oracle.mpnn_oracle.init_state_dict`,
seed 5).  One generator built without a policy (today's round, "plain") and one built with a policy whose
`set_sampling` steps through T in {0.7, 1.0, 1.3} x top_p in {0.9, 1.0} x top_k in {0, 10} batch by batch (one captured
round for all twelve), so clock and power drift hit every configuration alike.  Each batch is timed with CUDA events
around `build_graphs`; molecules/s is the median over `--repeats` repeats of `--batches` batches.  Reported per
configuration: molecules/s, rounds per batch, mean atoms, the fraction properly terminated and the fraction within
the package's gdb13 valence table.  `round_ms` is the plain generator's batch time over its rounds and
`policy_share_of_round` the all-three kernel time over it.  One JSON line per model and one for the kernel, with the
card name, power limit and SM clock read from nvidia-smi.
"""
import argparse
import ctypes
import json
import os
import sys
from collections import namedtuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_action_mask import GDB13_ATOMS, GDB13_CHARGES, models, within_table   # noqa: E402
from bench_generation import gpu_info   # noqa: E402

KERNEL_POLICIES = {"off": (1.0, 0, 1.0), "T": (0.7, 0, 1.0), "top_k": (1.0, 10, 1.0), "top_p": (1.0, 0, 0.9),
                   "all": (0.7, 10, 0.9)}


def kernel_times(dev, B, apd, launches):
    """ms per launch of today's sampler and of the policy sampler under each KERNEL_POLICIES entry"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import check, lib
    g = torch.Generator(device=dev).manual_seed(apd)
    x = 2 * torch.randn(B, apd, generator=g, device=dev)
    x[torch.rand(B, apd, generator=g, device=dev) < 0.2] = -float("inf")
    x[:, -1] = 0.0
    u = torch.rand(B, generator=g, device=dev)
    a = torch.empty(B, dtype=torch.int32, device=dev)
    lik = torch.empty(B, device=dev)
    pol = torch.zeros(4, dtype=torch.int32, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def plain():
        check(lib.gib_sample_actions(p(x), B, apd, p(u), p(a), p(lik), st), "gib_sample_actions")

    def policy():
        check(lib.gib_sample_actions_policy(p(x), B, apd, p(u), p(pol), p(a), p(lik), None, st),
              "gib_sample_actions_policy")

    def timed(fn):
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / launches

    out = {"plain": timed(plain)}
    for name, v in KERNEL_POLICIES.items():
        Fn.set_policy(pol, Fn.sampling_policy(*v))
        out[name] = timed(policy)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=3, help="timed batches per configuration and repeat")
    ap.add_argument("--repeats", type=int, default=3, help="repeats; molecules/s is their median")
    ap.add_argument("--launches", type=int, default=500, help="launches per kernel timing")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from graphinvent_b200.config import action_rule_table
    from graphinvent_b200.graphed import GraphedGenerator
    info = gpu_info(0)
    B = 1000
    kern = {apd: kernel_times(dev, B, apd, args.launches) for apd in (625, 16411)}
    print(json.dumps({"metric": "sampler ms per launch, batch 1000", "ms_per_launch": kern, "gpu": info}), flush=True)
    consts = namedtuple("C", "atom_types formal_charge")(GDB13_ATOMS, GDB13_CHARGES)
    V, order, _ = action_rule_table(5, 3, 3, 0, None, consts)
    grid = [(t, k, p) for t in (0.7, 1.0, 1.3) for p in (0.9, 1.0) for k in (0, 10)]
    for mname, net in models(dev).items():
        kw = dict(batch_size=B, n_atom_types=5, n_formal_charge=3, device=dev)
        plain = GraphedGenerator(net, **kw)
        pol = GraphedGenerator(net, temperature=0.7, top_k=10, top_p=0.9, **kw)
        arms = [("plain", None)] + [(f"T={t},k={k},p={p}", (t, k, p)) for t, k, p in grid]
        rng = torch.Generator(device=dev).manual_seed(3000)
        for gen in (plain, pol):                        # warm-up batch (the capture)
            try:
                gen.build_graphs(generator=rng)
            except RuntimeError:                        # the 2N-round limit: counted below, the round is captured
                pass
        graph = pol.graph
        runs = {name: [] for name, _ in arms}
        acc = {name: dict(batches=0, rounds=0, atoms=0.0, proper=0.0, valid=0.0, limit=0, ms=0.0) for name, _ in arms}
        for _ in range(args.repeats):
            timed = {name: [] for name, _ in arms}
            for _ in range(args.batches):
                for name, v in arms:
                    gen = plain if v is None else pol
                    if v is not None:
                        gen.set_sampling(*v)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    try:
                        gen.build_graphs(generator=rng)
                    except RuntimeError:
                        acc[name]["limit"] += 1
                        continue
                    e1.record()
                    timed[name].append((e0, e1, gen.rounds))
                    a = acc[name]
                    a["batches"] += 1
                    a["rounds"] += gen.rounds
                    a["atoms"] += float(gen.generated_n_nodes[:B].float().mean())
                    a["proper"] += float(gen.properly_terminated[:B].float().mean())
                    a["valid"] += within_table(gen.generated_nodes[:B], gen.generated_edges[:B],
                                               gen.generated_n_nodes[:B], V, order)
            torch.cuda.synchronize()
            for name, _ in arms:
                ms = sum(e0.elapsed_time(e1) for e0, e1, _ in timed[name])
                acc[name]["ms"] += ms
                runs[name].append(len(timed[name]) * B / (ms / 1e3) if ms else float("nan"))
        assert pol.graph is graph, "set_sampling recaptured the round"
        res = {}
        for name, _ in arms:
            a = acc[name]
            k = max(a["batches"], 1)
            res[name] = {"molecules_per_s": float(np.median(runs[name])), "runs": runs[name], "batches": a["batches"],
                         "round_limit_batches": a["limit"], "rounds_per_batch": a["rounds"] / k,
                         "mean_atoms": a["atoms"] / k, "fraction_properly_terminated": a["proper"] / k,
                         "fraction_within_valence_table": a["valid"] / k}
        round_ms = acc["plain"]["ms"] / max(acc["plain"]["rounds"], 1)     # plain batches all finish on these models
        print(json.dumps({"metric": f"policy-sampled generation molecules/s ({mname}, batch {B}, captured rounds)",
                          "value": res["T=1.0,k=0,p=1.0"]["molecules_per_s"], "unit": "molecules/s", "impls": res,
                          "round_ms": round_ms, "policy_share_of_round": kern[625]["all"] / round_ms,
                          "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
