"""Valid-actions-only sampling: the captured generator with the action mask off, "structure" and "valence".

    python tools/bench_action_mask.py [--batches 6] [--repeats 3]

Models: the reference's pretrained gdb13 GGNN (oracle/_ref/pretrained_model.pth, installed by
`__graft_entry__.build()`) and an EMN with seeded initial weights (`oracle.mpnn_oracle.init_state_dict`, seed 5), at
batch 1000 and 100.  The valence table is the package default for gdb13's C, N, O, S, Cl x charges -1, 0, +1.

The three configurations alternate batch by batch in one process on the same weights, so that clock and power drift
hit them alike; each batch is timed with CUDA events around `build_graphs`, and molecules/s is the median over
`--repeats` repeats of `--batches` batches.  Reported per configuration: molecules/s, rounds per batch, mean atoms,
the fraction of molecules properly terminated and the fraction within the valence table (every atom's bond orders
within its limit, computed in numpy on the returned tensors; off and "structure" are scored against the same table).
A batch that reaches the 2N-round limit is counted, not timed.  `mask_ms_per_round` times `gib_action_mask_logits`
alone over 200 launches on a batch's state and logits.  One JSON line per (model, batch), with the card name, power
limit and SM clock read from nvidia-smi.  A last line times `graphed.RouteScorer.score` on gdb13_1K/train with the
pretrained GGNN, batch 1000, mask off / "structure" / "valence" (median of 3 alternating calls each, end to end from
device int8 stacks; molecules over the valence table, which the valence scorer refuses, are left out of every arm).
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
from bench_generation import gpu_info   # noqa: E402

GDB13_ATOMS, GDB13_CHARGES = ["C", "N", "O", "S", "Cl"], [-1, 0, 1]


def models(dev):
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    out = {}
    path = os.path.join(ROOT, "oracle", "_ref", "pretrained_model.pth")
    if os.path.exists(path):
        net = mpnn.create(make_constants("GGNN"))
        net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
        out["GGNN_pretrained"] = net.to(dev).eval()
    C = make_constants("EMN")
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(O.make_constants("EMN"), seed=5))
    out["EMN_seeded"] = net.to(dev).eval()
    return out


def within_table(nodes, edges, n_nodes, V, order):
    """fraction of molecules whose every atom is within its valence limit (half-bond units)"""
    nodes, edges, n = nodes.cpu().numpy(), edges.cpu().numpy(), n_nodes.cpu().numpy().astype(np.int64)
    used = (edges * np.asarray(order)).sum((2, 3))                       # [B, N]
    t, q = nodes[..., :5].argmax(-1), nodes[..., 5:8].argmax(-1)
    limit = 2 * V[t, q]
    live = np.arange(nodes.shape[1])[None] < n[:, None]
    return float(((used <= limit) | ~live).all(1).mean())


def route_arm(net, V, order, dev, repeats=3):
    """RouteScorer on gdb13_1K/train with the mask off / "structure" / "valence", calls alternating, median ms per
    call; molecules over the valence table (the valence scorer refuses them) are left out of every arm"""
    from graphinvent_b200.graphed import RouteScorer
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]
    n = (nodes != 0).any(-1).sum(-1)
    keep = np.array([within_table(torch.from_numpy(nodes[m:m + 1]), torch.from_numpy(edges[m:m + 1]),
                                  torch.from_numpy(n[m:m + 1]), V, order) == 1.0 for m in range(nodes.shape[0])])
    nodes, edges = torch.from_numpy(nodes[keep]).to(dev), torch.from_numpy(edges[keep]).to(dev)
    kw = dict(batch_size=1000, n_atom_types=5, n_formal_charge=3)
    arms = {"off": RouteScorer(net, **kw), "structure": RouteScorer(net, action_mask="structure", **kw),
            "valence": RouteScorer(net, action_mask="valence", max_valence=V, **kw)}
    ms = {k: [] for k in arms}
    for k, sc in arms.items():                      # warm-up (the capture)
        sc.score(nodes, edges)
    for _ in range(repeats):
        for k, sc in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = sc.score(nodes, edges)
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    states = int(out.offsets[-1])
    return {"molecules": int(nodes.shape[0]), "left_out_over_table": int((~keep).sum()), "states": states,
            "ms_per_call": {k: float(np.median(v)) for k, v in ms.items()}, "runs_ms": ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=6, help="timed batches per configuration and repeat")
    ap.add_argument("--repeats", type=int, default=3, help="repeats; molecules/s is their median")
    ap.add_argument("--sizes", default="1000,100")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from graphinvent_b200.config import action_rule_table
    from graphinvent_b200.graphed import GraphedGenerator
    consts = namedtuple("C", "atom_types formal_charge")(GDB13_ATOMS, GDB13_CHARGES)
    V, order, _ = action_rule_table(5, 3, 3, 0, None, consts)
    info = gpu_info(0)
    for mname, net in models(dev).items():
        for B in (int(s) for s in args.sizes.split(",")):
            kw = dict(batch_size=B, n_atom_types=5, n_formal_charge=3, device=dev)
            gens = {"off": GraphedGenerator(net, **kw),
                    "structure": GraphedGenerator(net, action_mask="structure", **kw),
                    "valence": GraphedGenerator(net, action_mask="valence", max_valence=V, **kw)}
            rngs = {name: torch.Generator(device=dev).manual_seed(2000 + 10 * i) for i, name in enumerate(gens)}
            for name, gen in gens.items():                   # warm-up batch (the capture)
                try:
                    gen.build_graphs(generator=rngs[name])
                except RuntimeError:
                    pass
            torch.cuda.synchronize()
            runs = {name: [] for name in gens}
            acc = {name: dict(batches=0, rounds=0, atoms=0.0, proper=0.0, valid=0.0, limit=0) for name in gens}
            for _ in range(args.repeats):
                timed = {name: [] for name in gens}
                for _ in range(args.batches):
                    for name, gen in gens.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        try:
                            gen.build_graphs(generator=rngs[name])
                        except RuntimeError:
                            acc[name]["limit"] += 1
                            continue
                        e1.record()
                        timed[name].append((e0, e1))
                        a = acc[name]
                        a["batches"] += 1
                        a["rounds"] += gen.rounds
                        a["atoms"] += float(gen.generated_n_nodes[:B].float().mean())
                        a["proper"] += float(gen.properly_terminated[:B].float().mean())
                        a["valid"] += within_table(gen.generated_nodes[:B], gen.generated_edges[:B],
                                                   gen.generated_n_nodes[:B], V, order)
                torch.cuda.synchronize()
                for name in gens:
                    ms = sum(a.elapsed_time(b) for a, b in timed[name])
                    runs[name].append(len(timed[name]) * B / (ms / 1e3) if ms else float("nan"))
            res = {}
            for name in gens:
                a = acc[name]
                k = max(a["batches"], 1)
                res[name] = {"molecules_per_s": float(np.median(runs[name])), "runs": runs[name],
                             "batches": a["batches"], "round_limit_batches": a["limit"],
                             "rounds_per_batch": a["rounds"] / k, "mean_atoms": a["atoms"] / k,
                             "fraction_properly_terminated": a["proper"] / k, "fraction_within_valence_table":
                             a["valid"] / k}
            # the mask kernel alone, on the valence generator's last state and logits
            g = gens["valence"]
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            timings = {}
            for name in ("structure", "valence"):
                m = gens[name].action_mask
                logits = g.logits.clone()
                reps = 200
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    m.apply(B, logits, g.n_nodes, st, g.nodes, g.edges)
                e1.record()
                torch.cuda.synchronize()
                timings[name] = e0.elapsed_time(e1) / reps
            off = res["off"]["molecules_per_s"]
            line = {"metric": f"valid-actions-only generation molecules/s ({mname}, batch {B}, captured rounds)",
                    "value": res["valence"]["molecules_per_s"], "unit": "molecules/s", "impls": res,
                    "mask_ms_per_round": timings,
                    "over_off": {k: v["molecules_per_s"] / off for k, v in res.items()} if off else None,
                    "gpu": info}
            print(json.dumps(line), flush=True)
    nets = models(dev)
    if "GGNN_pretrained" in nets:
        print(json.dumps({"metric": "RouteScorer ms per call, gdb13_1K/train, pretrained GGNN, batch 1000",
                          "route_scorer": route_arm(nets["GGNN_pretrained"], V, order, dev), "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
