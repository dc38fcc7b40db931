"""Scaffold decoration throughput: captured rounds that grow each molecule from a gdb13 scaffold, with and without
attachment points, against the unconstrained captured generator and the eager scaffold generator.

    python tools/bench_scaffold_generation.py [--model EMN] [--batch 1000] [--batches 10] [--repeats 5]

Weights: the seeded recipe of tools/bench_generation.py (`--train-steps` full-batch Adam steps on the 256 recorded
gdb13_1K rows).  Scaffolds: decoding-route states of those rows, one per atom count 1..12 (12 = max_n_nodes - 1),
and a seeded choice of attachment points per scaffold (the last atom and about a third of the others).

The configurations alternate batch by batch in one process with the same weights, so that clock and power drift hit
them alike; each batch is timed with CUDA events around its `build_graphs` call, and molecules/s is the median over
`--repeats` repeats of `--batches` batches per configuration (`runs` lists every repeat).  A batch that reaches the
2N-round limit raises in every generator and is counted, not timed.  `mask_ms_per_round` times `gib_generation_mask_logits`
on its own over a batch of logits, the extra work a masked round does.  One JSON line, with the card name, power limit
and SM clock read from nvidia-smi.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_generation import gpu_info, train_weights   # noqa: E402


def gdb13_scaffolds(seed=0):
    from graphinvent_b200 import data
    nodes, edges, _ = data.read_hdf5_raw(os.path.join(ROOT, "tests", "golden", "gdb13_train_head256.h5"),
                                         13, 8, 3, 625)
    k = (nodes != 0).any(-1).sum(-1)
    rows = [int(np.flatnonzero(k == s)[0]) for s in range(1, 13)]
    rng = np.random.default_rng(seed)
    att = [sorted({int(n - 1)} | {int(i) for i in np.flatnonzero(rng.random(n) < 0.3)}) for n in k[rows]]
    return (nodes[rows].copy(), edges[rows].copy()), att


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="EMN", choices=["EMN", "GGNN", "MNN", "AttGGNN"])
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--batches", type=int, default=10, help="timed batches per configuration and repeat")
    ap.add_argument("--repeats", type=int, default=5, help="repeats; molecules/s is their median")
    ap.add_argument("--train-steps", type=int, default=300)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from graphinvent_b200._lib import check, lib
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import GraphedGenerator
    C, net, train_loss = train_weights(args.model, args.train_steps, dev)
    sc, att = gdb13_scaffolds()
    B = args.batch
    kw = dict(batch_size=B, n_atom_types=5, n_formal_charge=3, device=dev)
    gens = {"graphed_plain": GraphedGenerator(net, **kw),
            "graphed_scaffolds": GraphedGenerator(net, scaffolds=sc, **kw),
            "graphed_scaffolds_attachment": GraphedGenerator(net, scaffolds=sc, attachment=att, **kw),
            "eager_scaffolds": GraphGenerator(net, scaffolds=sc, **kw),
            "eager_scaffolds_attachment": GraphGenerator(net, scaffolds=sc, attachment=att, **kw)}
    rngs = {name: torch.Generator(device=dev).manual_seed(1000 + 100 * i) for i, name in enumerate(gens)}
    for name, gen in gens.items():                 # warm-up batch (graphed: the capture)
        try:
            gen.build_graphs(generator=rngs[name])
        except RuntimeError:
            pass
    torch.cuda.synchronize()
    runs = {name: [] for name in gens}                    # molecules/s of each repeat
    acc = {name: [0, 0, 0.0, 0] for name in gens}       # batches, rounds, atoms, round-limit batches
    for _ in range(args.repeats):
        timed = {name: [] for name in gens}
        for _ in range(args.batches):
            for name, gen in gens.items():
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                try:
                    gen.build_graphs(generator=rngs[name])
                except RuntimeError:
                    acc[name][3] += 1
                    continue
                ev1.record()
                timed[name].append((ev0, ev1))
                a = acc[name]
                a[0] += 1
                a[1] += gen.rounds
                a[2] += float(gen.generated_n_nodes[:B].float().sum())
        torch.cuda.synchronize()
        for name in gens:
            ms = sum(e0.elapsed_time(e1) for e0, e1 in timed[name])
            runs[name].append(len(timed[name]) * B / (ms / 1e3) if ms else float("nan"))
    results = {}
    for name in gens:
        batches, rounds, atoms, limit = acc[name]
        results[name] = {"molecules_per_s": float(np.median(runs[name])), "runs": runs[name], "batches": batches,
                         "round_limit_batches": limit, "rounds_per_batch": rounds / batches if batches else None,
                         "mean_atoms": atoms / (batches * B) if batches else None}
    # the mask kernel on its own, on the masked captured generator's state and logits
    g = gens["graphed_scaffolds_attachment"]
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    sc_struct = g._sc
    reps = 200
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(reps):
        check(lib.gib_generation_mask_logits(B, g.N, g.Ef, g.apd, ctypes.byref(sc_struct),
                                             ctypes.c_void_p(g._slot_ids.data_ptr()),
                                             ctypes.c_void_p(g.n_nodes.data_ptr()), None, None, None,
                                             ctypes.c_void_p(g.logits.data_ptr()), st), "gib_generation_mask_logits")
    ev1.record()
    torch.cuda.synchronize()
    plain = results["graphed_plain"]["molecules_per_s"]
    line = {"metric": f"scaffold decoration molecules/s ({args.model}, batch {B}, captured rounds)",
            "value": results["graphed_scaffolds_attachment"]["molecules_per_s"], "unit": "molecules/s",
            "impls": results, "mask_ms_per_round": ev0.elapsed_time(ev1) / reps,
            "scaffolds": {"S": int(sc[0].shape[0]), "atoms": list(range(1, 13))},
            "weights": f"seeded recipe: {args.train_steps} Adam steps on 256 gdb13 rows, final loss {train_loss:.4f}",
            "gpu": gpu_info(0)}
    if plain:
        line["scaffolds_over_plain"] = {k: (v["molecules_per_s"] / plain if v["molecules_per_s"] else None)
                                        for k, v in results.items()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
