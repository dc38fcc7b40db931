"""Generated batch -> reference `GenerationGraph`s + Analyzer statistics: the reference's per-atom path against one
device pass (graphinvent_b200.molecules).

    python tools/bench_molecules.py [--models GGNN,EMN] [--batch 1000] [--batches 10] [--ref-batches 2]

Batches of `--batch` molecules come from `graphed.GraphedGenerator` with the seeded weights recipe of
tools/bench_generation.py (`--train-steps` Adam steps on the 256 recorded gdb13 rows).  On each batch's CUDA tensors:

  reference   the unmodified reference's `graph_to_graph` for every molecule (GraphGenerator.py:659-804) and
              `Analyzer.get_molecular_properties` (Analyzer.py:311-599), loaded from oracle/_ref;
  device      `MoleculeBatch(...)`, `.generation_graphs()` and `.properties(...)`;
  end to end  `GraphedGenerator.sample_molecules()` + `.properties()` against `sample()` alone (the generation).

Both sides run with the same recording rdkit stub (tests/molecules_reference.py), so RDKit's own work is excluded from
both: the saving measured here is the device->host traffic and Python work around RDKit.  The saving including real
RDKit calls is not measured (RDKit is not installed on the measuring machine).  Times are host clocks around work that
ends in a device synchronise.  Device->host copies per batch are counted from torch.profiler memcpy records in a
separate run.  In a process that profiles several times the profiler can drop a run's memcpy records (one of the two
models has read 0 for the device path); tests/test_gpu_molecules.py asserts the device path's count exactly, in a
profiler run of its own.  One JSON line; the card's name, power limit and SM clock are read in the same call.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _d2h_copies(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "Memcpy DtoH" in e.name and e.device_type.name == "CUDA")


def _timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="GGNN,EMN")
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--batches", type=int, default=10, help="timed batches of the device path")
    ap.add_argument("--ref-batches", type=int, default=2, help="timed batches of the reference path")
    ap.add_argument("--train-steps", type=int, default=300)
    args = ap.parse_args()
    from graphinvent_b200.graphed import GraphedGenerator
    from graphinvent_b200.molecules import MoleculeBatch
    from tests import molecules_reference as R
    from tools.bench_generation import gpu_info, train_weights

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    RC = R.constants("L0", N=13, Ef=3, device="cuda")
    ref = R.load_reference(RC)
    if ref is None:
        raise SystemExit("oracle/_ref lacks the reference's MolecularGraph / GraphGenerator / Analyzer: run build()")
    R.set_constants(ref, RC)
    results = {}
    for model in args.models.split(","):
        C, net, loss = train_weights(model, args.train_steps, dev)
        gen = GraphedGenerator(net, batch_size=args.batch, n_atom_types=5, n_formal_charge=3, device=dev)
        rng = torch.Generator(device=dev).manual_seed(1000)
        batches = []
        for _ in range(max(args.batches, args.ref_batches)):
            (nodes, edges, n_nodes), _, _, term = gen.sample(generator=rng)
            batches.append((nodes, edges, n_nodes, term))

        def device_path(b):
            nodes, edges, n_nodes, term = b
            mb = MoleculeBatch(nodes, edges, n_nodes, RC)
            graphs = mb.generation_graphs()
            return mb.properties("Epoch 1", term, graphs)

        def reference_path(b):
            nodes, edges, n_nodes, term = b
            graphs, _ = R.reference_graphs(ref, nodes, edges, n_nodes)
            props, _ = R.reference_properties(ref, graphs, "Epoch 1", term)
            assert isinstance(props, dict), props
            return props

        device_path(batches[0])                                   # warm-up: module load, pinned allocations
        reference_path(batches[0])
        it = iter(batches)
        dev_ms = _timed(lambda: device_path(next(it)), args.batches)
        it = iter(batches)
        ref_ms = _timed(lambda: reference_path(next(it)), args.ref_batches)
        # same values: the device path's dict equals the reference's, bit for bit, on the first batch
        got, want = device_path(batches[0]), reference_path(batches[0])
        same = all(torch.equal(got[k], want[k]) if isinstance(want[k], torch.Tensor) else got[k] == want[k]
                   for k in want)
        gen_ms = _timed(lambda: gen.sample(generator=rng), args.batches)

        def end_to_end():
            graphs, _, _, term = gen.sample_molecules(generator=rng, constants=RC)
            gen.molecules.properties("Epoch 1", term, graphs)

        e2e_ms = _timed(end_to_end, args.batches)
        # the device path first: the reference's ~10^5 records can crowd the profiler's buffers of the run after it
        d2h_dev = _d2h_copies(lambda: device_path(batches[0]))
        d2h_ref = _d2h_copies(lambda: reference_path(batches[0]))
        med = lambda v: sorted(v)[len(v) // 2]                   # noqa: E731
        results[model] = {
            "reference_ms_per_batch": med(ref_ms), "device_ms_per_batch": med(dev_ms),
            "speedup": med(ref_ms) / med(dev_ms),
            "device_d2h_copies_per_batch": d2h_dev, "reference_d2h_copies_per_batch": d2h_ref,
            "generation_ms_per_batch": med(gen_ms), "sample_molecules_plus_properties_ms_per_batch": med(e2e_ms),
            "same_properties_as_reference": bool(same),
            "mean_atoms": float(batches[0][2].float().mean()),
            "weights": f"seeded recipe, {args.train_steps} Adam steps, final loss {loss:.4f}",
            "timed_batches": {"device": len(dev_ms), "reference": len(ref_ms)},
        }
    line = {"metric": "generated batch -> GenerationGraphs + Analyzer properties, ms per batch (median)",
            "batch": args.batch, "results": results, "gpu": gpu_info(0),
            "rdkit": "recording stub on both sides: RDKit's own cost excluded; the end-to-end saving with RDKit "
                     "is not measured"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
