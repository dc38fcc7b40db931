"""C5 (BASELINE.json configs[4]): `GraphGenerator.sample`, EMN model, 100 k molecules over 8 GPUs -- generation is
embarrassingly parallel: N independent replicas with distinct seeds, no data-path collective.

    python tools/bench_generation.py [--model EMN] [--molecules 12500] [--batch 1000] [--impl eager|graphed|both]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
           tools/bench_generation.py --molecules 12500          # 8 x 12 500 = 100 000 molecules

Weights.  A random-init EMN ends every rollout in round 1 (SURVEY.md 8d), so every replica first runs the same
seeded recipe: reference initialisers under torch.manual_seed(0), `--train-steps` (300) full-batch Adam steps
(lr 3e-4) on the 256 recorded real rows of gdb13_1K/train.h5 (tests/golden/gdb13_rows.npz), through this package's
training step.  `--checkpoint` loads a reference .pth instead (e.g. the shipped GGNN one with --model GGNN).

Implementations.  `--impl eager` is `generation.GraphGenerator` (two blocking reads per round), `graphed` is
`graphed.GraphedGenerator` (each round a replay of one captured CUDA graph, the stop rule on the device); `both`
alternates eager and graphed batches in one process with the same weights and batch size, so that clock and power
drift hit both alike.  Each batch is timed with CUDA events around its `build_graphs` call.

One JSON line (rank 0): per implementation molecules/s per GPU and in total (max over ranks), rounds and inert
rounds (graphed rounds launched past the end of a batch) per batch, mean atoms, fraction properly terminated; the
card name, power limit and SM clock read from nvidia-smi in the same call; `cpu_reference` = the unmodified reference
`GraphGenerator.build_graphs` with the same weights on this host's cores for ONE batch (bounded sample), when
oracle/_ref holds the reference modules.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_DIR = os.path.join(ROOT, "oracle", "_ref", "graphinvent")


def train_weights(model_name, steps, dev):
    """the seeded recipe; returns the module (eval mode) and its final training loss"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.optim import FlatAdam
    C = make_constants(model_name)
    torch.manual_seed(0)
    net = mpnn.create(C).to(dev)
    z = np.load(os.path.join(ROOT, "tests", "golden", "gdb13_rows.npz"))
    nodes = torch.from_numpy(z["nodes"]).to(dev)                 # int8, read directly by K0
    edges = torch.from_numpy(z["edges"]).to(dev)
    apds = torch.from_numpy(z["apds"]).float().to(dev)
    opt = FlatAdam(net.parameters(), lr=3e-4)
    loss = None
    keep = {0, 1, 2, 5, 10, 20, 39, 100, 200, steps - 1}
    traj = {}
    for i in range(steps):
        out = net(nodes, edges)
        loss = Fn.kl_loss(out, apds)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        if i in keep:
            traj[i] = loss.detach()
    train_weights.trajectory = {str(k): round(float(v), 4) for k, v in traj.items()}
    return C, net.eval(), (float(loss.detach()) if loss is not None else None)


def cpu_reference_generation(C, state_dict, batch, model_name):
    """the unmodified reference generator on the host cores (SURVEY.md Appendix C import recipe: three stub modules)"""
    if not os.path.isfile(os.path.join(REF_DIR, "GraphGenerator.py")):
        return None
    from collections import namedtuple
    N, A, CH, E = C.max_n_nodes, 5, 3, C.n_edge_features
    base = C._asdict()
    base.update(device="cpu", dim_nodes=[N, A + CH], dim_edges=[N, N, E], dim_f_add=[N, A, CH, E], dim_f_conn=[N, E],
                n_atom_types=A, n_formal_charge=CH, n_imp_H=0, n_chirality=0, use_explicit_H=False, ignore_H=True,
                use_chirality=False, atom_types=["C", "N", "O", "S", "Cl"], formal_charge=[-1, 0, 1],
                imp_H=[0, 1, 2, 3], chirality=["None", "R", "S"], generation_epoch=1, job_dir="/tmp/")
    RC = namedtuple("constants", sorted(base))(**base)
    for name in ("rdkit", "rdkit.Chem"):
        sys.modules.setdefault(name, types.ModuleType(name))
    mg = types.ModuleType("MolecularGraph")
    mg.GenerationGraph = type("GenerationGraph", (), {"__init__": lambda self, **kw: None})
    sys.modules["MolecularGraph"] = mg
    pkg = types.ModuleType("parameters")
    pkg.__path__ = []
    pc = types.ModuleType("parameters.constants")
    pc.constants = RC
    pkg.constants = pc
    sys.modules["parameters"] = pkg
    sys.modules["parameters.constants"] = pc
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    import gnn.mpnn as ref_mpnn
    import GraphGenerator as GG
    cls = {"GGNN": ref_mpnn.GGNN, "MNN": ref_mpnn.MNN, "AttGGNN": ref_mpnn.AttentionGGNN, "EMN": ref_mpnn.EMN}[model_name]
    net = cls(RC)
    net.load_state_dict({k: v.cpu() for k, v in state_dict.items()})
    net.eval()
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    # The reference keeps a dummy graph in slot 0 whose edges are never cleared (GraphGenerator.py:461-465 re-arms
    # nodes / n_nodes only): two "add" actions of different bond type in successive rounds leave a two-type bond there
    # and the reference's own EMN forward then fails (edge_mpnn.py:123-156 sizes its index lists by the summed bond
    # VALUES).  Whether that happens depends on the sampled trajectory of that one graph: retry with the next seed.
    failed = []
    for seed in range(1, 9):
        torch.manual_seed(seed)
        t0 = time.perf_counter()
        try:
            with torch.no_grad():
                gen = GG.GraphGenerator(model=net, batch_size=batch)
                n = gen.build_graphs()
        except RuntimeError as ex:
            failed.append({"seed": seed, "error": str(ex)[:120]})
            continue
        dt = time.perf_counter() - t0
        break
    else:
        return {"error": "the reference generator failed for every seed tried", "attempts": failed}
    nn = gen.generated_n_nodes[:n].float()
    return {"value": n / dt, "unit": "molecules/s", "seconds": dt, "n_generated": int(n), "batch": batch,
            "cores": torch.get_num_threads(), "kind": "reference", "mean_atoms": float(nn.mean()),
            "sample": "one GraphGenerator.build_graphs() call (unmodified reference, stubbed rdkit / constants)",
            "seed": seed, "failed_seeds": failed}


def gpu_info(index):
    """name, power limit and SM clock of the card, as nvidia-smi reports them now (None without nvidia-smi)"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None
    parts = [x.strip() for x in out.split(",")]
    return dict(zip(("name", "power_limit", "sm_clock"), parts)) if len(parts) == 3 else {"raw": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="EMN", choices=["EMN", "GGNN", "MNN", "AttGGNN"])
    ap.add_argument("--molecules", type=int, default=12500, help="per replica (8 x 12 500 = 100 000)")
    ap.add_argument("--batch", type=int, default=1000, help="generation batch (reference default, defaults.py:113)")
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--impl", default="eager", choices=["eager", "graphed", "both"])
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)      # measurement plumbing only (barrier + max of the timings)

    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import GraphedGenerator
    t_train0 = time.perf_counter()
    C, net, train_loss = train_weights(args.model, 0 if args.checkpoint else args.train_steps, dev)
    if args.checkpoint:
        net.load_state_dict(torch.load(args.checkpoint, map_location="cpu", weights_only=False))
    torch.cuda.synchronize()
    t_train = time.perf_counter() - t_train0

    impls = ["eager", "graphed"] if args.impl == "both" else [args.impl]
    cls = {"eager": GraphGenerator, "graphed": GraphedGenerator}
    gens, rngs = {}, {}
    for k, name in enumerate(impls):
        rngs[name] = torch.Generator(device=dev).manual_seed(1000 + 100 * k + rank)   # distinct streams per replica
        gens[name] = cls[name](net, batch_size=args.batch, n_atom_types=5, n_formal_charge=3, device=dev)
        gens[name].build_graphs(generator=rngs[name])                 # warm-up batch (graphed: the capture)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    B = args.batch
    events = {name: [] for name in impls}
    # per implementation: batches, rounds, inert rounds, atoms, properly terminated
    acc = {name: [0.0] * 5 for name in impls}
    done = 0
    while done < args.molecules:
        for name in impls:
            gen = gens[name]
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            gen.build_graphs(generator=rngs[name])
            ev1.record()
            events[name].append((ev0, ev1))
            a = acc[name]
            a[0] += 1
            a[1] += gen.rounds
            a[2] += getattr(gen, "inert_rounds", 0)
            a[3] += float(gen.generated_n_nodes[:B].float().sum())   # sample() hands out the first batch_size graphs
            a[4] += float(gen.properly_terminated[:B].float().sum())
        done += B
    torch.cuda.synchronize()
    results = {}
    for name in impls:
        ms = sum(e0.elapsed_time(e1) for e0, e1 in events[name])
        batches, rounds, inert, atoms, proper = acc[name]
        stats = torch.tensor([ms, batches * B, rounds, inert, atoms, proper], dtype=torch.float64, device=dev)
        ms_max = ms
        if world > 1:
            mx = stats.clone()
            dist.all_reduce(mx, op=dist.ReduceOp.MAX)
            dist.all_reduce(stats, op=dist.ReduceOp.SUM)
            ms_max = float(mx[0])
        total = float(stats[1])
        n_batches = total / B
        results[name] = {"value": total / (ms_max / 1e3), "unit": "molecules/s",
                         "per_gpu": total / world / (ms_max / 1e3), "molecules": int(total), "seconds": ms_max / 1e3,
                         "rounds_per_batch": float(stats[2]) / n_batches,
                         "inert_rounds_per_batch": float(stats[3]) / n_batches,
                         "mean_atoms": float(stats[4]) / total, "properly_terminated": float(stats[5]) / total}
    if rank == 0:
        main_impl = impls[-1]
        line = {"metric": f"generated molecules/s ({args.model}, GraphGenerator.sample, device-side rounds)",
                "value": results[main_impl]["value"], "unit": "molecules/s", "impl": args.impl,
                "n_gpus": world, "batch": args.batch, "impls": results, "gpu": gpu_info(local),
                "parallelism": f"{world} independent replicas, distinct seeds, no collective",
                "data": "synthetic (sampled)",
                "weights": (f"checkpoint {args.checkpoint}" if args.checkpoint else
                            f"seeded recipe: {args.train_steps} Adam steps (lr 3e-4) on 256 real gdb13 rows, final loss {train_loss:.4f}, {t_train:.1f} s"),
                "config": {"workload": "GraphGenerator.sample 100k-molecule batched generation, EMN model, 8xH100 embarrassingly parallel",
                           "name": "C5"}}
        if "graphed" in results and "eager" in results:
            line["graphed_over_eager"] = results["graphed"]["value"] / results["eager"]["value"]
        if getattr(train_weights, "trajectory", None):
            line["train_loss_trajectory"] = train_weights.trajectory
        if not args.no_cpu:
            try:
                line["cpu_reference"] = cpu_reference_generation(C, net.state_dict(), args.batch, args.model)
            except Exception as ex:
                import traceback
                line["cpu_reference"] = {"error": repr(ex), "where": traceback.format_exc().splitlines()[-8:]}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
