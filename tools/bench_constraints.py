"""Constrained generation: molecules/s, rounds per batch and the fraction of molecules within the set, with the
constraints as masks and as a post-filter on unconstrained generation, and the mask launch alone.

    python tools/bench_constraints.py [--batches 3] [--repeats 3] [--launches 500]

Model: the reference's pretrained gdb13 GGNN (oracle/_ref/pretrained_model.pth, installed by `__graft_entry__.build()`),
or, without it, a GGNN with seeded initial weights (`oracle.mpnn_oracle.init_state_dict`, seed 1).  At batch 1000 and
100, one `GraphedGenerator` without constraints ("none") and one with constraints whose `set_constraints` steps
through the sets below batch by batch (one captured round for all of them), so clock and power drift hit every
configuration alike:
    atoms_13      atoms=(13, 13)
    atoms_11      atoms=(11, 11)
    elements      at most 2 N and 2 O, no S, no Cl, no triple bond
    rings         min_ring_size=5, rings=(0, 2)
Each batch is timed with CUDA events around `build_graphs`; molecules/s is the median over `--repeats` repeats of
`--batches` batches.  A batch that needs more than the reference's 2N rounds raises, as without constraints, and is
counted in `round_limit_batches` (atoms=(13, 13) always does: one of the B - 1 slots has to make two molecules of at
least 14 rounds each).  Reported per set: molecules/s, rounds per batch, the fraction properly terminated and within
the set (`gib_constraints_check` flags none of over-max, small ring, under-min), the fraction ended at a dead end, and
the post-filter: the fraction of the unconstrained batch's molecules that are properly terminated and within the set,
and that times its molecules/s ("within_per_s").  The mask launch alone: `gib_action_mask_logits` (structure) and the
constrained launch under each set, on the state of a finished batch, `--launches` back-to-back launches between CUDA
events.  One JSON line per batch size with the card name, power limit and SM clock read from nvidia-smi.
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
from bench_action_mask import GDB13_ATOMS, GDB13_CHARGES   # noqa: E402
from bench_generation import gpu_info   # noqa: E402

SETS = {"atoms_13": dict(atoms=(13, 13)), "atoms_11": dict(atoms=(11, 11)),
        "elements": dict(atom_types={"N": (None, 2), "O": (None, 2), "S": (0, 0), "Cl": (0, 0)},
                         bonds={"TRIPLE": 0}),
        "rings": dict(min_ring_size=5, rings=(0, 2))}
BAD = 1 | 2 | 4                     # GIB_CONS_OVER_MAX | GIB_CONS_SMALL_RING | GIB_CONS_UNDER_MIN


def model(dev):
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = make_constants("GGNN")
    net = mpnn.create(C)
    path = os.path.join(ROOT, "oracle", "_ref", "pretrained_model.pth")
    if os.path.exists(path):
        net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
        name = "GGNN_pretrained"
    else:
        net.load_state_dict(O.init_state_dict(O.make_constants("GGNN"), seed=1))
        name = "GGNN_seeded"
    return name, net.to(dev).eval()


def mask_times(gen, masks, launches):
    """ms per launch of the structural mask and of each constrained mask on the generator's current state"""
    B = gen.batch_size
    x = torch.zeros(B, gen.apd, device=gen.device)
    st = ctypes.c_void_p(torch.cuda.current_stream(gen.device).cuda_stream)

    def timed(m):
        for _ in range(10):
            m.apply(B, x, gen.n_nodes, st, gen.nodes, gen.edges)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            m.apply(B, x, gen.n_nodes, st, gen.nodes, gen.edges)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / launches

    return {name: timed(m) for name, m in masks.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=3, help="timed batches per configuration and repeat")
    ap.add_argument("--repeats", type=int, default=3, help="repeats; molecules/s is their median")
    ap.add_argument("--launches", type=int, default=500, help="launches per mask timing")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from graphinvent_b200.generation import Constraints, make_action_mask
    from graphinvent_b200.graphed import GraphedGenerator
    info = gpu_info(0)
    consts = namedtuple("C", "atom_types formal_charge")(GDB13_ATOMS, GDB13_CHARGES)
    sets = {k: Constraints(**v, constants=consts) for k, v in SETS.items()}
    mname, net = model(dev)
    for B in (1000, 100):
        kw = dict(batch_size=B, n_atom_types=5, n_formal_charge=3, device=dev)
        plain = GraphedGenerator(net, **kw)
        con = GraphedGenerator(net, constraints=sets["rings"], **kw)
        layout, N, F_, Ef, apd = plain.layout, plain.N, plain.F, plain.Ef, plain.apd
        checks = {k: make_action_mask(None, None, consts, layout, N, F_, Ef, apd, dev, c) for k, c in sets.items()}
        rng = torch.Generator(device=dev).manual_seed(4000 + B)
        for gen in (plain, con):                        # warm-up batch (the capture)
            try:
                gen.build_graphs(generator=rng)
            except RuntimeError:
                pass
        graph = con.graph
        arms = ["none"] + list(sets)
        runs = {a: [] for a in arms}
        acc = {a: dict(batches=0, rounds=0, proper=0.0, within=0.0, dead=0.0, limit=0, atoms=0.0) for a in arms}
        post = {k: 0.0 for k in sets}
        for _ in range(args.repeats):
            timed = {a: [] for a in arms}
            for _ in range(args.batches):
                for a in arms:
                    gen = plain if a == "none" else con
                    if a != "none":
                        gen.set_constraints(sets[a])
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    try:
                        gen.build_graphs(generator=rng)
                    except RuntimeError:
                        acc[a]["limit"] += 1
                        continue
                    e1.record()
                    timed[a].append((e0, e1))
                    nodes, edges = gen.generated_nodes[:B], gen.generated_edges[:B]
                    n_at, pt = gen.generated_n_nodes[:B], gen.properly_terminated[:B].bool()
                    r = acc[a]
                    r["batches"] += 1
                    r["rounds"] += gen.rounds
                    r["proper"] += float(pt.float().mean())
                    r["atoms"] += float(n_at.float().mean())
                    if a == "none":
                        for k, m in checks.items():
                            f = m.check(nodes, edges, n_at)
                            post[k] += float((pt & ((f & BAD) == 0)).float().mean())
                    else:
                        f = checks[a].check(nodes, edges, n_at)
                        r["within"] += float((pt & ((f & BAD) == 0)).float().mean())
                        r["dead"] += float(((f & 8) != 0).float().mean())
            torch.cuda.synchronize()
            for a in arms:
                ms = sum(e0.elapsed_time(e1) for e0, e1 in timed[a])
                runs[a].append(len(timed[a]) * B / (ms / 1e3) if ms else float("nan"))
        assert con.graph is graph, "set_constraints recaptured the round"
        res = {}
        for a in arms:
            r = acc[a]
            k = max(r["batches"], 1)
            res[a] = {"molecules_per_s": float(np.median(runs[a])), "batches": r["batches"],
                      "round_limit_batches": r["limit"], "rounds_per_batch": r["rounds"] / k,
                      "mean_atoms": r["atoms"] / k, "fraction_properly_terminated": r["proper"] / k}
            if a != "none":
                res[a].update(fraction_within_set=r["within"] / k, fraction_dead_end=r["dead"] / k)
        k_none = max(acc["none"]["batches"], 1)
        for name in sets:
            frac = post[name] / k_none
            res[name]["post_filter"] = {"fraction_within_set": frac,
                                        "within_per_s": frac * res["none"]["molecules_per_s"]}
        struct = make_action_mask("structure", None, consts, layout, N, F_, Ef, apd, dev)
        masks = {"structure": struct, **{k: make_action_mask(None, None, consts, layout, N, F_, Ef, apd, dev, c)
                                         for k, c in sets.items()}}
        plain.build_graphs(generator=rng)
        ms = mask_times(plain, masks, args.launches)
        print(json.dumps({"metric": f"constrained generation molecules/s ({mname}, batch {B}, captured rounds)",
                          "impls": res, "mask_ms_per_launch": ms, "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
