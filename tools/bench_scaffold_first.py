"""Throughput of the scaffold-first decoding order, graphinvent_b200.preprocess.scaffold_first (`gib_scaffold_first`),
against the Python restatement of tests/scaffold_match_reference.py on the host.

    python tools/bench_scaffold_first.py [--repeats 5] [--synthetic 2000] [--host 200] [--out bench_scaffold_first.jsonl]

Sets: gdb13_1K/train (979 molecules; tests/golden/preprocess_gdb13.npz) and synthetic 38-atom molecules
(tests/scaffold_match_reference.random_molecule, Ef = 3), their atoms shuffled.  Scaffolds: 5-atom prefixes of the
unshuffled molecules.  Two modes per set:
  ids     scaffold_ids given: each molecule matched against its own prefix scaffold
  search  scaffold_ids=None over a table of 100 scaffolds (prefixes of molecules 0..99), first match wins
Device: host clock around the call, which ends in the status read (a device synchronise), rankings drawn on the
device; one warm-up call, then the median of --repeats calls.  Host: the restatement over the first --host molecules
of the set, with the device's rankings.  One JSON line per (set, mode), with the card's name and power limit read in
the same run.  No RDKit figure: RDKit is not a dependency of the package.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GDB13 = (5, 3, 0, 0)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # no nvidia-smi: the record says so
        return f"unknown ({e})"


def sets(n_synthetic):
    from tests import scaffold_match_reference as SM
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    out = {"gdb13_1K_train": (z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"])}
    rng = np.random.default_rng(0)
    mols = [SM.random_molecule(rng, int(rng.integers(20, 39)), 38, GDB13, 3, n_types=3) for _ in range(n_synthetic)]
    out["synthetic38"] = (np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=2000)
    ap.add_argument("--host", type=int, default=200)
    ap.add_argument("--out", default="bench_scaffold_first.jsonl")
    a = ap.parse_args()
    import torch
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200.generation import ScaffoldTable
    from tests import scaffold_match_reference as SM
    from tests import scaffold_route_reference as SR
    gpu = card()
    recs = []
    for name, (nodes, edges) in sets(a.synthetic).items():
        M, N, F = nodes.shape
        Ef = edges.shape[3]
        ks = np.array([min(5, SM.n_atoms(x)) for x in nodes])
        sn, se = SR.prefix_scaffolds(nodes, edges, ks)
        rng = np.random.default_rng(1)
        pairs = [SM.shuffle(nodes[m], edges[m], rng) for m in range(M)]
        X = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
        E = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
        for mode in ("ids", "search"):
            if mode == "ids":
                table, ids, S = ScaffoldTable(sn, se, None, N, F, Ef, GDB13, "cuda"), np.arange(M), M
            else:
                table, ids, S = ScaffoldTable(sn[:100], se[:100], None, N, F, Ef, GDB13, "cuda"), None, 100
            call = lambda: PP.scaffold_first(X, E, table, scaffold_ids=ids, seed=3, epoch=1, layout=GDB13)
            out = call()
            times = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                out = call()
                times.append(time.perf_counter() - t0)
            dev_s = float(np.median(times))
            matched = int((out[3] >= 0).sum())
            h = min(a.host, M)
            rk = PP.rankings([SM.n_atoms(x) for x in X[:h].cpu().numpy()], N, seed=3, epoch=1).cpu().numpy()
            t0 = time.perf_counter()
            ref = SM.scaffold_first(X[:h].cpu().numpy(), E[:h].cpu().numpy(), table.nodes.cpu().numpy(),
                                    table.edges.cpu().numpy(), rk, None, None if ids is None else ids[:h])
            host_s = time.perf_counter() - t0
            assert np.array_equal(ref[3], out[3][:h].cpu().numpy()), "device ids differ from the restatement"
            rec = dict(set=name, mode=mode, molecules=M, N=N, scaffolds=S, matched=matched,
                       device_ms=dev_s * 1e3, device_mol_per_s=M / dev_s, device_ms_all=[t * 1e3 for t in times],
                       host_molecules=h, host_mol_per_s=h / host_s, card=gpu)
            print(json.dumps(rec), flush=True)
            recs.append(rec)
    with open(a.out, "w") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
