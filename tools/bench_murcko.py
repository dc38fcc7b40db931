"""Throughput of the Murcko scaffold extraction and deduplication, graphinvent_b200.preprocess.murcko_scaffolds
(`gib_murcko`), against the Python restatement of tests/murcko_reference.py on the host.

    python tools/bench_murcko.py [--repeats 5] [--synthetic 5000] [--host 200] [--out bench_murcko.jsonl]

Sets: gdb13_1K/train (979 molecules; tests/golden/preprocess_gdb13.npz) and synthetic ring-rich 38-atom molecules
(tests/scaffold_match_reference.random_molecule with about one extra bond per two atoms, Ef = 3), atoms shuffled.
Two arms per set:
  host_input    numpy stacks in, the whole call (host-to-device copies, the device pass, the status reads)
  device_input  the stacks already on the device
Host clock around the call, which ends in the status read (a device synchronise); one warm-up call, then the median of
--repeats calls.  Host: the restatement over the first --host molecules.  One JSON line per (set, arm) with the
distinct scaffolds and the card's name and power limit read in the same run.  No RDKit figure: RDKit is not a
dependency of the package.
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
    mols = [SM.shuffle(*SM.random_molecule(rng, int(rng.integers(12, 39)), 38, GDB13, 3, n_types=3,
                                           extra_bonds=1.0), rng) for _ in range(n_synthetic)]
    out["synthetic38_rings"] = (np.stack([m[0] for m in mols]), np.stack([m[1] for m in mols]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=5000)
    ap.add_argument("--host", type=int, default=200)
    ap.add_argument("--out", default="bench_murcko.jsonl")
    a = ap.parse_args()
    import torch
    from graphinvent_b200 import preprocess as PP
    from tests import murcko_reference as MR
    gpu = card()
    recs = []
    for name, (nodes, edges) in sets(a.synthetic).items():
        M, N = nodes.shape[:2]
        h = min(a.host, M)
        t0 = time.perf_counter()
        ref = MR.murcko(nodes[:h], edges[:h])
        host_s = time.perf_counter() - t0
        inputs = {"host_input": (nodes, edges),
                  "device_input": (torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda())}
        for arm, (X, E) in inputs.items():
            call = lambda: PP.murcko_scaffolds(X, E, layout=GDB13)
            out = call()
            times = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                out = call()
                times.append(time.perf_counter() - t0)
            dev_s = float(np.median(times))
            head = PP.murcko_scaffolds(nodes[:h], edges[:h], layout=GDB13)
            assert np.array_equal(head.ids.cpu().numpy(), ref[1]), "device ids differ from the restatement"
            rec = dict(set=name, arm=arm, molecules=M, N=N, with_ring=int((out.ids >= 0).sum()),
                       distinct_scaffolds=int(out.nodes.shape[0]), device_ms=dev_s * 1e3,
                       device_mol_per_s=M / dev_s, device_ms_all=[t * 1e3 for t in times], host_molecules=h,
                       host_mol_per_s=h / host_s, card=gpu)
            print(json.dumps(rec), flush=True)
            recs.append(rec)
    with open(a.out, "w") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
