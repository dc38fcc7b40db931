"""Training-set construction: the device pass (graphinvent_b200.preprocess.groups) against the reference's
`DataProcesser.get_subgraphs` loop.

    python tools/bench_preprocess.py [--repeats 5] [--synthetic 20000] [--reference-groups 3]

Device pass: gdb13_1K/train (979 molecules, batch_size 1000; tests/golden/preprocess_gdb13.npz) and a synthetic set
of 38-atom molecules (graphinvent_b200.synthetic, batch_size 1000).  The time is the host clock around the whole
iteration of `groups()` -- uploads, kernels, the copies back and the per-group arrays -- which ends in a device
synchronise; one warm-up pass first, then the median of --repeats passes.  Reported as molecules/s and rows/s, with
the card's name and power limit.

Reference loop (--reference-groups > 0; needs the reference's DataProcesser.py and oracle/_ref, so it runs where the
reference is checked out, GPU or not): its own get_molecule_subset / get_subgraphs over the first groups of the same
sets, timed per group.  No extrapolation is made.  One JSON line per measurement.
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


def gdb13():
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    return z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]


def synthetic(M):
    from graphinvent_b200 import synthetic as S
    return S.random_graphs(M, 38, 5, 3, seed=38)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # no nvidia-smi: the record says so
        return f"unknown ({e})"


def device(name, nodes, edges, B, repeats):
    import torch
    from graphinvent_b200 import preprocess as PP
    if not torch.cuda.is_available():
        raise SystemExit("the device pass needs a CUDA device")

    def run():
        torch.cuda.synchronize()
        t = time.perf_counter()
        rows = sum(g.nodes.shape[0] for g in PP.groups(nodes, edges, B, 5, 3))
        torch.cuda.synchronize()
        return time.perf_counter() - t, rows

    run()
    times, rows = zip(*[run() for _ in range(repeats)])
    t = float(np.median(times))
    print(json.dumps(dict(set=name, impl="device", molecules=int(nodes.shape[0]), rows=int(rows[0]), batch_size=B,
                          seconds=t, spread=[float(min(times)), float(max(times))],
                          molecules_per_s=nodes.shape[0] / t, rows_per_s=rows[0] / t, device=card())))


def reference(name, nodes, edges, B, n_groups):
    import pytest
    from tests import test_preprocess_host as H

    class Patch:
        def setitem(self, d, k, v):
            d[k] = v
    times, mark = [], [0.0]

    def on_group():
        now = time.perf_counter()
        times.append(now - mark[0])
        mark[0] = now
    M = min(nodes.shape[0], n_groups * B)
    try:
        mark[0] = time.perf_counter()
        saved = H.live_groups(Patch(), nodes[:M], edges[:M], B, (5, 3, 0, 0), on_group=on_group, max_groups=n_groups)
    except pytest.skip.Exception as e:
        print(json.dumps(dict(set=name, impl="reference", skipped=str(e))))
        return
    print(json.dumps(dict(set=name, impl="reference get_subgraphs (host CPU)", batch_size=B, groups=len(saved),
                          group_seconds=times, group_rows=[g["group_size"] for g in saved],
                          group_molecules=[g["stop"] - g["start"] for g in saved])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=20000)
    ap.add_argument("--reference-groups", type=int, default=0)
    ap.add_argument("--no-device", action="store_true")
    a = ap.parse_args()
    sets = [("gdb13_1K/train", *gdb13()), (f"synthetic N=38 x{a.synthetic}", *synthetic(a.synthetic))]
    for name, nodes, edges in sets:
        if not a.no_device:
            device(name, nodes, edges, 1000, a.repeats)
        if a.reference_groups:
            reference(name, nodes, edges, 1000, a.reference_groups)


if __name__ == "__main__":
    main()
