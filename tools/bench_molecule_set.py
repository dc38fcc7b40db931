"""Time per call of the molecule set, graphinvent_b200.molecules.MoleculeSet (`gib_molset_identify`), against the
set's size, and the Python restatement of tests/molecule_set_reference.py on the host.

    python tools/bench_molecule_set.py [--repeats 7] [--sizes 0,10000,100000,1000000] [--out bench_molecule_set.jsonl]

Batches: --repeats + 1 seeded batches of 1000 molecules from the pretrained gdb13 GGNN (GraphedGenerator, float32 as
sampled; oracle/_ref/pretrained_model.pth).  Sets: filled to each size with distinct synthetic molecules (random
trees of 8-13 atoms with random atom and bond types, built on the device, added 65 536 at a time).  Per size, each
batch is looked up (`find`) and then inserted (`add`); the first batch warms up and is not counted.  Per call: device
events around it and the host clock around the whole call, which ends in its one status read; the median over the
batches.  One JSON line per size with the set's bytes, then one for the restatement's rate on the host CPU (a
CPU-bound figure, no device involved).  The card's name and power limit are read in the same run.  No RDKit figure:
RDKit is not a dependency of the package.
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
N, F, EF = 13, 8, 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # no nvidia-smi: the record says so
        return f"unknown ({e})"


def synthetic(M, seed):
    """int8 device stacks of M random connected molecules (trees) of 8..13 atoms, gdb13 layout, neutral atoms"""
    import torch
    g = torch.Generator("cuda").manual_seed(seed)
    n = torch.randint(8, N + 1, (M,), generator=g, device="cuda")
    atoms = torch.arange(N, device="cuda")[None] < n[:, None]
    nodes = torch.zeros((M, N, F), dtype=torch.int8, device="cuda")
    types = torch.randint(0, 5, (M, N), generator=g, device="cuda")
    nodes.scatter_(2, types[..., None], 1)
    nodes[..., 6] = 1                                       # formal charge 0
    nodes *= atoms[..., None].to(torch.int8)
    edges = torch.zeros((M, N, N, EF), dtype=torch.int8, device="cuda")
    rows = torch.arange(M, device="cuda")
    for a in range(1, N):
        b = (torch.rand(M, generator=g, device="cuda") * a).long()
        t = torch.randint(0, EF, (M,), generator=g, device="cuda")
        on = atoms[:, a]
        edges[rows[on], a, b[on], t[on]] = 1
        edges[rows[on], b[on], a, t[on]] = 1
    return nodes, edges


def generated(batches, B=1000):
    import torch
    from tests.conftest import pretrained_path
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator
    path = pretrained_path()
    if path is None:
        raise SystemExit("oracle/_ref/pretrained_model.pth is missing: run __graft_entry__.build() first")
    C = make_constants("GGNN")
    net = mpnn.create(C)
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    gen = GraphedGenerator(net.cuda().eval(), B, n_atom_types=5, n_formal_charge=3)
    out = []
    for seed in range(batches):
        U = torch.rand(2 * N, B, generator=torch.Generator("cuda").manual_seed(100 + seed), device="cuda")
        (nodes, edges, _), _, _, _ = gen.sample(uniforms=U)
        out.append((nodes, edges))
    return out


def timed(call):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    call()                                                  # ends in the status read: a synchronise
    b.record()
    wall = time.perf_counter() - t0
    b.synchronize()
    return a.elapsed_time(b), wall * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--sizes", default="0,10000,100000,1000000")
    ap.add_argument("--host", type=int, default=300)
    ap.add_argument("--out", default="bench_molecule_set.jsonl")
    a = ap.parse_args()
    import torch
    from graphinvent_b200.molecules import MoleculeSet
    from tests import molecule_set_reference as MS
    gpu = card()
    batches = generated(a.repeats + 1)
    recs = []
    for size in (int(x) for x in a.sizes.split(",")):
        s = MoleculeSet(N, F, EF, size + 1000 * len(batches), layout=GDB13)
        for pos in range(0, size, 65536):
            X, E = synthetic(min(65536, size - pos), seed=pos + 1)
            s.add(X, E)
        filled = len(s)
        times = {"find": [], "add": []}
        for i, (X, E) in enumerate(batches):
            for op in ("find", "add"):
                dev_ms, wall_ms = timed(lambda: getattr(s, op)(X, E))
                if i:
                    times[op].append((dev_ms, wall_ms))
        rec = dict(set_entries=filled, set_bytes=s.nbytes, batch=1000, batches=len(batches) - 1, card=gpu)
        for op, t in times.items():
            t = np.array(t)
            rec[f"{op}_device_ms"] = float(np.median(t[:, 0]))
            rec[f"{op}_wall_ms"] = float(np.median(t[:, 1]))
            rec[f"{op}_device_ms_all"] = t[:, 0].round(4).tolist()
        rec["entries_after"] = len(s)
        print(json.dumps(rec), flush=True)
        recs.append(rec)
        del s
        torch.cuda.empty_cache()
    X, E = (t.cpu().numpy().astype(np.int8) for t in batches[0])
    h = min(a.host, X.shape[0])
    ref = MS.MoleculeSet()
    t0 = time.perf_counter()
    ref.add(X[:h], E[:h])
    host_s = time.perf_counter() - t0
    rec = dict(restatement="tests/molecule_set_reference.py", host_cpu_bound=True, molecules=h,
               host_mol_per_s=h / host_s)
    print(json.dumps(rec), flush=True)
    recs.append(rec)
    with open(a.out, "w") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
