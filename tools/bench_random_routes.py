"""What a fresh random decoding route per pass costs: the per-pass rebuild of graphinvent_b200.loader.RandomRouteLoader
against the training pass it feeds.

    python tools/bench_random_routes.py [--passes 3] [--synthetic 2000] [--out bench_random_routes.jsonl]

Sets: gdb13_1K/train (979 molecules; tests/golden/preprocess_gdb13.npz) and a synthetic set of 38-atom molecules
(graphinvent_b200.synthetic), batch_size 1000 for both, a seeded GGNN of the reference's default sizes (oracle
make_constants / init_state_dict) in a graphed.TrainStep on int8 inputs.  Per pass, host clock around work that
ends in a device synchronise:
  reorder_s      preprocess.reorder with device-drawn rankings (the draw, the BFS and the reordered stacks)
  build_s        preprocess.file_rows over the reordered molecules (the construction, rows left on the device)
  train_s        TrainStep.train_epoch over the RandomRouteLoader pass (its rows already built by len())
  fixed_train_s  TrainStep.train_epoch over DeviceBlockLoader on a fixed preprocessed set (the epoch-0 file)
  rebuild_share  (reorder_s + build_s) / (reorder_s + build_s + train_s)
One warm-up pass first.  One JSON line per pass, with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

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
    from graphinvent_b200 import synthetic as S
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_gdb13.npz"))
    yield "gdb13_1K_train", z["gdb13_1K_train/nodes"], z["gdb13_1K_train/edges"]
    yield f"synthetic38_{n_synthetic}", *S.random_graphs(n_synthetic, 38, 5, 3, seed=38)


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def step_for(N, edges, B):
    import torch
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.optim import FlatAdam
    from oracle import mpnn_oracle as O
    C = O.make_constants("GGNN", max_n_nodes=N)
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=0))
    net = net.cuda()
    per_molecule = int((edges != 0).reshape(edges.shape[0], -1).sum(1).max())
    cap = -(-B * per_molecule // 128) * 128 + 128
    return TrainStep(net, FlatAdam(net.parameters(), lr=1e-4), batch_size=B, entry_capacity=cap,
                     input_dtype=torch.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--synthetic", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from graphinvent_b200 import preprocess as PP
    from graphinvent_b200.loader import DeviceBlockLoader, RandomRouteLoader
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = card()
    out = open(a.out, "a") if a.out else None
    B = a.batch
    for name, nodes, edges in sets(a.synthetic):
        N = nodes.shape[1]
        step = step_for(N, edges, B)
        loader = RandomRouteLoader(nodes, edges, batch_size=B, block_size=10 * B, seed=0, n_atom_types=5,
                                   n_formal_charge=3)
        dn, de = torch.from_numpy(nodes).cuda(), torch.from_numpy(edges).cuda()
        rows0, _ = PP.file_rows(*PP.reorder(dn, de, layout=GDB13)[:2], B, *GDB13)
        fixed = DeviceBlockLoader(types.SimpleNamespace(**{k: t.cpu().numpy() for k, t in
                                                           zip(("nodes", "edges", "apds"), rows0)}),
                                  batch_size=B, block_size=10 * B)
        del rows0
        for p in range(a.passes + 1):
            reorder_s, (rn, re_, _) = timed(lambda: PP.reorder(dn, de, "bfs", seed=0, epoch=p, layout=GDB13))
            build_s, (_, n_rows) = timed(lambda: PP.file_rows(rn, re_, B, *GDB13))
            del rn, re_
            loader.set_epoch(p)
            len_s, n_batches = timed(lambda: len(loader))
            train_s, _ = timed(lambda: step.train_epoch(loader))
            fixed_s, _ = timed(lambda: step.train_epoch(fixed))
            if p == 0:
                continue                                  # warm-up
            rec = dict(bench="random_routes", set=name, molecules=int(nodes.shape[0]), N=N, batch_size=B, pass_=p,
                       rows=int(n_rows), batches=int(n_batches), reorder_s=reorder_s, build_s=build_s,
                       len_s=len_s, train_s=train_s, fixed_train_s=fixed_s,
                       rebuild_share=(reorder_s + build_s) / (reorder_s + build_s + train_s), card=gpu)
            line = json.dumps(rec)
            print(line, flush=True)
            if out:
                out.write(line + "\n")
        del step, loader, fixed
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
