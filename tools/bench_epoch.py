"""One training epoch of a captured step (`graphed.TrainStep`) behind three data loaders, on one GPU.

    python tools/bench_epoch.py [--rows 200000] [--block 100000] [--batch 1000] [--config C2|C5T]

The set: `--rows` seeded synthetic int8 rows at gdb13 dims (the `--config` model's, bench.py's CONFIGS; C2 = GGNN
hidden 128, 4 message passes; C5T = the EMN), one-hot int8 APD targets.  Each arm trains a fresh copy of the same
initial model with FlatAdam over one epoch, with torch's default generator seeded alike, so all three see the same
batches in the same order:

  (a) reference  the unmodified reference BlockDataLoader + HDFDataset (oracle/_ref/, `h5py.File` replaced by the
                 in-memory arrays), n_workers 0, pinned batches, feeding a float32 step(nodes, edges, target);
  (b) host_int8  int8 host batches gathered by numpy in that order, pinned, feeding an int8 step(nodes, edges, target);
  (c) device     `loader.DeviceBlockLoader` + `TrainStep.train_epoch` (int8 step): one gather launch per batch.

Arms (b) and (c) then run a second epoch (`*_epoch2`): the first includes allocating the device loader's pinned
staging buffers and device slots; blocks still resident after it are not uploaded again.

Reported per arm: epoch seconds (host clock around the epoch, ended by a device synchronise), graphs/s, and the share
of the epoch the host spent outside `CUDAGraph.replay()`.  Also the gather kernel's CUDA-event time per batch (mean of
200 launches of a full batch), the card's name and power limit, and whether (b) and (c) end with bit-identical
parameters.  One JSON line.  Arm (a) is skipped, and reported as null, when oracle/_ref/ does not hold the reference.
"""
import argparse
import copy
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


def card():
    """name and power limit of the card, as nvidia-smi reports them now"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return dict(name=name, power_limit=power)
    except Exception:
        return dict(name=torch.cuda.get_device_name(0), power_limit=None)


def make_set(C, rows, seed):
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    base = min(rows, 10000)            # generating graphs is slow on the host; the loaders do not care about repeats
    nodes, edges = S.random_graphs(base, C.max_n_nodes, 5, 3, n_edge_features=C.n_edge_features, seed=seed,
                                   min_atoms=1)
    reps = -(-rows // base)
    nodes, edges = np.tile(nodes, (reps, 1, 1))[:rows], np.tile(edges, (reps, 1, 1, 1))[:rows]
    apd = apd_length(C)
    apds = np.zeros((rows, apd), np.int8)
    apds[np.arange(rows), np.random.default_rng(seed + 1).integers(0, apd, rows)] = 1
    return types.SimpleNamespace(nodes=nodes.astype(np.int8), edges=edges.astype(np.int8), apds=apds)


class ReplayClock:
    """host seconds spent inside CUDAGraph.replay() while active"""

    def __enter__(self):
        self.seconds, orig = 0.0, torch.cuda.CUDAGraph.replay
        self._orig = orig

        def replay(graph):
            t = time.perf_counter()
            orig(graph)
            self.seconds += time.perf_counter() - t
        torch.cuda.CUDAGraph.replay = replay
        return self

    def __exit__(self, *exc):
        torch.cuda.CUDAGraph.replay = self._orig


def make_step(net0, B, cap, in_dtype):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    net = copy.deepcopy(net0)
    return TrainStep(net, FlatAdam(net.parameters(), lr=1e-4), batch_size=B, entry_capacity=cap, input_dtype=in_dtype)


def timed_epoch(fn, n_graphs):
    torch.cuda.synchronize()
    with ReplayClock() as clock:
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        sec = time.perf_counter() - t
    return dict(epoch_s=sec, graphs_per_s=n_graphs / sec, host_outside_replay=1.0 - clock.seconds / sec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200000)
    ap.add_argument("--block", type=int, default=100000)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--config", default="C2", choices=["C2", "C5T"])
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_epoch.py needs a GPU"
    import bench
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.loader import DeviceBlockLoader
    from oracle import mpnn_oracle as O
    from tests.golden.make_loader_order import reference_loader, reference_module

    C = bench.make_constants_for(args.config)
    B = args.batch
    ds = make_set(C, args.rows, args.seed)
    net0 = mpnn.create(C)
    net0.load_state_dict(O.init_state_dict(C, seed=0))
    net0 = net0.cuda()
    by_type = args.config != "C5T"
    e = ds.edges != 0
    per_row = e.reshape(args.rows, -1).sum(1) if by_type else e.any(-1).reshape(args.rows, -1).sum(1)
    cap = int(np.sort(per_row)[-B:].sum()) + 256          # the densest possible batch fits
    loader = DeviceBlockLoader(ds, batch_size=B, block_size=args.block)

    def host_batches(in_dtype):
        for k, ix in loader.order():
            sel = (ix + k * args.block).numpy()
            n, e = torch.from_numpy(ds.nodes[sel]), torch.from_numpy(ds.edges[sel])
            if in_dtype == torch.float32:
                n, e = n.float(), e.float()
            yield n.pin_memory(), e.pin_memory(), torch.from_numpy(ds.apds[sel]).float().pin_memory()

    def run_host(step, batches):
        slots = torch.zeros(len(loader), device="cuda")
        for idx, (n, e, t) in enumerate(batches):
            slots[idx:idx + 1].copy_(step(n, e, t).view(1))
        step.check()
        return torch.mean(slots)

    # warm every arm's step (capture, FlatAdam flattening) on one batch, identically for (b) and (c)
    steps = {"host_int8": make_step(net0, B, cap, torch.int8), "device": make_step(net0, B, cap, torch.int8)}
    mod = reference_module()
    if mod is not None:
        steps["reference"] = make_step(net0, B, cap, torch.float32)
    torch.manual_seed(args.seed)
    warm = next(host_batches(torch.int8))
    for name, step in steps.items():
        n, e, t = warm if name != "reference" else (warm[0].float(), warm[1].float(), warm[2])
        step(n, e, t)
    torch.cuda.synchronize()
    # the device arm's epoch includes its block uploads; the other arms read arrays already in host memory
    res = {}
    if mod is not None:
        ref_loader = reference_loader(mod, ds.nodes, ds.edges, ds.apds, batch_size=B, block_size=args.block,
                                      shuffle=True, n_workers=0, pin_memory=True)
        torch.manual_seed(args.seed + 1)
        res["reference"] = timed_epoch(lambda: run_host(steps["reference"], iter(ref_loader)), args.rows)
    torch.manual_seed(args.seed + 1)
    res["host_int8"] = timed_epoch(lambda: run_host(steps["host_int8"], host_batches(torch.int8)), args.rows)
    torch.manual_seed(args.seed + 1)
    res["device"] = timed_epoch(lambda: steps["device"].train_epoch(loader), args.rows)
    # a second epoch of (b) and (c): the device loader's staging buffers exist, blocks still resident are kept
    uploads_first = loader.uploads
    torch.manual_seed(args.seed + 2)
    res["host_int8_epoch2"] = timed_epoch(lambda: run_host(steps["host_int8"], host_batches(torch.int8)), args.rows)
    torch.manual_seed(args.seed + 2)
    res["device_epoch2"] = timed_epoch(lambda: steps["device"].train_epoch(loader), args.rows)
    uploads_second = loader.uploads - uploads_first
    same = all(torch.equal(p.view(torch.int32), q.view(torch.int32))
               for p, q in zip(steps["host_int8"].model.parameters(), steps["device"].model.parameters()))

    # the gather kernel alone: a full batch into the device step's static inputs
    step = steps["device"]
    item = next(iter(loader.batches()))
    for _ in range(10):
        loader.gather(item, step.nodes, step.edges, step.target, step.ctl)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        loader.gather(item, step.nodes, step.edges, step.target, step.ctl)
    e1.record()
    torch.cuda.synchronize()
    gather_us = e0.elapsed_time(e1) * 1000 / 200
    step_ms = res["device"]["epoch_s"] * 1000 / len(loader)
    out = dict(tool="bench_epoch", config=args.config, rows=args.rows, block=args.block, batch=B,
               batches=len(loader), card=card(), arms={k: res.get(k) for k in
               ("reference", "host_int8", "device", "host_int8_epoch2", "device_epoch2")},
               gather_us_per_batch=gather_us, gather_share_of_step=gather_us / 1000 / step_ms,
               host_int8_equals_device_bitwise=same, uploads_epoch1=uploads_first,
               uploads_epoch2=uploads_second)
    print(json.dumps(out))
    if not same:
        sys.exit("host_int8 and device arms ended with different parameters")


if __name__ == "__main__":
    main()
