"""The default precision (3xTF32) against torch.autocast in bf16 and fp16, on the same seeded inputs.

    python tools/bench_autocast.py [--steps 50] [--warmup 10] [--repeats 3] [--gen-batches 3]

Per mode (default, bf16, fp16), alternating, `--repeats` times; each object is built inside the mode's autocast
context and keeps its mode for its replays.  The fp16 training step runs with a `torch.amp.GradScaler` (dynamic loss
scaling on the device, `TrainStep(grad_scaler=)`); default and bf16 run without one:
  - the C2 and C5T training steps of bench.py (graphed.TrainStep, int8 batches, FlatAdam): ms/step and graphs/s from
    CUDA events around `--steps` replays after `--warmup`; for fp16 also the time of the loss-scaling launches of one
    step (the non-finite check, the gated Adam and the scale update) against the plain Adam step of the same bucket;
  - the tensor-core GEMM classes of one profiled step (gib_profile_records, classes 0 forward/dX and 1 weight
    gradients): ms per step and achieved TFLOP/s (algorithmic FLOPs over kernel time);
  - C5 generation (graphed.GraphedGenerator, EMN gdb13 dims, batch 1000): ms per batch over `--gen-batches` batches
    on fixed uniforms;
  - the largest logit difference of each 16-bit mode from the default mode on the first C2 batch.
One JSON line, with the card's name, power limit and maximum SM clock read from nvidia-smi in the same call.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:
        return f"nvidia-smi unavailable ({e})"


DTYPE = {"default": None, "bf16": torch.bfloat16, "fp16": torch.float16}


def mode_ctx(mode):
    import contextlib
    return torch.autocast("cuda", dtype=DTYPE[mode]) if DTYPE[mode] is not None else contextlib.nullcontext()


def train_step(cfg, mode):
    import bench
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    C, nodes, edges, target, _ = bench.make_batch(cfg, seed=1002)
    torch.manual_seed(0)
    net = mpnn.create(C).cuda()
    opt = FlatAdam(net.parameters(), lr=1e-4)
    cap = int(torch.count_nonzero(edges).item()) + 1024
    scaler = torch.amp.GradScaler("cuda") if mode == "fp16" else None
    with mode_ctx(mode):
        step = TrainStep(net, opt, batch_size=nodes.shape[0], entry_capacity=cap, input_dtype=torch.int8,
                         grad_scaler=scaler)
    assert step.autocast_dtype is DTYPE[mode]
    batch = (nodes.to(torch.int8).cuda(), edges.to(torch.int8).cuda(), target.float().cuda())
    return step, batch, net


def time_steps(step, batch, steps, warmup):
    for _ in range(warmup):
        step(*batch)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step(*batch)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def scaling_launches(step, reps=20):
    """ms of (non-finite check + gated Adam + scale update) and of the plain Adam step alone, on the step's bucket
    (CUDA events around `reps` repetitions of each)"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import check, lib
    flat, found, opt = step.gflat, step.found_inf, step.optimizer
    saved = [t.clone() for t in (opt._flat, opt._m, opt._v)]
    def scaled():
        check(lib.gib_nonfinite_check(Fn._ptr(flat), flat.numel(), Fn._ptr(found), Fn._stream(step.dev)), "check")
        opt.scaled_step(found, step.grad_scaler)
    def plain():
        check(lib.gib_adam_step(Fn._ptr(opt._flat), Fn._ptr(flat), Fn._ptr(opt._m), Fn._ptr(opt._v), flat.numel(), 1,
                                1e-4, 0.9, 0.999, 1e-8, 0.0, 1.0, Fn._stream(step.dev)), "gib_adam_step")
    out = []
    for fn in (scaled, plain):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(round(e0.elapsed_time(e1) / reps, 4))
    for t, v in zip((opt._flat, opt._m, opt._v), saved):
        t.copy_(v)
    return {"check_gated_adam_update_ms": out[0], "plain_adam_ms": out[1], "bucket_floats": flat.numel()}


def gemm_classes(step):
    """one eager pass of the step's launch sequence with per-launch records: {class: (ms, TFLOP/s)}"""
    from graphinvent_b200._lib import lib
    torch.cuda.synchronize()
    lib.gib_profile_enable(1)
    try:
        step._enqueue_all()
        torch.cuda.synchronize()
        cap = 8192
        ms, work, cls = (ctypes.c_double * cap)(), (ctypes.c_double * cap)(), (ctypes.c_int * cap)()
        n = lib.gib_profile_records(ms, work, cls, cap)
        k = 5     # GIB_PROFILE_CLASSES
        lib.gib_profile_collect((ctypes.c_double * k)(), (ctypes.c_double * k)(), (ctypes.c_longlong * k)())   # clears
    finally:
        lib.gib_profile_enable(0)
    out = {}
    for c in (0, 1):
        t = sum(ms[i] for i in range(n) if cls[i] == c)
        w = sum(work[i] for i in range(n) if cls[i] == c)
        out[c] = (round(t, 4), round(w / (t * 1e-3) / 1e12, 2) if t > 0 else None)
    return out


def generation(mode, batches):
    from graphinvent_b200.config import make_constants
    from graphinvent_b200.gnn import mpnn
    from graphinvent_b200.graphed import GraphedGenerator
    C = make_constants("EMN")
    torch.manual_seed(0)
    net = mpnn.create(C).cuda().eval()
    with mode_ctx(mode):
        gen = GraphedGenerator(net, 1000, constants=C, n_atom_types=5, n_formal_charge=3)
    assert gen.autocast_dtype is DTYPE[mode]
    g = torch.Generator(device="cuda").manual_seed(7)
    U = torch.rand(2 * C.max_n_nodes, 1000, generator=g, device="cuda")
    gen.build_graphs(uniforms=U)                   # capture + warm-up
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(batches):
        gen.build_graphs(uniforms=U)
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / batches, 3), gen.rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--gen-batches", type=int, default=3)
    args = ap.parse_args()
    res = {"card": card(), "runs": []}
    import bench
    logits = {}
    for r in range(args.repeats):
        for mode in ("default", "bf16", "fp16"):
            row = {"repeat": r, "mode": mode}
            for cfg in ("C2", "C5T"):
                step, batch, net = train_step(cfg, mode)
                ms = time_steps(step, batch, args.steps, args.warmup)
                B = batch[0].shape[0]
                row[cfg] = {"ms_per_step": round(ms, 3), "graphs_per_s": round(B / ms * 1e3, 1),
                            "gemm_classes": gemm_classes(step)}
                if step.grad_scaler is not None:
                    row[cfg]["loss_scale"] = step.grad_scaler.get_scale()
                    row[cfg]["scaling"] = scaling_launches(step)
                del step, net
                if cfg == "C2" and r == 0:
                    C, nodes, edges, _, _ = bench.make_batch(cfg, seed=1002)
                    torch.manual_seed(0)
                    from graphinvent_b200.gnn import mpnn
                    fresh = mpnn.create(C).cuda()
                    with torch.no_grad(), mode_ctx(mode):
                        logits[mode] = fresh(nodes.cuda().float(), edges.cuda().float())
            row["C5_generation_ms_per_batch"], row["C5_rounds"] = generation(mode, args.gen_batches)
            res["runs"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    for mode in ("bf16", "fp16"):
        res[f"c2_logit_max_abs_diff_{mode}_vs_default"] = float((logits["default"] - logits[mode]).abs().max())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
