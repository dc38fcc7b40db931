"""GPU: the device-resident data loader (graphinvent_b200.loader.DeviceBlockLoader) and the whole passes that take it.

  1. gib_gather_rows against torch indexing plus cast, bit for bit: random int8 blocks with negative bytes, b in
     {0, 1, 7, B - 1, B}, both output dtypes, gdb13 dims and N = 38; padding rows exactly zero, ctl = {b, 1/b}; every
     buffer guarded; the refusals;
  2. plain iteration over the gdb13 fixture and over a 4-block set with a one-row last block: every batch equals the
     rows of the reference's order (tests/golden/loader_order.npz) widened to float32, and the default generator ends
     where the reference's pass leaves it, after a full and after a broken pass;
  3. TrainStep.train_epoch for the four models, float32 and int8 steps, OneCycleLR, two epochs: parameters, FlatAdam
     state, loss slots and mean bit-identical to a twin step fed host pinned batches in the same order; once more
     under fp16 autocast with a GradScaler; a one-block set is uploaded once;
  4. EvalStep.validation_epoch / validation_likelihood from the loader, alone and with share=, bit-identical to the
     host-fed passes in the same order, the early break and the generator state after it included;
  5. a batch over entry_capacity in the middle of an epoch makes train_epoch raise at its end;
  6. the device memory the loader adds over a 4-block epoch.
"""
import copy
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN, load_small
from tests.guarded import Guarded
from tests.test_gpu_partial_and_eval import _capacity

pytestmark = pytest.mark.gpu

FIXTURE = np.load(os.path.join(GOLDEN, "loader_order.npz"))
MODELS = ["GGNN", "MNN", "AttGGNN", "EMN"]


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous()


def _random_rows(n, N, F, Ef, apd, seed):
    g = np.random.default_rng(seed)
    return (g.integers(-128, 128, (n, N, F), dtype=np.int8), g.integers(-128, 128, (n, N, N, Ef), dtype=np.int8),
            g.integers(-128, 128, (n, apd), dtype=np.int8))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(13, 8, 3, 625), (38, 9, 4, 761)], ids=["gdb13", "N38"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.int8], ids=["f32", "i8"])
def test_gather_rows_matches_indexing(dims, out_dtype):
    from graphinvent_b200._lib import BatchCtl, check, lib
    N, F_, Ef, apd = dims
    rows_in_block, B = 300, 64
    blk = [torch.from_numpy(a) for a in _random_rows(rows_in_block, N, F_, Ef, apd, seed=N)]
    src = [Guarded.like(a) for a in blk]
    rb = (N * F_, N * N * Ef, apd)
    g = torch.Generator().manual_seed(3)
    for b in (0, 1, 7, B - 1, B):
        rows = torch.randperm(rows_in_block, generator=g)[:b].to(torch.int32)
        grow = Guarded.like(rows if b else torch.zeros(1, dtype=torch.int32))
        esz = 4 if out_dtype == torch.float32 else 1
        outs = [Guarded(B * rb[0] * esz), Guarded(B * rb[1] * esz), Guarded(B * rb[2] * 4)]
        ctl = Guarded(8)
        check(lib.gib_gather_rows(*(ctypes.c_void_p(s.ptr()) for s in src), ctypes.c_void_p(grow.ptr()), b, B, *rb,
                                  ctypes.c_void_p(outs[0].ptr()), ctypes.c_void_p(outs[1].ptr()),
                                  int(out_dtype == torch.int8), ctypes.c_void_p(outs[2].ptr()),
                                  ctypes.c_void_p(ctl.ptr()), _st()), "gib_gather_rows")
        torch.cuda.synchronize()
        idx = rows.long()
        for k, (a, o) in enumerate(zip(blk, outs)):
            dt = torch.float32 if k == 2 else out_dtype
            want = torch.zeros((B,) + tuple(a.shape[1:]), dtype=dt)
            want[:b] = a[idx].to(dt)
            got = o.view(dt, want.shape).cpu()
            assert torch.equal(_bits(got), _bits(want)), (b, k)
            assert (_bits(got[b:]) == 0).all()                           # padding rows: exact (+0) zeros
            assert o.intact(), (b, k, o.damage())
        c = BatchCtl.from_buffer_copy(bytes(ctl.t.cpu().numpy()))
        assert c.live == b and c.scale == (np.float32(1.0 / b) if b else 0.0)
        assert all(s.intact() for s in src) and grow.intact() and ctl.intact()
        # ctl may be NULL
        check(lib.gib_gather_rows(*(ctypes.c_void_p(s.ptr()) for s in src), ctypes.c_void_p(grow.ptr()), b, B, *rb,
                                  ctypes.c_void_p(outs[0].ptr()), ctypes.c_void_p(outs[1].ptr()),
                                  int(out_dtype == torch.int8), ctypes.c_void_p(outs[2].ptr()), None, _st()), "")
        torch.cuda.synchronize()
    # refusals
    p = [ctypes.c_void_p(s.ptr()) for s in src]
    o = [ctypes.c_void_p(x.ptr()) for x in outs]
    for args in ((*p, o[0], B + 1, B, *rb, o[0], o[1], 0, o[2], None, _st()),
                 (*p, o[0], 1, B, 0, rb[1], rb[2], o[0], o[1], 0, o[2], None, _st()),
                 (*p, o[0], 1, B, *rb, None, o[1], 0, o[2], None, _st()),
                 (*p, o[0], 1, B, *rb, ctypes.c_void_p(outs[0].ptr() + 1), o[1], 0, o[2], None, _st())):
        assert lib.gib_gather_rows(*args) < 0


# ---------------------------------------------------------------------------------------------------------------------
# 2. plain iteration
# ---------------------------------------------------------------------------------------------------------------------
def _fixture_case(rows, batch, block, stop):
    for i in range(len([k for k in FIXTURE.files if k.endswith("/params")])):
        p = [int(v) for v in FIXTURE[f"case{i}/params"]]
        if (p[0], p[1], p[2], p[6]) == (rows, batch, block, stop):
            return (p, FIXTURE[f"case{i}/sizes"], FIXTURE[f"case{i}/indices"], FIXTURE[f"case{i}/rand"],
                    int(FIXTURE[f"case{i}/len"]))
    raise KeyError((rows, batch, block, stop))


def _gdb13():
    from graphinvent_b200 import data
    return data.read_hdf5_raw(os.path.join(GOLDEN, "gdb13_train_head256.h5"), 13, 8, 3, 625)


@pytest.mark.parametrize("which", ["gdb13_head256", "synthetic_4_blocks"])
def test_plain_iteration_equals_the_reference_order(which):
    from graphinvent_b200.loader import DeviceBlockLoader
    rows = 256 if which == "gdb13_head256" else 301
    arrays = _gdb13() if which == "gdb13_head256" else _random_rows(301, 13, 8, 3, 625, seed=5)
    ds = types.SimpleNamespace(nodes=arrays[0], edges=arrays[1], apds=arrays[2])
    loader = DeviceBlockLoader(ds, batch_size=32, block_size=100)
    for stop in (-1, 4 if rows == 256 else 5):
        params, sizes, indices, rand, n_batches = _fixture_case(rows, 32, 100, stop)
        assert len(loader) == n_batches
        torch.manual_seed(params[5])
        off = 0
        for idx, (n, e, t) in enumerate(loader):
            if idx == stop:
                break
            assert n.is_cuda and n.dtype == e.dtype == t.dtype == torch.float32
            if sizes[idx] < 0:                                # the one-row last block: one molecule (the deviation)
                sel = np.array([rows - 1])
            else:
                sel = indices[off:off + sizes[idx]]
                off += sizes[idx]
            for got, a in zip((n, e, t), arrays):
                assert torch.equal(_bits(got.cpu()), _bits(torch.from_numpy(a[sel]).float()))
        assert idx == (len(sizes) - 1 if stop < 0 else stop)
        assert np.array_equal(torch.rand(4).numpy(), rand)


# ---------------------------------------------------------------------------------------------------------------------
# 3. train_epoch
# ---------------------------------------------------------------------------------------------------------------------
def _tiled_set(model, reps, seed):
    """the small_<model> fixture's molecules tiled `reps` times, with seeded one-hot int8 targets"""
    fx = load_small(model)
    nodes = fx["nodes"].to(torch.int8).repeat(reps, 1, 1).numpy()
    edges = fx["edges"].to(torch.int8).repeat(reps, 1, 1, 1).numpy()
    n, apd = nodes.shape[0], fx["target"].shape[1]
    apds = np.zeros((n, apd), np.int8)
    apds[np.arange(n), np.random.default_rng(seed).integers(0, apd, n)] = 1
    return fx, types.SimpleNamespace(nodes=nodes, edges=edges, apds=apds)


def _net(fx):
    from graphinvent_b200.gnn import mpnn
    net = mpnn.create(fx["C"])
    net.load_state_dict(fx["sd"])
    return net.cuda()


def _host_batches(loader, ds, in_dtype):
    """the loader's order (drawn now), as pinned host batches"""
    for k, ix in loader.order():
        sel = (ix + k * loader.block_size).numpy()
        n, e = torch.from_numpy(ds.nodes[sel]), torch.from_numpy(ds.edges[sel])
        if in_dtype == torch.float32:
            n, e = n.float(), e.float()
        yield n.pin_memory(), e.pin_memory(), torch.from_numpy(ds.apds[sel]).float().pin_memory()


def _pair(fx, ds, in_dtype, B, cap, scaler_kw=None):
    """(step, scheduler) twice: two equal models with FlatAdam and OneCycleLR"""
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    out = []
    base = _net(fx)
    for _ in range(2):
        net = copy.deepcopy(base)
        opt = FlatAdam(net.parameters(), lr=1e-3)
        sch = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=1e-2, total_steps=1000)
        scaler = torch.amp.GradScaler("cuda", **scaler_kw) if scaler_kw is not None else None
        step = TrainStep(net, opt, batch_size=B, entry_capacity=cap, input_dtype=in_dtype, grad_scaler=scaler)
        out.append((step, sch, scaler))
    return out


def _assert_same_training(a, b):
    for p, q in zip(a.model.parameters(), b.model.parameters()):
        assert torch.equal(_bits(p.detach()), _bits(q.detach()))
    for x, y in ((a.optimizer._m, b.optimizer._m), (a.optimizer._v, b.optimizer._v)):
        assert torch.equal(_bits(x), _bits(y))
    a.optimizer._pull_steps()
    b.optimizer._pull_steps()
    assert a.optimizer._steps == b.optimizer._steps


def _run_pair(fx, ds, in_dtype, block, B=24, epochs=2, scaler_kw=None, autocast=None):
    from graphinvent_b200.loader import DeviceBlockLoader
    cap = _capacity(fx["edges"].cuda(), fx["C"])
    if autocast is not None:
        with torch.autocast("cuda", dtype=autocast):
            (dev, sch_d, _), (host, sch_h, _) = _pair(fx, ds, in_dtype, B, cap, scaler_kw)
    else:
        (dev, sch_d, _), (host, sch_h, _) = _pair(fx, ds, in_dtype, B, cap, scaler_kw)
    loader = DeviceBlockLoader(ds, batch_size=B, block_size=block)
    for epoch in range(epochs):
        torch.manual_seed(100 + epoch)
        got = dev.train_epoch(loader, sch_d)
        rand_d = torch.rand(4)
        torch.manual_seed(100 + epoch)
        slots = torch.zeros(len(loader), device="cuda")
        for idx, (n, e, t) in enumerate(_host_batches(loader, ds, in_dtype)):
            slots[idx:idx + 1].copy_(host(n, e, t).view(1))
            sch_h.step()
        host.check()
        want = torch.mean(slots)
        assert torch.equal(torch.rand(4), rand_d)
        assert torch.equal(_bits(got.view(1)), _bits(want.view(1))), (epoch, float(got), float(want))
        _assert_same_training(dev, host)
    return dev, loader


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("in_dtype", [torch.float32, torch.int8], ids=["f32", "i8"])
def test_train_epoch_equals_host_fed_steps(model, in_dtype):
    fx, ds = _tiled_set(model, reps=7, seed=1)            # 224 rows, block 64: 4 blocks, short batches in each
    _, loader = _run_pair(fx, ds, in_dtype, block=64)
    assert loader.n_blocks == 4


def test_train_epoch_fp16_autocast_with_grad_scaler():
    fx, ds = _tiled_set("GGNN", reps=5, seed=2)
    dev, _ = _run_pair(fx, ds, torch.float32, block=64, scaler_kw=dict(init_scale=2.0 ** 12),
                       autocast=torch.float16)
    assert dev.grad_scaler is not None and dev.autocast_dtype == torch.float16


def test_one_block_set_is_uploaded_once():
    fx, ds = _tiled_set("GGNN", reps=2, seed=3)           # 64 rows: one block
    _, loader = _run_pair(fx, ds, torch.int8, block=100)
    assert loader.n_blocks == 1 and loader.uploads == 1


def test_train_epoch_refusals():
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.loader import DeviceBlockLoader
    from graphinvent_b200.optim import FlatAdam
    fx, ds = _tiled_set("GGNN", reps=2, seed=4)
    net = _net(fx)
    step = TrainStep(net, FlatAdam(net.parameters()), batch_size=24, entry_capacity=_capacity(fx["edges"].cuda(),
                                                                                             fx["C"]))
    with pytest.raises(TypeError):
        step.train_epoch([(fx["nodes"], fx["edges"], fx["target"])])
    with pytest.raises(ValueError, match="batch size"):
        step.train_epoch(DeviceBlockLoader(ds, batch_size=16, block_size=64))
    other = types.SimpleNamespace(nodes=ds.nodes[:, :6, :], edges=ds.edges[:, :6, :6], apds=ds.apds)
    with pytest.raises(ValueError, match="dims"):
        step.train_epoch(DeviceBlockLoader(other, batch_size=24, block_size=64))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the validation passes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("share", [False, True], ids=["alone", "share"])
@pytest.mark.parametrize("model", ["GGNN", "EMN"])
def test_validation_passes_from_the_loader(model, share):
    from graphinvent_b200.graphed import EvalStep, TrainStep
    from graphinvent_b200.loader import DeviceBlockLoader
    from graphinvent_b200.optim import FlatAdam
    fx, ds = _tiled_set(model, reps=7, seed=6)
    B = 24
    cap = _capacity(fx["edges"].cuda(), fx["C"])
    net = _net(fx)
    step = TrainStep(net, FlatAdam(net.parameters()), batch_size=B, entry_capacity=cap) if share else None
    ev = EvalStep(net, batch_size=B, entry_capacity=cap, share=step)
    loader = DeviceBlockLoader(ds, batch_size=B, block_size=64)
    torch.manual_seed(7)
    got = ev.validation_epoch(loader)
    torch.manual_seed(7)
    want = ev.validation_epoch(list(_host_batches(loader, ds, torch.float32)))
    assert torch.equal(_bits(got.view(1)), _bits(want.view(1)))
    for n_samples in (10 ** 6, 2 * B - 1):                 # a full pass, and a pass broken at batch 2
        torch.manual_seed(8)
        lik, avg = ev.validation_likelihood(loader, n_samples)
        batches_d, rand_d = ev.batches, torch.rand(4)
        torch.manual_seed(8)
        lik2, avg2 = ev.validation_likelihood(_host_batches(loader, ds, torch.float32), n_samples)
        assert ev.batches == batches_d and torch.equal(torch.rand(4), rand_d)
        assert torch.equal(_bits(lik), _bits(lik2)) and torch.equal(_bits(avg), _bits(avg2))
    assert batches_d == 2


# ---------------------------------------------------------------------------------------------------------------------
# 5. an overflow in the middle of an epoch
# ---------------------------------------------------------------------------------------------------------------------
def test_overflow_mid_epoch_raises_at_the_end():
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.loader import DeviceBlockLoader
    fx, ds = _tiled_set("GGNN", reps=7, seed=9)
    N = ds.edges.shape[1]
    ds.edges[64:] = 0                                      # blocks 2..4: complete graphs of one bond type
    ds.edges[64:, :, :, 0] = 1 - np.eye(N, dtype=np.int8)
    cap = _capacity(fx["edges"][:1].cuda(), fx["C"])      # fits the first block's batches, not the complete graphs
    assert 24 * N * (N - 1) > cap
    net = _net(fx)
    step = TrainStep(net, torch.optim.SGD(net.parameters(), lr=0.0), batch_size=24, entry_capacity=cap)
    counter = types.SimpleNamespace(n=0)
    sch = types.SimpleNamespace(step=lambda: setattr(counter, "n", counter.n + 1))
    loader = DeviceBlockLoader(ds, batch_size=24, block_size=64)
    torch.manual_seed(0)
    with pytest.raises(RuntimeError, match="entry_capacity"):
        step.train_epoch(loader, sch)
    assert counter.n == len(loader)                        # every batch ran: the error comes at the end


# ---------------------------------------------------------------------------------------------------------------------
# 6. memory
# ---------------------------------------------------------------------------------------------------------------------
def test_loader_memory_is_two_blocks():
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.loader import DeviceBlockLoader
    from graphinvent_b200.optim import FlatAdam
    fx, ds = _tiled_set("GGNN", reps=64, seed=10)         # 2048 rows, block 512: 4 blocks
    net = _net(fx)
    step = TrainStep(net, FlatAdam(net.parameters()), batch_size=32,
                     entry_capacity=_capacity(fx["edges"].cuda(), fx["C"]))
    fx_n, fx_e, fx_t = (x.cuda() for x in (fx["nodes"], fx["edges"], fx["target"]))
    step(fx_n, fx_e, fx_t)                                 # FlatAdam flattens the parameters at its first step
    loader = DeviceBlockLoader(ds, batch_size=32, block_size=512)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(0)
    step.train_epoch(loader)
    torch.cuda.synchronize()
    block_bytes = 512 * sum(loader.row_bytes)
    margin = 256 * 1024                                    # row indices, loss slots, flags, allocator rounding
    assert loader.n_blocks == 4 and loader.uploads == 4
    assert torch.cuda.max_memory_allocated() - base <= 2 * block_bytes + margin
    assert sum(t.numel() for slot in loader._slots for t in slot) == 2 * block_bytes
