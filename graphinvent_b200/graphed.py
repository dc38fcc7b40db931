"""
One training step of the hot path as ONE CUDA-graph launch (SURVEY.md 8b: "no host sync, static capacities,
CUDA-graph capturable").

    step = graphinvent_b200.graphed.TrainStep(model, optimizer, batch_size=B, entry_capacity=E_cap)
    for nodes, edges, target in loader:              # host (pinned) or device tensors, float32 or int8
        loss = step(nodes, edges, target)            # device scalar; float(loss) when the host wants it
        ...
    step.check()                                     # raises if a batch exceeded the capacity (one 64-byte read)

or, over a `loader.DeviceBlockLoader`, a whole epoch with one gather launch per batch and no host copies:

    loss = step.train_epoch(loader, scheduler)       # Workflow.train_epoch's return value

replaces the body of `Workflow.train_epoch` (Workflow.py:781-796: batch -> device, `model(nodes, edges)`, `loss`,
`zero_grad`, `backward`, `optimizer.step`) by: three copies into static input buffers, one graph launch
(K0 -> weight packing -> forward -> fused KL loss -> explicit backward into ONE flat gradient bucket), the
data-parallel all-reduce when a process group is given, and the optimizer step.  Capacity mode (functional.GraphBatch)
keeps every data-dependent extent in device memory, so the captured launch parameters never depend on the batch
content; a batch with more bond entries than `entry_capacity` is truncated and flagged, `check()` reports it.

The optimizer is stepped eagerly after the graph (its learning-rate schedule is host state, and so is its step count
unless a gradient scaler is given); with `optim.FlatAdam` that is one more launch.  There is no CPU path.  A batch may hold fewer than `batch_size` molecules
(the tail batch of each block of the reference's loader): the live count and the loss scale are device memory
(`gib_batch_ctl`), so the same graph serves it.

The validation pass (`Workflow.validation_epoch`, `Analyzer.get_validation_likelihood`) as replays of one captured
graph per batch (`EvalStep`), optionally on a TrainStep's buffers:

    ev = graphinvent_b200.graphed.EvalStep(model, batch_size=B, entry_capacity=E_cap, share=step)
    val_loss = ev.validation_epoch(valid_loader)
    lik, avg = ev.validation_likelihood(loader, n_samples)

Generation rounds as replays of ONE captured round (`GraphedGenerator`, a drop-in for `generation.GraphGenerator`):

    gen = graphinvent_b200.graphed.GraphedGenerator(model, batch_size=1000)
    graphs, flat, final, proper = gen.sample(generator=g)     # what GraphGenerator.sample returns

The captured round is K0 -> forward -> `gib_generation_sample_round`, whose round index, uniforms row and stop rule
live in device memory, so the host replays the same graph until a status copied back asynchronously says the batch
is done; it keeps two rounds in flight and never waits on the round it just launched.

The RL rollout of `Workflow.learning_step` as replays of captured rounds (`GraphedGeneratorRL`, a drop-in for
`generation.GraphGeneratorRL`):

    gen = graphinvent_b200.graphed.GraphedGeneratorRL(agent, batch_size=1000)      # once
    graphs, agent_ll, prior_ll, proper = gen.sample(agent, prior)                # per rollout; autograd tensors

Each rollout keeps only the int8 input of every round; `loss.backward()` recomputes each round's forward before its
backward, one captured backward round per model that needs gradients.

The likelihood of molecules under a model, p(action | state) over each molecule's decoding route, as replays of one
captured fill -> K0 -> forward -> probability graph per batch of route states (`RouteScorer`):

    lik, offsets, nll, final = graphinvent_b200.graphed.RouteScorer(model, batch_size=1000).score(nodes, edges)

With `score(nodes, edges, requires_grad=True)` they are autograd tensors; the backward recomputes each batch's forward
in a second captured graph, as the RL backward does.

Matmul precision: each of these objects reads torch's float32 matmul precision once, at construction
(`config.tf32_enabled`, exposed as its `tf32` attribute), and bakes it into its graphs -- single-pass TF32 GEMMs when
the user allowed TF32, 3xTF32 otherwise -- as torch's own captured cuBLAS calls keep the math mode of their capture.
Changing the setting afterwards does not change what a replay computes (the RL backward rounds included); build a new
object to switch.  The same holds for `torch.autocast("cuda", dtype=torch.bfloat16 | torch.float16)`: built inside
such a context, an object runs its tensor-core GEMMs on bf16 / fp16 operands (`config.matmul_code`; exposed as its
`autocast_dtype`, None otherwise) whether or not later replays run inside one.  `TrainStep` without a gradient scaler
honours bf16 only: built under fp16 autocast it keeps the fp32-input precision (`autocast_dtype` None), because
unscaled fp16 gradients underflow.  With `grad_scaler=` an enabled `torch.amp.GradScaler("cuda")` and a `FlatAdam`, it
takes every mode, fp16 included, and runs torch's dynamic loss scaling on the device:

    scaler = torch.amp.GradScaler("cuda")
    with torch.autocast("cuda", dtype=torch.float16):
        step = graphinvent_b200.graphed.TrainStep(model, FlatAdam(model.parameters()), B, E_cap, grad_scaler=scaler)

Each step then equals, bit for bit, the eager `scaler.scale(loss).backward(); scaler.step(opt); scaler.update()`: the
loss gradient is multiplied by the scaler's scale inside the fused loss, a check over the gradient bucket sets
`step.found_inf`, and `FlatAdam.scaled_step` skips or takes the Adam step and updates the scaler's own `_scale` /
`_growth_tracker` tensors, all in stream order without a host read.
"""
import ctypes
import types
from collections import namedtuple

import numpy as np
import torch

from . import functional as F
from .config import matmul_code
from ._lib import (CONS_OVER_MAX, CONS_SMALL_RING, CONS_UNDER_MIN, FLAG_MULTITYPE, FLAG_OVERFLOW, HDR_FLAGS,
                   HDR_INTS, PP_STATUS_INTS, ROUTE_ACTION, ROUTE_BAD_ID, ROUTE_MASKED, ROUTE_NOT_PREFIX, EvalPass, check,
                   lib)
from .generation import GraphGenerator, _LogitMasks, _mask_logits

_u8 = torch.uint8


def _set_ctl(ctl, live, denominator):
    """gib_batch_ctl {live, 1 / denominator} by device-side fills: no host buffer that a queued copy could still read,
    no synchronisation"""
    ctl[0:1].fill_(live)
    ctl[1:2].view(torch.float32).fill_(1.0 / denominator if denominator > 0 else 0.0)


def _batch_rows(step, name, nodes, edges, target):
    b = nodes.shape[0]
    if not 0 <= b <= step.B:
        raise ValueError(f"{name} was built for batches of up to {step.B} molecules, got {b}")
    if edges.shape[0] != b or target.shape[0] != b:
        raise ValueError(f"nodes, edges and target hold {b}, {edges.shape[0]} and {target.shape[0]} molecules")
    return b


def _load_rows(step, b, nodes, edges, target):
    """rows [0, b) of the static inputs from the batch (pinned host tensors: asynchronous H2D), rows [b, B) zeroed:
    empty molecules, which every model maps to finite logits"""
    for dst, src in ((step.nodes, nodes), (step.edges, edges), (step.target, target)):
        dst[:b].copy_(src, non_blocking=True)
        if b < step.B:
            dst[b:].zero_()


_SCALER_STATE = ("_scale", "_growth_tracker", "_growth_factor", "_backoff_factor", "_growth_interval",
                 "_lazy_init_scale_growth_tracker")


def _grad_scaler(scaler, optimizer):
    """the scaler TrainStep runs with: None without one or for a disabled one; refuses what it cannot run"""
    if scaler is None:
        return None
    if not isinstance(scaler, torch.amp.GradScaler):
        raise TypeError(f"grad_scaler must be a torch.amp.GradScaler, got {type(scaler).__name__}")
    if not scaler.is_enabled():
        return None
    if getattr(scaler, "_device", "cuda") != "cuda":
        raise ValueError("grad_scaler must be a CUDA GradScaler: torch.amp.GradScaler(\"cuda\")")
    from .optim import FlatAdam
    if not isinstance(optimizer, FlatAdam):
        raise ValueError("TrainStep(grad_scaler=) needs a graphinvent_b200.optim.FlatAdam optimizer (its step is gated "
                         f"and unscaled on the device), got {type(optimizer).__name__}")
    missing = [a for a in _SCALER_STATE if not hasattr(scaler, a)]
    if missing:
        raise RuntimeError(f"this torch's GradScaler lacks {missing}: TrainStep(grad_scaler=) updates the scaler's "
                           "scale and growth-tracker tensors in place and cannot run with it")
    return scaler


# ---- the static model call of the captured objects ------------------------------------------------------------
def _static_dims(obj, model, batch, in_dtype, tf32=None):
    """obj.d for a static call of `model` on its CUDA parameters, checked against the parameter table, and the
    precision attributes obj.tf32 / obj.autocast_dtype: torch's matmul precision at construction unless `tf32` is
    given, baked into the object's graphs; returns the parameter table"""
    params = list(model.parameters())
    F._require_cuda(*params)
    obj.d = F.make_dims(model, batch, in_dtype, tf32=tf32)
    obj.tf32 = obj.d.tf32 == 1
    obj.autocast_dtype = F.autocast_dtype_of(obj.d)
    F._check_params(model, obj.d, params)
    return params


def _static_inputs(d, dev):
    """zeroed static nodes / edges (int8 for int8 batches, float32 otherwise) and target of dims d"""
    dt = torch.int8 if d.in_dtype else torch.float32
    return (torch.zeros(d.B, d.N, d.F, dtype=dt, device=dev), torch.zeros(d.B, d.N, d.N, d.Ef, dtype=dt, device=dev),
            torch.zeros(d.B, d.N * (d.f_add + d.f_conn) + 1, dtype=torch.float32, device=dev))


def _model_buffers(d, edges, capacity):
    """the static buffers of a capacity-mode model call on `edges`, sized by a probe GraphBatch: (cws, gbuf, hdr_np,
    hdr, ws, workspace_bytes) -- K0's count workspace, graph buffer and host header, and the forward workspace.  The
    caller allocates the packed arena(s)."""
    probe = F.GraphBatch(d, edges, capacity=capacity)
    ws = F._workspace(d, probe.hdr, edges.device)
    return probe.cws, probe.buf, probe.hdr_np, probe.hdr, ws, ws.numel()


def _k0_forward(s, nodes, edges, runs, st, params=None):
    """K0 on `edges` into s.cws / s.gbuf, then one forward on s.ws per (packed arena, logits) pair of `runs`;
    `params`: a parameter table packed into the first arena between the two (the training step repacks every step)"""
    bd = ctypes.byref(s.d)
    check(lib.gib_graph_count(bd, F._ptr(edges), F._ptr(s.cws), st), "gib_graph_count")
    check(lib.gib_graph_fill(bd, F._ptr(edges), F._ptr(s.cws), s.hdr, F._ptr(s.gbuf), st), "gib_graph_fill")
    if params is not None:
        check(lib.gib_model_pack(bd, F._ptr_table(params), F._ptr(runs[0][0]), st), "gib_model_pack")
    for packed, out in runs:
        check(lib.gib_model_forward(bd, s.hdr, F._ptr(nodes), F._ptr(edges), F._ptr(s.gbuf), F._ptr(packed),
                                    F._ptr(s.ws), F._ptr(out), st), "gib_model_forward")


def _capture(dev, enqueues):
    """one CUDA graph per enqueue function, in order.  All of them run once first, in order, on a side stream and
    outside capture (lazy per-device init, function attributes)."""
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for enqueue in enqueues:
            enqueue()
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    graphs = []
    for enqueue in enqueues:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            enqueue()
        graphs.append(g)
    return graphs


def _check_flags(flags, d, overflow):
    """raises the error of the K0 `flags` of a model call with dims d (`overflow`: the caller's message for a batch
    over the entry capacity); returns the flags"""
    if flags & FLAG_OVERFLOW:
        raise RuntimeError(overflow)
    if flags & FLAG_MULTITYPE and d.model == F.MODEL_ID["AttGGNN"]:
        raise RuntimeError("AttentionGGNN requires one bond type per bond (as the reference's AggregationMPNN does)")
    return flags


def _device_loader(obj, loader, name):
    """True for a DeviceBlockLoader whose batches fit `obj`'s static inputs; raises for one that does not"""
    from .loader import DeviceBlockLoader
    if not isinstance(loader, DeviceBlockLoader):
        return False
    d = obj.d
    if (loader.batch_size != obj.B or (loader.N, loader.F, loader.Ef, loader.apd) != (d.N, d.F, d.Ef, obj.apd)
            or loader.device != torch.device(obj.dev)):
        raise ValueError(f"{name} needs a DeviceBlockLoader of the step's batch size {obj.B}, dims (N, F, Ef, apd) = "
                         f"{(d.N, d.F, d.Ef, obj.apd)} and device {obj.dev}; got batch size {loader.batch_size}, dims "
                         f"{(loader.N, loader.F, loader.Ef, loader.apd)} on {loader.device}")
    return True


class TrainStep:
    @staticmethod
    def precision_code(grad_scaler=None):
        """the matmul precision code a TrainStep built now bakes in: torch's autocast / TF32 state, except that fp16
        autocast counts only with an enabled gradient scaler"""
        if grad_scaler is not None and grad_scaler.is_enabled():
            return matmul_code()
        return matmul_code(fp16=False)

    def __init__(self, model, optimizer, batch_size, entry_capacity, input_dtype=torch.float32, global_batch=None,
                 group=None, device=None, warmup=True, grad_scaler=None):
        self.grad_scaler = _grad_scaler(grad_scaler, optimizer)
        self.B = int(batch_size)
        self.code = 1 if input_dtype == torch.int8 else 0
        # fp16 autocast only with a gradient scaler: unscaled fp16 gradients underflow
        self.params = params = _static_dims(self, model, self.B, self.code, tf32=self.precision_code(self.grad_scaler))
        self.model, self.optimizer = model, optimizer
        self.dev = dev = device or params[0].device
        self.global_batch = int(global_batch) if global_batch else self.B
        self.group = group
        self.capacity = int(entry_capacity)
        # static buffers (addresses are baked into the graph)
        self.nodes, self.edges, self.target = _static_inputs(self.d, dev)
        self.apd = self.target.shape[1]
        self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
            self.d, self.edges, self.capacity)
        self.packed = torch.empty(lib.gib_model_packed_bytes(ctypes.byref(self.d)), dtype=_u8, device=dev)
        self.scratch = torch.empty(lib.gib_model_bwd_scratch_bytes(ctypes.byref(self.d), self.hdr), dtype=_u8,
                                   device=dev)
        self.out = torch.empty(self.B, self.apd, dtype=torch.float32, device=dev)
        self.dout = torch.empty_like(self.out)
        self.rows = torch.empty(self.B, dtype=torch.float32, device=dev)
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        # gib_batch_ctl {live, scale}: the captured loss kernels read the live molecule count and the loss scale here
        self.ctl = torch.zeros(2, dtype=torch.int32, device=dev)
        _set_ctl(self.ctl, self.B, self.global_batch)
        total = sum(p.numel() for p in params)
        self.gflat = torch.zeros(total, dtype=torch.float32, device=dev)   # ONE bucket: grads are views of it
        self.views = F._bucket_views(self.gflat, params)
        for p, v in zip(params, self.views):
            p.grad = v
        # dynamic loss scaling: 1.0 when the last step's gradient bucket held an inf or NaN (that step was skipped)
        self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        if self.grad_scaler is not None:
            if self.grad_scaler._scale is None:
                self.grad_scaler._lazy_init_scale_growth_tracker(dev)
            optimizer.device_step_counts()
        # data parallel: the gradients of the readout parameters (gather.*, APDReadout.*: the tail of the parameter
        # order, 79 % of the bucket) are final after the first part of the backward; their all-reduce runs on a side
        # stream while the message-passing backward (second captured graph) still executes (SURVEY.md 8e)
        self.world = 1
        if group is not False and torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(group)
        self.tail_off = total
        if self.world > 1:
            names = [n for n, _ in model.named_parameters()]
            i = len(names)
            while i > 0 and names[i - 1].startswith(("gather.", "APDReadout.")):
                i -= 1
            self.tail_off = sum(p.numel() for p in params[:i])
            self.comm_stream = torch.cuda.Stream(dev)
        self.graph = None
        self.graph2 = None
        self.steps = 0
        self._param_ptrs = None
        if warmup:
            self.capture()

    # ---- the captured region ------------------------------------------------------------------------------
    def _enqueue(self):
        st = F._stream(self.dev)
        _k0_forward(self, self.nodes, self.edges, [(self.packed, self.out)], st, params=self.params)
        # Workflow.loss (Workflow.py:833-860) over the live rows, the batch-mean taken over ctl's denominator (the
        # GLOBAL batch of data-parallel shards); padding rows get dout = 0 and add exact zeros to every gradient
        if self.grad_scaler is None:
            check(lib.gib_kl_loss_fwd_bwd_ctl(F._ptr(self.out), F._ptr(self.target), self.B, self.apd,
                                              F._ptr(self.ctl), F._ptr(self.rows), F._ptr(self.dout), st),
                  "gib_kl_loss_fwd_bwd_ctl")
        else:
            # scaler.scale(loss).backward(): the loss gradient times the scaler's current scale, read on the device
            check(lib.gib_fill_zero(F._ptr(self.found_inf), 4, st), "gib_fill_zero")
            check(lib.gib_kl_loss_fwd_bwd_ctl_scaled(F._ptr(self.out), F._ptr(self.target), self.B, self.apd,
                                                     F._ptr(self.ctl), F._ptr(self.grad_scaler._scale),
                                                     F._ptr(self.rows), F._ptr(self.dout), st),
                  "gib_kl_loss_fwd_bwd_ctl_scaled")
        check(lib.gib_sum_scaled_ctl(F._ptr(self.rows), self.B, F._ptr(self.ctl), F._ptr(self.loss), st),
              "gib_sum_scaled_ctl")
        check(lib.gib_fill_zero(F._ptr(self.gflat), self.gflat.numel() * 4, st), "gib_fill_zero")
        self._backward(1 if self.world > 1 else 0)
        if self.grad_scaler is not None and self.world == 1:
            self._check_grads()

    def _check_grads(self):
        """found_inf = 1 if the (all-reduced) gradient bucket holds an inf or NaN: the last node of the captured graph on
        one GPU; after both all-reduces, outside the graphs, with a process group, so that every rank sees the same
        bucket and skips the same steps"""
        check(lib.gib_nonfinite_check(F._ptr(self.gflat), self.gflat.numel(), F._ptr(self.found_inf),
                                      F._stream(self.dev)), "gib_nonfinite_check")

    def _backward(self, part):
        st = F._stream(self.dev)
        check(lib.gib_model_backward_part(ctypes.byref(self.d), self.hdr, F._ptr(self.nodes), F._ptr(self.edges),
                                          F._ptr(self.gbuf), F._ptr(self.packed), F._ptr(self.ws),
                                          F._ptr(self.out), F._ptr(self.dout), F._ptr_table(self.views),
                                          F._ptr(self.scratch), part, st), "gib_model_backward_part")

    def _enqueue_all(self):
        """the whole step's launch sequence, eagerly (warm-up, kernel-class timing)"""
        self._enqueue()
        if self.world > 1:
            self._backward(2)

    def capture(self):
        """(re)capture; called by the constructor and again if the parameters were moved (e.g. by FlatAdam).  The
        warm-up runs `_enqueue_all`'s sequence."""
        if self.world > 1:
            self.graph, self.graph2 = _capture(self.dev, [self._enqueue, lambda: self._backward(2)])
        else:
            self.graph, = _capture(self.dev, [self._enqueue])
        self._param_ptrs = self._captured_ptrs()

    def _captured_ptrs(self):
        """the addresses the graphs read that live outside this object: the parameters and the scaler's scale"""
        ptrs = [p.data_ptr() for p in self.params]
        if self.grad_scaler is not None:
            if self.grad_scaler._scale is None:
                self.grad_scaler._lazy_init_scale_growth_tracker(self.dev)
            ptrs.append(self.grad_scaler._scale.data_ptr())
        return ptrs

    # ---- one step -----------------------------------------------------------------------------------------
    def load(self, nodes, edges, target, global_batch=None):
        """copy one batch of 0 <= b <= batch_size molecules into the static input buffers (pinned host tensors:
        asynchronous H2D).  A short batch -- the tail batch of every block of the reference's BlockDataLoader -- fills
        rows [0, b); rows [b, batch_size) become empty molecules whose loss rows and gradients are exact zeros.  The
        loss is the batch mean over `global_batch` molecules: by default batch_size's `global_batch` for a full batch
        and b for a short one (KLDivLoss(batchmean) on a b-row batch).  A data-parallel rank passes the global size
        of a short global batch; a rank whose shard is empty runs with b = 0 and still joins the all-reduce."""
        b = _batch_rows(self, "TrainStep", nodes, edges, target)
        if global_batch is None:
            if b < self.B and self.world > 1:
                raise ValueError("a short batch on a data-parallel rank needs the global batch size: "
                                 "load(..., global_batch=<molecules over all ranks>)")
            global_batch = self.global_batch if b == self.B else b
        _load_rows(self, b, nodes, edges, target)
        _set_ctl(self.ctl, b, int(global_batch))

    def __call__(self, nodes=None, edges=None, target=None, global_batch=None):
        if nodes is not None:
            self.load(nodes, edges, target, global_batch=global_batch)
        if self._captured_ptrs() != self._param_ptrs:
            self.capture()                        # the parameters moved (optimizer re-flattened them)
        for p, v in zip(self.params, self.views):
            if p.grad is not v:
                p.grad = v                        # zero_grad(set_to_none=True) of the reference loop (Workflow.py:787)
        self.graph.replay()
        if self.world > 1:
            # per-rank gradients are already scaled by 1/global_batch: a plain sum is the global batch mean
            dist, cur = torch.distributed, torch.cuda.current_stream(self.dev)
            grp = self.group if self.group not in (None, False) else None
            self.comm_stream.wait_stream(cur)
            with torch.cuda.stream(self.comm_stream):          # readout gradients: overlapped with graph 2
                if self.tail_off < self.gflat.numel():
                    dist.all_reduce(self.gflat[self.tail_off:], op=dist.ReduceOp.SUM, group=grp)
            self.graph2.replay()                               # message-passing backward
            if self.tail_off > 0:
                dist.all_reduce(self.gflat[:self.tail_off], op=dist.ReduceOp.SUM, group=grp)
            cur.wait_stream(self.comm_stream)
            if self.grad_scaler is not None:
                self._check_grads()
        if self.grad_scaler is not None:
            self.optimizer.scaled_step(self.found_inf, self.grad_scaler)     # scaler.step(opt); scaler.update()
        else:
            self.optimizer.step()
        F.invalidate_packed_weights()
        self.steps += 1
        return self.loss

    def train_epoch(self, loader, scheduler=None):
        """Workflow.train_epoch (Workflow.py:774-798) over a `loader.DeviceBlockLoader`: per batch one gather launch
        into the static inputs (and `ctl`), the replay and the optimizer step as `__call__` runs them, then
        `scheduler.step()` if a scheduler is given, and the batch loss into slot idx of len(loader) zero-initialised
        device slots.  Returns their mean as a 0-d device tensor.  The K0 flags of every batch are OR-ed on the device
        and read once, at the end: a batch over the entry capacity (or a multi-type AttentionGGNN batch) anywhere in
        the epoch raises then, with check()'s message."""
        if not _device_loader(self, loader, "TrainStep.train_epoch"):
            raise TypeError(f"TrainStep.train_epoch takes a graphinvent_b200.loader.DeviceBlockLoader, got "
                            f"{type(loader).__name__}; feed other loaders batch by batch through step(nodes, edges, "
                            "target)")
        if self.world > 1 or self.global_batch != self.B:
            raise ValueError("TrainStep.train_epoch runs one process's whole batches: build the step without a "
                             "data-parallel group or global_batch")
        slots = torch.zeros(len(loader), dtype=torch.float32, device=self.dev)
        flags = torch.zeros(1, dtype=torch.int32, device=self.dev)
        hdr_flags = self.cws[: HDR_INTS * 4].view(torch.int32)[HDR_FLAGS:HDR_FLAGS + 1]
        for idx, item in enumerate(loader.batches()):
            if idx >= slots.numel():
                raise IndexError(f"the loader yielded more than len(loader) = {slots.numel()} batches")
            loader.gather(item, self.nodes, self.edges, self.target, self.ctl)
            loss = self()
            flags.bitwise_or_(hdr_flags)
            slots[idx:idx + 1].copy_(loss.view(1))
            if scheduler is not None:
                scheduler.step()
        _check_flags(int(flags.item()), self.d, f"a batch of the epoch held more bond entries than entry_capacity="
                     f"{self.capacity}; the results of that step are invalid -- rebuild TrainStep with a larger "
                     "capacity")
        return torch.mean(slots)

    def check(self):
        """synchronising read of the K0 flags of the LAST step; raises if it did not fit the capacity"""
        flags = int(self.cws[: 64].view(torch.int32).cpu()[HDR_FLAGS])
        return _check_flags(flags, self.d, f"a batch held more bond entries than entry_capacity={self.capacity}; "
                            "the results of that step are invalid -- rebuild TrainStep with a larger capacity")


# ---- the validation pass --------------------------------------------------------------------------------------
class EvalStep:
    """The validation pass as replays of ONE captured graph: K0 (capacity mode) -> forward -> KL loss rows
    (`gib_kl_loss_fwd_bwd_ctl`, no dout) -> NLL rows (`gib_validation_nll_ctl`) -> `gib_eval_collect`, which writes the
    batch's slot of the pass, compacts its non-NaN NLL rows into the likelihood buffer and counts its sub-graphs, all
    on the device.  No backward, scratch or gradient bucket.

        ev = graphinvent_b200.graphed.EvalStep(model, batch_size=B, entry_capacity=cap, share=step)
        val_loss = ev.validation_epoch(valid_loader)              # Workflow.validation_epoch's value
        lik, avg = ev.validation_likelihood(loader, n_samples)    # Analyzer.get_validation_likelihood's values
        ev.check()                                                # raises if a batch of the last pass overflowed

    The weights are packed once per pass, outside the graph, and a pass reads the device once, at its end.  Batches
    of 0 <= b <= batch_size molecules are taken as `TrainStep` takes them; a loader of another batch size would move
    the reference's write offsets (idx * batch_size), so it must yield at most `batch_size` molecules per batch.

    `share=` a TrainStep of equal dims, capacity and input dtype: the pass runs on the step's static inputs, K0 buffers,
    packed arena, forward workspace and logits, and allocates only its slots and its likelihood buffer.  The step's
    graph rewrites everything it reads from its inputs (the weights repacked included), so training results do not
    change; load the next batch into the step before its next replay.  The forward has no dropout: the model is
    evaluated as in eval mode, whatever its dropout_p."""

    def __init__(self, model, batch_size, entry_capacity, input_dtype=torch.float32, share=None, device=None):
        self.B = int(batch_size)
        self.code = 1 if input_dtype == torch.int8 else 0
        params = _static_dims(self, model, self.B, self.code)
        self.model = model
        self.dev = dev = device or params[0].device
        self.capacity = int(entry_capacity)
        C = model.constants
        self.N = C.max_n_nodes
        self.apd = self.N * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
        if share is not None:
            if (not isinstance(share, TrainStep) or F.key_of(share.d) != F.key_of(self.d)
                    or share.capacity != self.capacity or share.dev != torch.device(dev)):
                raise ValueError("EvalStep(share=) needs a TrainStep of equal model dims, batch size, entry capacity, "
                                 "input dtype, matmul precision and device")
            self._share = share               # keeps the step's host header alive
            for name in ("nodes", "edges", "target", "cws", "gbuf", "hdr_np", "hdr", "packed", "ws", "out",
                         "workspace_bytes"):
                setattr(self, name, getattr(share, name))
        else:
            self.nodes, self.edges, self.target = _static_inputs(self.d, dev)
            self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
                self.d, self.edges, self.capacity)
            self.packed = torch.empty(lib.gib_model_packed_bytes(ctypes.byref(self.d)), dtype=_u8, device=dev)
            self.out = torch.empty(self.B, self.apd, dtype=torch.float32, device=dev)
        self.rows = torch.zeros(self.B, dtype=torch.float32, device=dev)
        self.nll = torch.zeros(self.B, dtype=torch.float32, device=dev)
        self.ctl = torch.zeros(2, dtype=torch.int32, device=dev)
        _set_ctl(self.ctl, self.B, self.B)
        # gib_eval_pass: written from pinned memory at the start of a pass, read back once at its end
        self._pass = torch.zeros(ctypes.sizeof(EvalPass), dtype=_u8, device=dev)
        self._pass_host = torch.zeros(ctypes.sizeof(EvalPass), dtype=_u8, pin_memory=True)
        self._pass_copied = torch.cuda.Event()
        self.flags, self.clipped, self.batches = 0, 0, 0
        self.graph = None
        self.capture()

    def _enqueue(self):
        st = F._stream(self.dev)
        _k0_forward(self, self.nodes, self.edges, [(self.packed, self.out)], st)
        check(lib.gib_kl_loss_fwd_bwd_ctl(F._ptr(self.out), F._ptr(self.target), self.B, self.apd, F._ptr(self.ctl),
                                          F._ptr(self.rows), None, st), "gib_kl_loss_fwd_bwd_ctl")
        check(lib.gib_validation_nll_ctl(F._ptr(self.out), F._ptr(self.target), self.B, self.apd, F._ptr(self.ctl),
                                         F._ptr(self.nll), st), "gib_validation_nll_ctl")
        check(lib.gib_eval_collect(F._ptr(self.rows), F._ptr(self.nll), F._ptr(self.target), self.B, self.apd,
                                   F._ptr(self.ctl), F._ptr(self.cws), F._ptr(self._pass), st), "gib_eval_collect")

    def capture(self):
        """the warm-up's pass state is overwritten by the next pass's start"""
        self.graph, = _capture(self.dev, [self._enqueue])

    # ---- one pass -----------------------------------------------------------------------------------------
    def _begin(self, slots, lik):
        params = list(self.model.parameters())
        F._require_cuda(*params)
        F._check_params(self.model, self.d, params)
        st = F._stream(self.dev)
        check(lib.gib_model_pack(ctypes.byref(self.d), F._ptr_table(params), F._ptr(self.packed), st),
              "gib_model_pack")
        desc = EvalPass(batch_loss=slots.data_ptr() if slots.numel() else None,
                        lik=lik.data_ptr() if lik is not None and lik.numel() else None,
                        lik_len=lik.numel() if lik is not None else 0, n_slots=slots.numel())
        self._pass_copied.synchronize()            # the previous pass's copy has read the pinned buffer
        self._pass_host.copy_(torch.frombuffer(bytearray(desc), dtype=_u8))
        self._pass.copy_(self._pass_host, non_blocking=True)
        self._pass_copied.record(torch.cuda.current_stream(self.dev))

    def _replay(self, batch, loader=None):
        """one batch: a host or device (nodes, edges, target), or with `loader` a DeviceBlockLoader batch item"""
        if loader is not None:
            loader.gather(batch, self.nodes, self.edges, self.target, self.ctl)
        else:
            nodes, edges, target = batch
            b = _batch_rows(self, "EvalStep", nodes, edges, target)
            _load_rows(self, b, nodes, edges, target)
            _set_ctl(self.ctl, b, b)
        self.graph.replay()

    def _batches(self, loader, name):
        """(batches, the loader for _replay): a DeviceBlockLoader's batch items, or any other loader's batches"""
        if _device_loader(self, loader, name):
            return loader.batches(), loader
        return loader, None

    def _end(self):
        """the pass's one synchronising read: batch count, K0 flags OR-ed over its batches, clipped likelihood rows"""
        desc = EvalPass.from_buffer_copy(bytes(self._pass.cpu().numpy()))
        self.batches, self.flags, self.clipped = desc.idx, desc.flags, desc.clipped
        return desc

    @torch.no_grad()
    def validation_epoch(self, loader):
        """Workflow.validation_epoch (Workflow.py:813-831): the KLDivLoss(batchmean) of every batch into one of
        len(loader) zero-initialised slots, their mean as a 0-d device tensor (NaN if a target row is all zero)"""
        slots = torch.zeros(len(loader), dtype=torch.float32, device=self.dev)
        batches, dev_loader = self._batches(loader, "EvalStep.validation_epoch")
        self._begin(slots, None)
        for idx, batch in enumerate(batches):
            if idx >= slots.numel():
                raise IndexError(f"the loader yielded more than len(loader) = {slots.numel()} batches")
            self._replay(batch, dev_loader)
        self._end()
        return torch.mean(slots)

    @torch.no_grad()
    def validation_likelihood(self, loader, n_samples):
        """Analyzer.get_validation_likelihood (Analyzer.py:734-778): the NLL of the "correct" actions of the first
        batches (until idx * batch_size > min(100000, n_samples)), each batch's non-NaN rows written from
        idx * batch_size into n * (max_n_nodes + 5) zeros; returns (likelihoods, sum(likelihoods) / n_structures)"""
        n = min(100000, int(n_samples))
        lik = torch.zeros(n * (self.N + 5), dtype=torch.float32, device=self.dev)
        batches, dev_loader = self._batches(loader, "EvalStep.validation_likelihood")
        self._begin(lik[:0], lik)
        for idx, batch in enumerate(batches):
            if idx * self.B > n:
                break
            self._replay(batch, dev_loader)
        desc = self._end()
        if desc.clipped:
            raise RuntimeError(f"{desc.clipped} likelihood rows fall past the end of the {lik.numel()}-element buffer "
                               f"(n_samples = {n}, max_n_nodes + 5 = {self.N + 5}): the reference's slice assignment "
                               "raises there too")
        off = EvalPass.n_structures.offset
        n_structures = self._pass[off:off + 4].view(torch.float32).clone()
        return lik, torch.sum(lik, dim=0) / n_structures[0]

    def check(self):
        """raises if a batch of the last pass exceeded the entry capacity (or an AttentionGGNN batch had a bond of
        several types); the read already happened at the end of the pass"""
        return _check_flags(self.flags, self.d, f"a batch held more bond entries than entry_capacity={self.capacity}; "
                            "the results of that pass are invalid -- rebuild EvalStep with a larger capacity")


# ---- generation -----------------------------------------------------------------------------------------------
def entry_capacity(batch_size, max_n_nodes, n_edge_features):
    """bond entries a generation batch can ever hand to the model: a round adds at most one bond (two `edges`
    non-zeros) per slot -- an add into a non-empty graph or a connect; terminate, invalid and a first atom add none,
    terminated slots are zeroed, the never-reset dummy slot 0 starts with one self-loop and gains at most two per
    round as well -- and a batch runs at most 2N rounds: 1 + 2 * B * 2N.  Nor can there be more non-zeros than
    `edges` has elements.  The AttentionGGNN slot-0 view only removes entries."""
    B, N, Ef = int(batch_size), int(max_n_nodes), int(n_edge_features)
    return min(1 + 4 * B * N, B * N * N * Ef)


def scaffold_entry_capacity(batch_size, max_n_nodes, n_edge_features, max_scaffold_bonds):
    """`entry_capacity` of a batch that decorates scaffolds of at most m_max = `max_scaffold_bonds` bonds: a slot
    b >= 1 starts, and restarts after each molecule it finishes, from a scaffold of 2 * m_s <= 2 * m_max entries; from
    then on each round adds at most two (an add into a non-empty graph or a connect; terminate and invalid actions add
    none), and a batch runs at most 2N rounds, so it never holds more than 2 * m_max + 4N.  Slot 0 keeps its bound of
    1 + 4N.  In all, 1 + 4N + (B - 1) * (2 * m_max + 4N) = 1 + 4 * B * N + 2 * (B - 1) * m_max, and never more than
    `edges` has elements."""
    B, N, Ef, m = int(batch_size), int(max_n_nodes), int(n_edge_features), int(max_scaffold_bonds)
    return min(1 + 4 * B * N + 2 * (B - 1) * m, B * N * N * Ef)


class GraphedGenerator(GraphGenerator):
    """`GraphGenerator` with each round a replay of one captured CUDA graph:

      1. the AttentionGGNN slot-0 view (`GraphGenerator._model_inputs`) into a static copy of `edges`,
      2. K0 (`gib_graph_count` / `gib_graph_fill`) in capacity mode at `entry_capacity(B, N, Ef)` entries, which no
         batch can exceed,
      3. `gib_model_forward` on a static packed-weight arena,
      4. `gib_generation_sample_round`: sample row state[0] of `uniforms` [2N, B] and run that round; a call after the
         batch finished (or hit the 2N-round limit) changes nothing.

    Every buffer is allocated once and reset in place between batches.  After each replay the counters and the round
    state are copied into pinned host memory and an event is recorded; before launching round r + 2 the host waits
    for round r only, and stops once a copy shows the batch finished, so one inert round per batch is launched past
    the end (`inert_rounds`).  With the same uniforms the results equal, bit for bit, those of the eager
    `GraphGenerator` with the model in capacity mode at the same capacity (`model.entry_capacity =
    gen.entry_capacity`).  Exact mode can differ in the last bits of the logits: with few bond entries it runs some
    message GEMMs on the fp32 SIMT kernel, capacity mode always on the 3xTF32 tensor-core kernel.

    The weights are re-packed into the arena (one launch per batch, not per round) whenever a parameter's storage,
    in-place version or `functional.invalidate_packed_weights` epoch changed; the graph reads only the arena, so no
    recapture is needed for that.  Generation with recorded actions (`replay=`) stays with the eager generator; the
    RL rollout has its own captured form, `GraphedGeneratorRL`.

    Scaffolds (`scaffolds=`, `attachment=`, `set_scaffolds`, see `generation.ScaffoldTable`): the table is a static
    buffer the captured round reads; each batch starts with `gib_generation_scaffold_init`, and with attachment points
    the round masks the logits (`gib_generation_mask_logits`) between the forward and the sampler.  The entry
    capacity is then `scaffold_entry_capacity(B, N, Ef, m_max)`.  `set_scaffolds` copies a new set into the table in
    place when it has the same number of scaffolds, at most the bonds the capacity was sized for and attachment points
    given in both or in neither; otherwise it reallocates and the next batch recaptures.

    The sampling policy (`temperature=`, `top_k=`, `top_p=`, `set_sampling`, see `generation.GraphGenerator`): built
    with one, the round samples with `gib_generation_sample_round_policy`, which reads the policy from a device struct
    on every replay, so `set_sampling` between batches only rewrites that struct.  Built without one (or with the
    default (1, 0, 1)) the round keeps today's sampler; the first `set_sampling` to another policy makes the next batch
    capture the round once more, and later ones reuse it.  The likelihoods stay the model's.

    Constraints (`constraints=`, `set_constraints`, see `generation.GraphGenerator`): the round's mask launch reads
    the constraint table from device memory on every replay, so `set_constraints` on a generator built with
    constraints rewrites that table only; on one built without them (or to None) it rebuilds the mask and the next
    batch captures the round again, once."""

    def __init__(self, model, batch_size, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None,
                 n_chirality=None, device="cuda", scaffolds=None, attachment=None, action_mask=None,
                 max_valence=None, temperature=1.0, top_k=0, top_p=1.0, constraints=None):
        super().__init__(model, batch_size, constants=constants, n_atom_types=n_atom_types,
                         n_formal_charge=n_formal_charge, n_imp_H=n_imp_H, n_chirality=n_chirality, device=device,
                         action_mask=action_mask, max_valence=max_valence, temperature=temperature, top_k=top_k,
                         top_p=top_p, constraints=constraints)
        if not hasattr(model, "dims"):
            raise TypeError("GraphedGenerator runs this package's models (graphinvent_b200.gnn.mpnn) only")
        B, N, dev = self.batch_size, self.N, self.device
        self.params = _static_dims(self, model, B, 0)
        self.entry_capacity = entry_capacity(B, N, self.Ef)
        self._att_view = getattr(model, "MODEL", None) == "AttGGNN"
        self._edges_in = torch.zeros_like(self.edges) if self._att_view else self.edges
        self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
            self.d, self._edges_in, self.entry_capacity)
        self.packed = torch.empty(lib.gib_model_packed_bytes(ctypes.byref(self.d)), dtype=_u8, device=dev)
        self.logits = torch.empty(B, self.apd, dtype=torch.float32, device=dev)
        self.action = torch.zeros(B, dtype=torch.int32, device=dev)
        self.lik = torch.zeros(B, dtype=torch.float32, device=dev)
        self.uniforms = torch.zeros(2 * N, B, dtype=torch.float32, device=dev)
        # one row per replay: counters[0..1], state[0..1], K0 flags OR-ed over the batch.  A batch launches at most
        # 2N + 1 rounds (the last one inert)
        self._host = torch.zeros(2 * N + 1, 5, dtype=torch.int32, pin_memory=True)
        self._host_np = self._host.numpy()
        self._events = [torch.cuda.Event() for _ in range(2 * N + 1)]
        self._hdr_flags = self.cws[: HDR_INTS * 4].view(torch.int32)[HDR_FLAGS:HDR_FLAGS + 1]
        self._packed_key = None
        self.graph = None
        self.inert_rounds = 0
        self._scaffold_m, self.scaffold_version = 0, 0
        self._init_policy()
        if scaffolds is not None:
            self.set_scaffolds(scaffolds, attachment)

    # ---- the sampling policy ------------------------------------------------------------------------------
    def _init_policy(self):
        """the device struct the captured round reads the policy from; without a policy the round keeps today's
        sampler"""
        self._policy = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._policy_round = False
        self.set_sampling(*self._sampling)

    def set_sampling(self, temperature=1.0, top_k=0, top_p=1.0):
        """the sampling policy of the following batches.  A round captured with a policy reads it from device memory,
        so this only rewrites that struct; the first policy other than (1, 0, 1) on a generator built without one
        makes the next batch capture its round again, once."""
        pol = F.sampling_policy(temperature, top_k, top_p)
        self._sampling = pol
        if pol != F.SAMPLING_OFF and not self._policy_round:
            self._policy_round = True
            self._invalidate_rounds()
        if self._policy_round:
            F.set_policy(self._policy, pol)

    def _invalidate_rounds(self):
        self.graph = None

    def _masks_rebuilt(self):
        self._invalidate_graphs()

    def _sample_round_fn(self, plain, scaffold):
        """(entry point, name, leading scaffold args, trailing policy args) of the round's sampler"""
        if self.scaffolds is None:
            name, sc = plain, ()
        else:
            name, sc = scaffold, (ctypes.byref(self._sc),)
        if self._policy_round:
            return getattr(lib, name + "_policy"), name + "_policy", sc, (F._ptr(self._policy),)
        return getattr(lib, name), name, sc, ()

    # ---- scaffolds --------------------------------------------------------------------------------------------
    def _set_capacity(self, capacity):
        """K0 / forward buffers for `capacity` bond entries (the captured graphs must be captured again)"""
        self.entry_capacity = capacity
        self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
            self.d, self._k0_edges(), capacity)
        self._hdr_flags = self.cws[: HDR_INTS * 4].view(torch.int32)[HDR_FLAGS:HDR_FLAGS + 1]

    def _k0_edges(self):
        return self._edges_in

    def _invalidate_graphs(self):
        self.graph = None

    def set_scaffolds(self, scaffolds, attachment=None):
        """decorate `scaffolds` = (nodes, edges) from the next batch on (None: the empty graph again).  In place when
        the new set fits the static table; otherwise the table is reallocated and the round captured again."""
        new = self._table(scaffolds, attachment)
        old = self.scaffolds
        if (new is not None and old is not None and new.S == old.S and new.m_max <= self._scaffold_m
                and (new.protect is None) == (old.protect is None)):
            old.copy_(new)
            self.scaffold_version += 1
            return
        self.scaffolds = new
        self.scaffold_version += 1
        self._invalidate_graphs()
        B, N, dev = self.batch_size, self.N, self.device
        if new is None:
            self._scaffold_m = 0
            self._set_capacity(entry_capacity(B, N, self.Ef))
            return
        self._slot_ids = torch.zeros(B, dtype=torch.int32, device=dev)
        self._started = torch.zeros(1, dtype=torch.int32, device=dev)
        self._gen_scaffolds = torch.full((self.capacity,), -1, dtype=torch.int32, device=dev)
        self._sc = self._scaffold_struct()
        self._scaffold_m = new.m_max
        self._set_capacity(scaffold_entry_capacity(B, N, self.Ef, new.m_max))

    def _allocate(self):
        super()._allocate()
        # counters [2], round state [2] and the batch's K0 flags in one word group: one copy back per round
        self._ctl = torch.zeros(5, dtype=torch.int32, device=self.device)
        self._counters, self._state, self._flags = self._ctl[0:2], self._ctl[2:4], self._ctl[4:5]

    def _reset(self):
        """initialize_graph_batch's start state (GraphGenerator._allocate), in place: the graph keeps its addresses"""
        for t in (self.nodes, self.edges, self.n_nodes, self.likelihoods, self.generated_nodes, self.generated_edges,
                  self.generated_n_nodes, self.generated_likelihoods, self.properly_terminated, self._ctl):
            t.zero_()
        self.nodes[0].fill_(1.0)                    # fill_, not __setitem__: no host scalar is copied to the device
        self.edges[0, 0, 0, 0].fill_(1.0)
        self.n_nodes[0].fill_(1)
        if self.scaffolds is not None:
            self._gen_scaffolds.fill_(-1)
            self._scaffold_init(F._stream(self.device))

    def _mask_round(self, logits, st):
        """the attachment and action masks on a captured round's logits, gated by the round state"""
        sc, ids = (self._sc, self._slot_ids) if self.masked else (None, None)
        _mask_logits(self.action_mask, logits, st, self.nodes, self.edges, self.n_nodes, sc, ids, state=self._state,
                     counters=self._counters)

    def _pack(self):
        self.model._check_dropout()
        params = list(self.model.parameters())
        key = F._weights_key(self.d.tf32, params)
        if key == self._packed_key:
            return
        self._pack_arena(self.packed, params)
        self.params = params
        self._packed_key = key

    def _pack_arena(self, packed, params):
        """`params` into the arena `packed`; they must have the shapes of the table the generator was built for"""
        if len(params) != len(self.params) or any(p.shape != q.shape for p, q in zip(params, self.params)):
            raise RuntimeError(f"the model's parameter table changed after the {type(self).__name__} was built")
        F._require_cuda(*params)
        check(lib.gib_model_pack(ctypes.byref(self.d), F._ptr_table(params), F._ptr(packed),
                                 F._stream(self.device)), "gib_model_pack")

    # ---- the captured round -------------------------------------------------------------------------------
    def _enqueue_round(self):
        st = F._stream(self.device)
        if self._att_view:                          # GraphGenerator._model_inputs, into the static copy
            self._edges_in.copy_(self.edges)
            e0 = self.edges[0]
            nz = e0 != 0
            self._edges_in[0].copy_(e0 * (nz & (nz.to(torch.int32).cumsum(-1) == 1)).to(e0.dtype))
        _k0_forward(self, self.nodes, self._edges_in, [(self.packed, self.logits)], st)
        self._flags.bitwise_or_(self._hdr_flags)
        if self.masks_logits:
            self._mask_round(self.logits, st)
        fn, name, sc, pol = self._sample_round_fn("gib_generation_sample_round", "gib_generation_sample_round_scaffold")
        check(fn(
            self.batch_size, self.N, self.F, self.Ef, self.A, self.CH, self.n_imp_H, self.n_chirality, *sc,
            F._ptr(self.logits), self.apd, F._ptr(self.uniforms), F._ptr(self._state), F._ptr(self.action),
            F._ptr(self.lik), F._ptr(self.nodes), F._ptr(self.edges), F._ptr(self.n_nodes), F._ptr(self.likelihoods),
            F._ptr(self.generated_nodes), F._ptr(self.generated_edges), F._ptr(self.generated_n_nodes),
            F._ptr(self.generated_likelihoods), F._ptr(self.properly_terminated), self.capacity,
            F._ptr(self._counters), F._ptr(self._scratch), st, *pol), name)

    def capture(self):
        self.graph, = _capture(self.device, [self._enqueue_round])

    # ---- one batch ----------------------------------------------------------------------------------------
    @torch.no_grad()
    def build_graphs(self, generator=None, uniforms=None):
        """uniforms: optional [2N, batch_size] draws, row r feeding round r (instead of torch.rand(2N, B,
        generator=generator)); returns the number of finished molecules (may exceed batch_size, as in the reference)"""
        B, N = self.batch_size, self.N
        if uniforms is not None and tuple(uniforms.shape) != (2 * N, B):
            raise ValueError(f"uniforms must have shape [2*max_n_nodes, batch_size] = [{2 * N}, {B}]")
        self._pack()
        if self.graph is None:
            self.capture()
        self._reset()
        if uniforms is not None:
            self.uniforms.copy_(uniforms)
        else:
            torch.rand(2 * N, B, generator=generator, device=self.device, out=self.uniforms)
        rows, events, cur = self._host_np, self._events, torch.cuda.current_stream(self.device)
        i = 0
        while True:
            if i >= 2:                              # round i - 2 has ended: is the batch done?
                events[i - 2].synchronize()
                if rows[i - 2, 0] >= B or rows[i - 2, 3] != 0:
                    break
            if i == len(events):
                raise RuntimeError("GraphedGenerator: the round state did not stop the batch after 2N rounds")
            self.graph.replay()
            self._host[i].copy_(self._ctl, non_blocking=True)
            events[i].record(cur)
            i += 1
        events[i - 1].synchronize()
        n_generated, _, rounds, status, flags = (int(v) for v in rows[i - 1])
        self.rounds, self.inert_rounds = rounds, i - rounds
        _check_flags(flags, self.d, f"a generation round held more than {self.entry_capacity} bond entries: the static "
                     "entry capacity is wrong, the batch is invalid")
        if status != 0:
            raise RuntimeError("generation needs more than 2*max_n_nodes rounds: the per-slot likelihood buffer "
                               "(GraphGenerator.py:173, 'the 2 is arbitrary') would overflow, as in the reference")
        self._keep_scaffold_ids()
        return n_generated

    def sample(self, generator=None, uniforms=None):
        """what GraphGenerator.sample returns, as copies: the static buffers are overwritten by the next batch"""
        self.build_graphs(generator=generator, uniforms=uniforms)
        B = self.batch_size
        final = torch.log(self.generated_likelihoods.sum(dim=1)[:B])
        flat = self.generated_likelihoods[self.generated_likelihoods != 0]
        graphs = (self.generated_nodes[:B].clone(), self.generated_edges[:B].clone(), self.generated_n_nodes[:B].clone())
        return graphs, flat, final, self.properly_terminated[:B].clone()


# ---- the RL rollout -------------------------------------------------------------------------------------------
def rl_record_bytes(batch_size, max_n_nodes, n_node_features, n_edge_features, masked=False, action_mask=False):
    """device bytes one `GraphedGeneratorRL.sample()` keeps for its backward at the 2N-round limit (a rollout of R
    rounds keeps R / 2N of the per-round part): the int8 model input of every round, the action and both models'
    probabilities per (round, slot), and the (molecule, round) -> slot map [2B, 2N] in fp32.  masked=True (scaffolds
    with attachment points): also each (round, slot)'s scaffold id and atom count, int32 each; action_mask=True
    without attachment points: the atom count alone"""
    B, N, F_, Ef = int(batch_size), int(max_n_nodes), int(n_node_features), int(n_edge_features)
    per_round = B * (N * F_ + N * N * Ef) + B * (4 + 4 + 4) + (B * 8 if masked else B * 4 if action_mask else 0)
    return 2 * N * per_round + 2 * B * 2 * N * 4


class _RolloutLikelihoods(torch.autograd.Function):
    """generated_{agent,prior}_likelihoods [2B, 2N] of one rollout as a function of both models' parameters; the
    backward recomputes every round's forward (GraphedGeneratorRL._backward)"""

    @staticmethod
    def forward(ctx, gen, rec, n_a, *params):
        ctx.gen, ctx.rec, ctx.n_a = gen, rec, n_a
        ctx.ptrs = [p.data_ptr() for p in params]
        ctx.save_for_backward(*params)
        return gen._gather(rec)

    @staticmethod
    def backward(ctx, d_a, d_b):
        params = ctx.saved_tensors          # autograd raises here if a parameter was modified in place since the rollout
        if [p.data_ptr() for p in params] != ctx.ptrs:
            raise RuntimeError("one of the variables needed for gradient computation has been modified by an inplace "
                               "operation: a parameter's storage changed between the RL rollout and its backward")
        n_a, need = ctx.n_a, ctx.needs_input_grad[3:]
        pa, pb = params[:n_a], params[n_a:]
        ga, gb = ctx.gen._backward(ctx.rec, d_a, d_b, pa if any(need[:n_a]) else None, pb if any(need[n_a:]) else None)
        return (None, None, None, *(ga if ga is not None else [None] * len(pa)),
                *(gb if gb is not None else [None] * len(pb)))


class GraphedGeneratorRL(GraphedGenerator):
    """`generation.GraphGeneratorRL` with each rollout round a replay of one captured CUDA graph, and a backward that
    recomputes each round's forward instead of keeping its activations.

    Rollout round (two rounds in flight, round state in device memory, as `GraphedGenerator`):
      1. `gib_rl_snapshot`: the live `nodes` / `edges` as int8 into a static model input (the AttentionGGNN view of
         slot 0 applied) and into row r of the rollout record,
      2. K0 in capacity mode at `entry_capacity(B, N, Ef)`, shared by both models,
      3. the agent's and the prior's forward on one workspace,
      4. `gib_rl_sample_round`: sample from the agent (row r of `uniforms`, or row r of recorded `actions`), keep the
         action and its probability under both models per (round, slot), run the round with slot tags.

    `sample()` returns what the eager class returns, as copies; the two log-likelihood vectors are autograd tensors.
    Each call owns its rollout record (`rl_record_bytes`: int8 inputs, actions, both probability tables, the owner
    map), so several rollouts can wait for one `loss.backward()` as in `Workflow.learning_step`.  The backward inverts
    the owner map (`gib_rl_scatter_grad`), then, for each model whose parameters require grad, repacks the weights and
    replays a captured backward round R times in ascending order: restore round r's input, K0, forward,
    `gib_rl_dlogits`, `gib_model_backward` into one flat gradient bucket.  The kernels are deterministic and int8
    inputs give the float inputs' logits bit for bit, so the recomputed probabilities equal the rollout's
    (`recomputed_p`).  A frozen model costs no backward at all.

    The agent and the prior must be this package's models of the generator's family with equal dims (in
    `learning_step` they are deep copies of one model); other pairs raise ValueError.  A parameter modified in place,
    or moved, between a rollout and its backward makes the backward raise, as autograd does.

    With scaffolds and attachment points both models' logits are masked before `gib_rl_sample_round_scaffold`, and
    the record also keeps each (round, slot)'s scaffold id and atom count (`gib_rl_snapshot_scaffold`), from which the
    backward round masks the recomputed logits the same way before `gib_rl_dlogits`: the recomputed probabilities
    still equal the rollout's.  A `set_scaffolds` between a rollout and its backward makes that backward raise.

    With `action_mask=` both models' logits go through the action mask (with attachment points too, in the same
    launch) and the record keeps each (round, slot)'s atom count; the backward round rebuilds the mask from the
    restored int8 state and those counts.

    The sampling policy (`temperature=`, `top_k=`, `top_p=`, `set_sampling`, as `GraphedGenerator`) applies to the
    agent's draw only (`gib_rl_sample_round_policy`); p_a / p_b stay the two models' probabilities of the drawn action,
    so the log-likelihoods, the loss and the recomputing backward are unchanged.  Recorded `actions=` are replayed as
    they are.

    With `constraints=` the constraint rule runs in the action mask's launch, in the rollout and in the backward
    round, which reads the constraint table as it is then: a `set_constraints` between a rollout and its backward
    makes that backward raise."""

    def __init__(self, model, batch_size, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None,
                 n_chirality=None, device="cuda", scaffolds=None, attachment=None, action_mask=None,
                 max_valence=None, temperature=1.0, top_k=0, top_p=1.0, constraints=None):
        GraphGenerator.__init__(self, model, batch_size, constants=constants, n_atom_types=n_atom_types,
                                n_formal_charge=n_formal_charge, n_imp_H=n_imp_H, n_chirality=n_chirality,
                                device=device, action_mask=action_mask, max_valence=max_valence,
                                temperature=temperature, top_k=top_k, top_p=top_p, constraints=constraints)
        if not hasattr(model, "dims"):
            raise TypeError("GraphedGeneratorRL runs this package's models (graphinvent_b200.gnn.mpnn) only")
        B, N, dev = self.batch_size, self.N, self.device
        if B + 1 >= 1 << 24:
            raise ValueError("batch_size must stay below 2**24 (slot ids travel as fp32)")
        # int8 model inputs: the 0/1 state, bit-exact logits; the precision holds for rollouts and backward rounds
        self.params = _static_dims(self, model, B, 1)
        self._key = F.key_of(self.d)
        self.entry_capacity = entry_capacity(B, N, self.Ef)
        self._att_view = getattr(model, "MODEL", None) == "AttGGNN"
        i8, f32, i32 = torch.int8, torch.float32, torch.int32
        self.in_nodes = torch.zeros(B, N, self.F, dtype=i8, device=dev)
        self.in_edges = torch.zeros(B, N, N, self.Ef, dtype=i8, device=dev)
        self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
            self.d, self.in_edges, self.entry_capacity)
        pbytes = lib.gib_model_packed_bytes(ctypes.byref(self.d))
        self.packed = [torch.empty(pbytes, dtype=_u8, device=dev) for _ in range(2)]   # agent, prior
        self.logits = [torch.empty(B, self.apd, dtype=f32, device=dev) for _ in range(2)]
        self.action = torch.zeros(B, dtype=i32, device=dev)
        self.lik = torch.zeros(B, dtype=f32, device=dev)             # the slot tags b + 1
        self.uniforms = torch.zeros(2 * N, B, dtype=f32, device=dev)
        self.actions = torch.full((2 * N, B), -1, dtype=i32, device=dev)
        # the static rollout record: every round's int8 input, its actions and both models' probabilities
        self.rec_nodes = torch.zeros(2 * N, B, N, self.F, dtype=i8, device=dev)
        self.rec_edges = torch.zeros(2 * N, B, N, N, self.Ef, dtype=i8, device=dev)
        self.act_rec = torch.zeros(2 * N, B, dtype=i32, device=dev)
        self.p_a = torch.zeros(2 * N, B, dtype=f32, device=dev)
        self.p_b = torch.zeros(2 * N, B, dtype=f32, device=dev)
        self._host = torch.zeros(2 * N + 1, 5, dtype=torch.int32, pin_memory=True)
        self._host_np = self._host.numpy()
        self._events = [torch.cuda.Event() for _ in range(2 * N + 1)]
        self._hdr_flags = self.cws[: HDR_INTS * 4].view(torch.int32)[HDR_FLAGS:HDR_FLAGS + 1]
        self._packed_key = None
        self.graph = None
        self._graphs = {}                               # sampling / replaying recorded actions
        self._replay = False
        self._pair = (model, model)
        self._bwd = None
        self.inert_rounds = 0
        self.backward_rounds = [0, 0]
        self._scaffold_m, self.scaffold_version = 0, 0
        self.rec_ids = None
        self.rec_n = torch.zeros(2 * N, B, dtype=torch.int32, device=dev) if self.action_mask is not None else None
        self._init_policy()
        if scaffolds is not None:
            self.set_scaffolds(scaffolds, attachment)

    def _k0_edges(self):
        return self.in_edges

    def _invalidate_graphs(self):
        self.graph, self._graphs, self._bwd = None, {}, None

    def _invalidate_rounds(self):
        self.graph, self._graphs = None, {}

    def _masks_rebuilt(self):
        self._invalidate_graphs()
        if self.action_mask is not None and getattr(self, "rec_n", None) is None:
            self.rec_n = torch.zeros(2 * self.N, self.batch_size, dtype=torch.int32, device=self.device)

    def set_scaffolds(self, scaffolds, attachment=None):
        GraphedGenerator.set_scaffolds(self, scaffolds, attachment)
        if self.masked and getattr(self, "rec_ids", None) is None:
            B, N, dev = self.batch_size, self.N, self.device
            self.rec_ids = torch.full((2 * N, B), -1, dtype=torch.int32, device=dev)
            if getattr(self, "rec_n", None) is None:
                self.rec_n = torch.zeros(2 * N, B, dtype=torch.int32, device=dev)

    def _check_pair(self, agent, prior):
        for m in (agent, prior):
            if (not hasattr(m, "dims") or type(m) is not type(self.model)
                    or F.dims_key(m, self.batch_size, 1, self.d.tf32) != self._key):
                raise ValueError("GraphedGeneratorRL needs the agent and the prior to be this package's models of the "
                                 "generator's family with equal dims (Workflow.learning_step's deep copies); use "
                                 "generation.GraphGeneratorRL for other pairs")

    def _pack(self):
        for m in self._pair:
            m._check_dropout()
        tables = [list(m.parameters()) for m in self._pair]
        key = F._weights_key(self.d.tf32, *tables)
        if key == self._packed_key:
            return
        for packed, ps in zip(self.packed, tables):
            self._pack_arena(packed, ps)
        self._packed_key = key

    # ---- the captured rollout round -----------------------------------------------------------------------
    def _enqueue_round(self):
        B, N, st = self.batch_size, self.N, F._stream(self.device)
        check(lib.gib_rl_snapshot(B, N, self.F, self.Ef, int(self._att_view), F._ptr(self.nodes), F._ptr(self.edges),
                                  F._ptr(self._state), F._ptr(self._counters), F._ptr(self.rec_nodes),
                                  F._ptr(self.rec_edges), F._ptr(self.in_nodes), F._ptr(self.in_edges), st),
              "gib_rl_snapshot")
        if self.masks_logits:
            ids = (self._slot_ids, self.rec_ids) if self.masked else (None, None)
            check(lib.gib_rl_snapshot_scaffold(B, N, F._ptr(ids[0]), F._ptr(self.n_nodes), F._ptr(self._state),
                                               F._ptr(self._counters), F._ptr(ids[1]), F._ptr(self.rec_n), st),
                  "gib_rl_snapshot_scaffold")
        _k0_forward(self, self.in_nodes, self.in_edges, list(zip(self.packed, self.logits)), st)
        self._flags.bitwise_or_(self._hdr_flags)
        if self.masks_logits:
            for logits in self.logits:
                self._mask_round(logits, st)
        fn, name, sc, pol = self._sample_round_fn("gib_rl_sample_round", "gib_rl_sample_round_scaffold")
        check(fn(
            B, N, self.F, self.Ef, self.A, self.CH, self.n_imp_H, self.n_chirality, *sc, F._ptr(self.logits[0]),
            F._ptr(self.logits[1]), self.apd, F._ptr(self.uniforms), F._ptr(self.actions if self._replay else None),
            F._ptr(self._state), F._ptr(self.act_rec), F._ptr(self.p_a), F._ptr(self.p_b), F._ptr(self.action),
            F._ptr(self.lik), F._ptr(self.nodes), F._ptr(self.edges), F._ptr(self.n_nodes), F._ptr(self.likelihoods),
            F._ptr(self.generated_nodes), F._ptr(self.generated_edges), F._ptr(self.generated_n_nodes),
            F._ptr(self.generated_likelihoods), F._ptr(self.properly_terminated), self.capacity,
            F._ptr(self._counters), F._ptr(self._scratch), st, *pol), name)

    # ---- the captured backward round ----------------------------------------------------------------------
    def _enqueue_backward_round(self, slot):
        """round bctl[0] of model `slot`: restore its input, recompute the forward, dlogits, accumulate the gradient"""
        b, B, st = self._bwd, self.batch_size, F._stream(self.device)
        check(lib.gib_rl_restore(B, self.N, self.F, self.Ef, F._ptr(self.rec_nodes), F._ptr(self.rec_edges),
                                 F._ptr(b.ctl), F._ptr(self.in_nodes), F._ptr(self.in_edges), st), "gib_rl_restore")
        _k0_forward(self, self.in_nodes, self.in_edges, [(self.packed[slot], self.logits[0])], st)
        sampled = self.logits[0]
        if self.masks_logits:
            # the rollout's masks, from the restored state and the round's recorded atom counts (and scaffold ids), on
            # a copy: the model backward reads the unmasked output
            sampled = self.logits[1]
            sampled.copy_(self.logits[0])
            sc, ids = (self._sc, self.rec_ids) if self.masked else (None, None)
            _mask_logits(self.action_mask, sampled, st, self.in_nodes, self.in_edges, self.rec_n, sc, ids, int8=True,
                         row=b.ctl)
        check(lib.gib_rl_dlogits(B, self.apd, F._ptr(sampled), F._ptr(self.act_rec), F._ptr(b.dp[slot]),
                                 F._ptr(b.ctl), F._ptr(b.dlogits), F._ptr(self.recomputed_p[slot]), st), "gib_rl_dlogits")
        check(lib.gib_model_backward(ctypes.byref(self.d), self.hdr, F._ptr(self.in_nodes), F._ptr(self.in_edges),
                                     F._ptr(self.gbuf), F._ptr(self.packed[slot]), F._ptr(self.ws),
                                     F._ptr(self.logits[0]), F._ptr(b.dlogits), F._ptr_table(b.views[slot]),
                                     F._ptr(b.scratch), st), "gib_model_backward")
        check(lib.gib_rl_next_round(F._ptr(b.ctl), st), "gib_rl_next_round")

    def _ensure_backward(self):
        """backward buffers and the two captured backward rounds, built by the first rollout that needs gradients"""
        if self._bwd is not None:
            return
        B, N, dev = self.batch_size, self.N, self.device
        total = sum(p.numel() for p in self.params)
        b = types.SimpleNamespace()
        b.scratch = torch.empty(lib.gib_model_bwd_scratch_bytes(ctypes.byref(self.d), self.hdr), dtype=_u8, device=dev)
        b.dlogits = torch.empty(B, self.apd, dtype=torch.float32, device=dev)
        b.dp = torch.zeros(2, 2 * N, B, dtype=torch.float32, device=dev)
        b.gflat = torch.zeros(2, total, dtype=torch.float32, device=dev)
        b.views = [F._bucket_views(b.gflat[slot], self.params) for slot in range(2)]
        b.ctl = torch.zeros(1, dtype=torch.int32, device=dev)
        self.recomputed_p = torch.zeros(2, 2 * N, B, dtype=torch.float32, device=dev)
        self._bwd = b
        b.graphs = _capture(dev, [lambda: self._enqueue_backward_round(0), lambda: self._enqueue_backward_round(1)])

    def _gather(self, rec):
        """both [2B, 2N] generated-likelihood tables of a rollout record"""
        out = [torch.zeros_like(rec.owner) for _ in range(2)]
        check(lib.gib_rl_gather(self.batch_size, rec.owner.shape[0], rec.owner.shape[1], F._ptr(rec.owner),
                                F._ptr(rec.p_a), F._ptr(rec.p_b), F._ptr(out[0]), F._ptr(out[1]),
                                F._stream(self.device)), "gib_rl_gather")
        return tuple(out)

    @torch.no_grad()
    def _backward(self, rec, d_a, d_b, params_a, params_b):
        """gradients of sum(d_a * agent table + d_b * prior table) w.r.t. the models given (None: frozen, skipped)"""
        B, N, R, st = self.batch_size, self.N, rec.rounds, F._stream(self.device)
        if rec.scaffold_version != self.scaffold_version:
            raise RuntimeError("set_scaffolds was called between an RL rollout and its backward: the backward would "
                               "mask the recomputed logits with other scaffolds")
        if rec.constraints_version != self.constraints_version:
            raise RuntimeError("set_constraints was called between an RL rollout and its backward: the backward would "
                               "mask the recomputed logits with other constraints")
        self._ensure_backward()
        b = self._bwd
        self.backward_rounds = [0, 0]
        self.rec_nodes[:R].copy_(rec.nodes)
        self.rec_edges[:R].copy_(rec.edges)
        self.act_rec[:R].copy_(rec.act)
        if self.masked:
            self.rec_ids[:R].copy_(rec.ids)
        if self.masks_logits:
            self.rec_n[:R].copy_(rec.n)
        grads = [d.contiguous().float() if ps is not None else None
                 for d, ps in ((d_a, params_a), (d_b, params_b))]
        check(lib.gib_rl_scatter_grad(B, 2 * B, 2 * N, F._ptr(rec.owner), F._ptr(grads[0]), F._ptr(grads[1]),
                                      F._ptr(b.dp[0]), F._ptr(b.dp[1]), st), "gib_rl_scatter_grad")
        out = []
        for slot, params in enumerate((params_a, params_b)):
            if params is None:
                out.append(None)
                continue
            self._pack_arena(self.packed[slot], params)     # the arenas may hold another rollout's models by now
            b.gflat[slot].zero_()
            b.ctl.zero_()
            for _ in range(R):
                b.graphs[slot].replay()
            self.backward_rounds[slot] = R
            # a fresh bucket: autograd may keep it as .grad
            out.append(F._bucket_views(b.gflat[slot].clone(), params))
        self._packed_key = None
        return out

    # ---- one rollout --------------------------------------------------------------------------------------
    @torch.no_grad()
    def build_graphs(self, agent_model=None, prior_model=None, generator=None, uniforms=None, actions=None):
        """uniforms: optional [2N, B] draws (instead of torch.rand); actions: optional [R, B] recorded flat APD indices
        replayed instead of sampling (both models are still evaluated).  Returns the number of finished molecules."""
        agent = agent_model if agent_model is not None else self.model
        prior = prior_model if prior_model is not None else self.model
        self._check_pair(agent, prior)
        B, N = self.batch_size, self.N
        replay = actions is not None
        if replay:
            actions = torch.as_tensor(actions)
            if actions.dim() != 2 or actions.shape[1] != B or not 1 <= actions.shape[0] <= 2 * N:
                raise ValueError(f"actions must have shape [rounds, batch_size] with 1 <= rounds <= 2*max_n_nodes = {2 * N}")
            self.actions.fill_(-1)                      # past the trace: an invalid action that ends every slot
            self.actions[:actions.shape[0]].copy_(actions)
        self._pair = (agent, prior)
        self._replay = replay
        self.graph = self._graphs.get(replay)
        n = GraphedGenerator.build_graphs(self, generator=generator, uniforms=uniforms)
        self._graphs[replay] = self.graph
        if replay and self.rounds > actions.shape[0]:
            raise RuntimeError("replay trace ended before batch_size molecules were finished")
        return n

    def sample(self, agent_model, prior_model, generator=None, uniforms=None, actions=None):
        """what GraphGeneratorRL.sample returns, as copies: (nodes, edges, n_nodes), agent_ll, prior_ll,
        properly_terminated; agent_ll / prior_ll are differentiable w.r.t. every model parameter that requires grad"""
        self.build_graphs(agent_model, prior_model, generator=generator, uniforms=uniforms, actions=actions)
        agent, prior = self._pair
        B, R = self.batch_size, self.rounds
        pa, pb = list(agent.parameters()), list(prior.parameters())
        rec = types.SimpleNamespace(owner=self.generated_likelihoods.clone(), p_a=self.p_a[:R].clone(),
                                    p_b=self.p_b[:R].clone(), rounds=R, scaffold_version=self.scaffold_version,
                                    constraints_version=self.constraints_version)
        if torch.is_grad_enabled() and any(p.requires_grad for p in pa + pb):
            self._ensure_backward()
            rec.nodes, rec.edges, rec.act = self.rec_nodes[:R].clone(), self.rec_edges[:R].clone(), self.act_rec[:R].clone()
            if self.masked:
                rec.ids = self.rec_ids[:R].clone()
            if self.masks_logits:
                rec.n = self.rec_n[:R].clone()
            lik_a, lik_b = _RolloutLikelihoods.apply(self, rec, len(pa), *pa, *pb)
        else:
            lik_a, lik_b = self._gather(rec)
        self.generated_agent_likelihoods, self.generated_prior_likelihoods = lik_a, lik_b
        agent_ll = torch.log(torch.sum(lik_a, dim=1)[:B])          # GraphGeneratorRL.py:92-97
        prior_ll = torch.log(torch.sum(lik_b, dim=1)[:B])
        graphs = (self.generated_nodes[:B].clone(), self.generated_edges[:B].clone(), self.generated_n_nodes[:B].clone())
        return graphs, agent_ll, prior_ll, self.properly_terminated[:B].clone()


# ---- the likelihood of a molecule's decoding route -------------------------------------------------------------
RouteScores = namedtuple("RouteScores", "likelihoods offsets nll final")
RouteScores.__doc__ = """What `RouteScorer.score` returns, all device tensors:
likelihoods float32 [S]: p(action | state) of every route state; molecule m's are likelihoods[offsets[m]:offsets[m+1]],
    n_edges + 2 of them, in build order (the empty graph with its first "add" action first, the full graph with the
    terminate action last), the order the generator records its rounds in
offsets int64 [M + 1]
nll float32 [M]: -sum(log p) over the molecule's states, accumulated in fp64 in build order and rounded once
final float32 [M]: log(sum p), GraphGenerator.sample's `final` convention (GraphGenerator.py:81-83), in fp64 likewise"""


_ROUTE_REASONS = (
    (ROUTE_NOT_PREFIX, "the molecule does not begin with its scaffold (it has fewer atoms, another atom in the "
                       "scaffold's rows, or another bond among the scaffold's atoms -- an extra bond between two "
                       "scaffold atoms too: its canonical route does not pass through the scaffold's state)"),
    (ROUTE_MASKED, "its conditional route takes an action the scaffold's attachment points forbid (probability 0)"),
    (ROUTE_BAD_ID, "the scaffold id lies outside [-1, S)"),
    (ROUTE_ACTION, "its route takes an action the action mask forbids (probability 0): with 'valence', an atom of the "
                   "molecule is over its limit in the valence table"))

ROUTE_MIN_BATCH = 256        # rows from which the forward GEMMs take the tensor-core kernel (csrc/gemm_simt.cu)


def route_entry_capacity(batch_size, max_n_nodes, n_edge_features):
    """bond entries a batch of route states can hand to the model: a state holds a subset of a valid molecule's bonds,
    at most N (N - 1) / 2 of them with one type each, two `edges` non-zeros per bond"""
    B, N, Ef = int(batch_size), int(max_n_nodes), int(n_edge_features)
    return max(1, min(B * N * (N - 1), B * N * N * Ef))


class _RouteLikelihoods(torch.autograd.Function):
    """RouteScores (likelihoods, offsets, nll, final) of one `score()` call as a function of the model's parameters;
    the backward recomputes every batch of route states (RouteScorer._backward)"""

    @staticmethod
    def forward(ctx, scorer, nodes, edges, rec, *params):
        ctx.set_materialize_grads(False)            # outputs the loss does not use come back as None
        out = scorer._score(nodes, edges, rec, ids=rec.ids)
        ctx.scorer, ctx.rec = scorer, rec
        ctx.ptrs = [p.data_ptr() for p in params]
        ctx.save_for_backward(out.likelihoods, *params)
        ctx.mark_non_differentiable(out.offsets)
        return tuple(out)

    @staticmethod
    def backward(ctx, g_lik, g_off, g_nll, g_final):
        lik, *params = ctx.saved_tensors    # autograd raises here if a parameter was modified in place since score()
        if [p.data_ptr() for p in params] != ctx.ptrs:
            raise RuntimeError("one of the variables needed for gradient computation has been modified by an inplace "
                               "operation: a parameter's storage changed between RouteScorer.score() and its backward")
        grads = ctx.scorer._backward(ctx.rec, lik, params, g_lik, g_nll, g_final)
        return (None, None, None, None,
                *(g if p.requires_grad else None for g, p in zip(grads, params)))


def _int8_stack(x, name, ndim):
    t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
    if not isinstance(t, torch.Tensor) or t.dtype != torch.int8 or t.dim() != ndim:
        raise ValueError(f"{name} must be an int8 numpy array or torch tensor of {ndim} dims (nodes [M, N, F], edges "
                         f"[M, N, N, Ef]), got {getattr(t, 'dtype', type(t).__name__)} "
                         f"{tuple(getattr(t, 'shape', ()))}")
    return t.contiguous()


class RouteScorer(_LogitMasks):
    """The likelihood of molecules under a model: for every state of each molecule's decoding route (the states
    `PreprocessingGraph.get_decoding_route_state` walks, MolecularGraph.py:676-732), p(action | state) =
    softmax(model(state))[action], the probability the generator gives the action that rebuilds the molecule.

        scorer = graphinvent_b200.graphed.RouteScorer(model, batch_size=1000)
        lik, offsets, nll, final = scorer.score(nodes, edges)      # int8 [M, N, F] / [M, N, N, Ef], host or device

    Per chunk of `chunk_molecules` molecules: one upload, `gib_route_plan` (the training-set construction's route
    kernels: each state's action, node count and the step at which each bond goes; one status read), then
    ceil(S / batch_size) replays of ONE captured graph -- `gib_route_fill` (the next batch_size states into the int8
    static inputs, the batch index in device memory), K0 in capacity mode at `route_entry_capacity`, the forward,
    `gib_route_probs` (the RL sampler's softmax reduction), the batch index advanced -- and `gib_route_reduce`.  The
    K0 flags are OR-ed on the device and read once per chunk.

    The graph holds max(batch_size, ROUTE_MIN_BATCH) states (`B`): below 256 rows the graph-level GEMMs would run on
    the fp32 SIMT kernel instead of the tensor-core kernel, and the results would depend on the batch size in the last
    bits.  With it, every output is bit-identical for any batch_size and chunk_molecules, from host or device input.

    The layout arguments are `GraphedGenerator`'s and are checked the same way.  Molecules the route cannot take raise
    `preprocess.groups`' ValueError, naming the first.  The model is scored as in eval mode (a dropout_p > 0 model
    like its dropout-free twin); the matmul precision (`tf32`, `autocast_dtype`) is read at construction and baked
    into the graph; the weights are repacked once per `score()` when a parameter changed.

    Training on the route likelihoods (fine-tuning on a set of molecules, or RL on molecules the agent did not just
    sample):

        out = scorer.score(nodes, edges, requires_grad=True)
        (w * out.nll).sum().backward()                          # any function of likelihoods / nll / final

    With grad enabled and a parameter requiring grad, `likelihoods`, `nll` and `final` are autograd tensors of the
    model's parameters.  Each such call keeps a record -- a private copy of the int8 nodes / edges where they came
    from, each chunk's state count and the forward's likelihoods -- and no activations, so several calls can wait for
    one backward.  The backward repacks the weights, then per chunk: the upload, `gib_route_plan` again (deterministic,
    no status read), `gib_route_grad_coef` (dL/d log p per state), and ceil(S / B) replays of ONE second captured
    graph -- `gib_route_fill`, K0, the forward, `gib_route_dlogits`, `gib_model_backward` into one flat gradient bucket,
    the batch index advanced.  The recomputed probabilities equal the forward's bit for bit (`lik` holds the last
    chunk's after a backward).  It adds the backward scratch, one [B, apd] dlogits buffer, one coefficient per state
    of a chunk and the bucket to the scorer's buffers.  A parameter modified in place, or moved, between `score()` and
    the backward makes the backward raise, as autograd does.

    Conditional likelihoods p(molecule | scaffold), the probability a scaffold generator gives to a known decoration
    (`scaffolds=(nodes, edges)`, `attachment=`, `set_scaffolds`: the generators' arguments and `generation.ScaffoldTable`):

        scorer = RouteScorer(model, 1000, scaffolds=(sc_nodes, sc_edges), attachment=points)
        out = scorer.score(nodes, edges, scaffold_ids=ids)          # ids int [M]: a scaffold, or -1 (the whole route)

    Molecule m must begin, in decoding order, with scaffold s = ids[m]: its first k_s atoms, with every bond among
    them, are exactly the scaffold (the state S_k).  The reference's canonical route removes the last atom's bonds one
    at a time, so it passes through S_k, as state 1 + m_k in build order (m_k: the scaffold's bonds); the scored
    states are the route's last n_bonds - m_k + 1, from S_k to the terminate action.  With attachment points each of
    their logits rows goes through the generator's mask (`gib_route_mask_logits`) before the softmax.  `likelihoods`,
    `offsets`, `nll` and `final` keep their meaning over these states, as the generator's likelihoods cover only the
    decoration actions.  Molecules the rule cannot score are refused, naming the first, before any state of their
    chunk is scored: one that does not begin with its scaffold (fewer atoms, another atom or another bond among the
    scaffold's atoms -- an extra bond between two scaffold atoms too: the unmasked generator can make that molecule,
    but its canonical route does not pass through S_k), and, with attachment points, one whose conditional route takes
    a forbidden action (probability 0).  A generator's output scores as it is:

        scorer.score(gen.generated_nodes[:n].to(torch.int8), gen.generated_edges[:n].to(torch.int8),
                     scaffold_ids=gen.generated_scaffolds[:n])

    which scores each molecule's canonical route from its scaffold -- not the order in which the generator happened to
    place the bonds.  Per chunk the plan (`gib_route_plan_scaffold`) checks the prefixes and the masked actions with
    its route kernels and reads the status words once; the captured graph is fill (`gib_route_fill_scaffold`), K0, the
    forward, the mask (with attachment points), `gib_route_probs`.  The backward masks a copy of the recomputed logits
    (the model backward reads the unmasked output), so masked entries get zero dlogits; a `set_scaffolds` between
    `score()` and its backward makes the backward raise.  `scaffold_ids=None` runs the unconditional path unchanged.

    `action_mask="structure"` / `"valence"` and `max_valence=` (the generators' arguments, `generation.ActionMask`):
    p(molecule) under the masked generator.  Every logits row of a route batch goes through `gib_action_mask_logits`
    before the softmax (slot 0 too: a route batch has no dummy slot; each state's atom count is its number of
    non-empty node rows), with the attachment points in the same launch; the backward masks the
    recomputed logits the same way.  Per chunk the plan is checked by `gib_route_check_actions`, and a molecule whose
    route takes a forbidden action -- with "valence", any molecule with an atom over its limit -- is refused by name
    before its chunk is scored.

    `constraints=` (`generation.Constraints`, `set_constraints`): p(molecule) under the constrained generator.  The
    constraint rule runs in the action mask's launch (`gib_action_mask_logits_constrained`, forward and backward), and
    per chunk `gib_constraints_check` judges the molecules: one over a maximum, with a ring shorter than
    min_ring_size, or under a minimum while its last state allowed another action -- a route of probability 0 -- is
    refused by name before its chunk is scored.  The maxima and the ring-size bound do not depend on the route
    (graphinvent_b200/csrc/constraints.cuh), so the check needs only the molecule.  A scaffold's own atoms, bonds and
    rings count toward the bounds.  A `set_constraints` between `score()` and its backward makes the backward raise."""

    def __init__(self, model, batch_size, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None,
                 n_chirality=None, chunk_molecules=4096, device=None, scaffolds=None, attachment=None,
                 action_mask=None, max_valence=None, constraints=None):
        from .generation import action_layout
        from ._lib import PPDims
        C, A, CH, H, X = action_layout(model, constants, n_atom_types, n_formal_charge, n_imp_H, n_chirality)
        self.layout = (A, CH, H, X)
        if not hasattr(model, "dims"):
            raise TypeError("RouteScorer runs this package's models (graphinvent_b200.gnn.mpnn) only")
        self.model, self.constants = model, C
        self.batch_size = int(batch_size)
        if self.batch_size < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        # the captured batch: from ROUTE_MIN_BATCH rows on, every GEMM of the forward whose kernel depends on its row
        # count runs on the tensor-core kernel, so each state's logits do not depend on the batch size
        self.B = B = max(self.batch_size, ROUTE_MIN_BATCH)
        self.params = _static_dims(self, model, B, 1)
        self.dev = dev = torch.device(device) if device is not None else self.params[0].device
        self.N, self.F, self.Ef = N, F_, Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
        self.apd = N * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
        self.chunk = chunk = max(1, int(chunk_molecules))
        from .generation import make_action_mask
        self._mask_args = (action_mask, max_valence, C, self.layout, N, F_, Ef, self.apd, dev)
        self.constraints_version = 0
        self.action_mask = make_action_mask(*self._mask_args, constraints)
        self.cons_flags = torch.zeros(chunk, dtype=torch.int32, device=dev)
        self.pp = PPDims(N=N, F=F_, Ef=Ef, n_atom_types=A, n_formal_charge=CH, n_imp_H=H, n_chirality=X, batch_size=B)
        pd = ctypes.byref(self.pp)
        ws_bytes, max_states = lib.gib_route_plan_ws_bytes(pd, chunk), lib.gib_route_max_states(pd, chunk)
        if ws_bytes == 0 or max_states < 0 or lib.gib_preprocess_apd_length(pd) != self.apd:
            raise ValueError(f"RouteScorer: {lib.gib_last_error().decode()}")
        i8, i32 = torch.int8, torch.int32
        self.in_nodes = torch.zeros(chunk, N, F_, dtype=i8, device=dev)
        self.in_edges = torch.zeros(chunk, N, N, Ef, dtype=i8, device=dev)
        self.plan_ws = torch.empty(ws_bytes, dtype=_u8, device=dev)
        self.offsets = torch.zeros(chunk + 1, dtype=i32, device=dev)
        # [5] the chunk's state count, [6] the captured graph's batch index (gib_route_plan zeroes it); with the
        # action mask [PP_STATUS_INTS:] the result of gib_route_check_actions, read back with the rest
        self.status = torch.zeros(PP_STATUS_INTS + 2, dtype=i32, device=dev)
        self.slots = torch.zeros(2 * B, dtype=i32, device=dev)
        self.ctl = torch.zeros(2, dtype=i32, device=dev)
        self.lik = torch.zeros(max_states, dtype=torch.float32, device=dev)
        self.nodes, self.edges, _ = _static_inputs(self.d, dev)
        self.capacity = route_entry_capacity(B, N, Ef)
        self.cws, self.gbuf, self.hdr_np, self.hdr, self.ws, self.workspace_bytes = _model_buffers(
            self.d, self.edges, self.capacity)
        self.packed = torch.empty(lib.gib_model_packed_bytes(ctypes.byref(self.d)), dtype=_u8, device=dev)
        self.logits = torch.empty(B, self.apd, dtype=torch.float32, device=dev)
        self._flags = torch.zeros(1, dtype=i32, device=dev)
        self._hdr_flags = self.cws[: HDR_INTS * 4].view(torch.int32)[HDR_FLAGS:HDR_FLAGS + 1]
        self._packed_key = None
        self.graph = None
        self.replays = 0
        self._bwd = None
        self.backward_replays = 0
        self.scaffolds, self.scaffold_version, self._sgraph = None, 0, None
        # the masked copy of the logits the backward reads (attachment points or the action mask)
        self.masked_logits = torch.empty(B, self.apd, dtype=torch.float32, device=dev)
        if scaffolds is not None or attachment is not None:
            self.set_scaffolds(scaffolds, attachment)

    # ---- scaffolds ----------------------------------------------------------------------------------------------
    def set_scaffolds(self, scaffolds, attachment=None):
        """score conditional routes from `scaffolds` = (nodes, edges) with optional `attachment` points from the next
        score() on (None: no table).  In place when the new set has as many scaffolds and attachment points given in
        both or in neither; otherwise the table is reallocated and the conditional graphs are captured again."""
        from .generation import scaffold_table
        new = scaffold_table(scaffolds, attachment, self.N, self.F, self.Ef, self.layout, self.dev)
        old = self.scaffolds
        self.scaffold_version += 1
        if new is not None and old is not None and new.S == old.S and (new.protect is None) == (old.protect is None):
            old.copy_(new)
            return
        self.scaffolds = new
        self._sgraph = None
        if self._bwd is not None:
            self._bwd.sgraph = None
        if new is not None and not hasattr(self, "in_ids"):
            i32 = torch.int32
            self.in_ids = torch.zeros(self.chunk, dtype=i32, device=self.dev)
            self.slot_ids = torch.full((self.B,), -1, dtype=i32, device=self.dev)
            self.slot_n = torch.full((self.B,), -1, dtype=i32, device=self.dev)

    # ---- constraints ----------------------------------------------------------------------------------------
    def _masks_rebuilt(self):
        self.graph, self._sgraph, self._bwd = None, None, None

    def _refuse_constraints(self, n, pos, stop):
        """the ValueError naming the first molecule of the chunk whose route has probability 0 under the constraints"""
        flags = self.cons_flags[:n].cpu().numpy()
        bad = np.flatnonzero(flags & (CONS_OVER_MAX | CONS_SMALL_RING | CONS_UNDER_MIN))
        if not bad.size:
            return
        f = int(flags[bad[0]])
        why = [w for bit, w in ((CONS_OVER_MAX, "it is over a maximum"),
                                (CONS_SMALL_RING, "it has a ring shorter than min_ring_size"),
                                (CONS_UNDER_MIN, "it is under a minimum while its last state allowed another action"))
               if f & bit]
        raise ValueError(f"molecule {pos + int(bad[0])} (of molecules [{pos}, {stop})): its route has probability 0 "
                         f"under the constraints: {'; '.join(why)}")

    def _scaffold_ids(self, ids, M):
        """scaffold_ids as a contiguous int32 tensor where it came from, checked against the table"""
        if self.scaffolds is None:
            raise ValueError("scaffold_ids need a scaffold table: RouteScorer(..., scaffolds=) or set_scaffolds()")
        t = torch.from_numpy(np.ascontiguousarray(ids)) if isinstance(ids, np.ndarray) else ids
        if (not isinstance(t, torch.Tensor) or t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool
                or t.dim() != 1 or t.shape[0] != M):
            raise ValueError(f"scaffold_ids must be an integer numpy array or torch tensor of shape [M] = [{M}], got "
                             f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))}")
        S = self.scaffolds.S
        bad = (t < -1) | (t >= S)
        if M and bool(bad.any()):
            m = int(bad.nonzero()[0, 0])
            raise ValueError(f"scaffold_ids[{m}] = {int(t[m])} lies outside [-1, {S}): the table holds {S} scaffolds "
                             "(-1 scores the whole route)")
        return t.to(torch.int32).contiguous()

    def _refuse_scaffold(self, status, ids, start, stop):
        """the ValueError naming the first molecule of the chunk the conditional route cannot score (GIB_ROUTE_*
        flags in status[1], the molecule in status[2])"""
        if not status[1]:
            return
        m = start + int(status[2])
        why = "; ".join(r for bit, r in _ROUTE_REASONS if status[1] & bit)
        raise ValueError(f"molecule {m} (or a later one in molecules [{start}, {stop})), scaffold {int(ids[m])}: {why}")

    def _pack(self, params=None):
        """the model's parameters (or `params`, always repacked) into the arena when they changed"""
        force = params is not None
        params = list(self.model.parameters()) if params is None else list(params)
        key = F._weights_key(self.d.tf32, params)
        if key == self._packed_key and not force:
            return
        if len(params) != len(self.params) or any(p.shape != q.shape for p, q in zip(params, self.params)):
            raise RuntimeError("the model's parameter table changed after the RouteScorer was built")
        F._require_cuda(*params)
        check(lib.gib_model_pack(ctypes.byref(self.d), F._ptr_table(params), F._ptr(self.packed), F._stream(self.dev)),
              "gib_model_pack")
        self.params = params
        self._packed_key = key

    def _fill(self, st, scaffold):
        """the next batch of the planned chunk into the static inputs (`scaffold`: of a conditional plan, with each
        slot's scaffold id and atom count)"""
        if not scaffold:
            check(lib.gib_route_fill(ctypes.byref(self.pp), F._ptr(self.in_nodes), F._ptr(self.in_edges), self.chunk,
                                     F._ptr(self.plan_ws), F._ptr(self.offsets), F._ptr(self.status),
                                     F._ptr(self.ctl), F._ptr(self.slots), F._ptr(self.nodes), F._ptr(self.edges), st),
                  "gib_route_fill")
            return
        check(lib.gib_route_fill_scaffold(ctypes.byref(self.pp), F._ptr(self.in_nodes), F._ptr(self.in_edges),
                                          self.chunk, F._ptr(self.plan_ws), F._ptr(self.offsets), F._ptr(self.status),
                                          F._ptr(self.in_ids), F._ptr(self.ctl), F._ptr(self.slots),
                                          F._ptr(self.slot_ids), F._ptr(self.slot_n), F._ptr(self.nodes),
                                          F._ptr(self.edges), st), "gib_route_fill_scaffold")

    def _mask(self, logits, st, scaffold=True):
        """the action mask (with the attachment points of a conditional batch, in the same launch) or the
        attachment-point mask alone on every slot of the batch, in place"""
        masked = scaffold and self.masked
        self._sc = self.scaffolds.struct() if masked else None
        # with the action mask the atom counts are the states' non-empty node rows: slot_n is -1 for molecules scored
        # whole
        _mask_logits(self.action_mask, logits, st, self.nodes, self.edges,
                     self.slot_n if self.action_mask is None else None, self._sc,
                     self.slot_ids if masked else None, int8=True, first_slot=0)

    def _enqueue(self, scaffold=False):
        st = F._stream(self.dev)
        self._fill(st, scaffold)
        _k0_forward(self, self.nodes, self.edges, [(self.packed, self.logits)], st)
        self._flags.bitwise_or_(self._hdr_flags)
        if self.action_mask is not None or (scaffold and self.masked):
            self._mask(self.logits, st, scaffold)
        check(lib.gib_route_probs(self.B, self.apd, F._ptr(self.logits), F._ptr(self.slots), F._ptr(self.lik), st),
              "gib_route_probs")
        check(lib.gib_rl_next_round(F._ptr(self.status[6:7]), st), "gib_rl_next_round")

    def capture(self, scaffold=False):
        """the warm-up runs on the zeroed plan (no state): it writes zero rows and no likelihood"""
        if not scaffold:
            self.graph, = _capture(self.dev, [self._enqueue])
            return
        self.status.zero_()
        self._sgraph, = _capture(self.dev, [lambda: self._enqueue(True)])

    # ---- the captured backward batch ----------------------------------------------------------------------
    def _enqueue_backward(self, scaffold=False):
        """batch status[6] of the planned chunk: fill, recompute the forward, dlogits from the coefficients (the
        recomputed p into `lik`), accumulate the gradient into the bucket, advance the batch index.  With attachment
        points the mask goes on a copy of the logits: the model backward reads the unmasked output."""
        b, st = self._bwd, F._stream(self.dev)
        self._fill(st, scaffold)
        _k0_forward(self, self.nodes, self.edges, [(self.packed, self.logits)], st)
        self._flags.bitwise_or_(self._hdr_flags)
        sampled = self.logits
        if self.action_mask is not None or (scaffold and self.masked):
            sampled = self.masked_logits
            sampled.copy_(self.logits)
            self._mask(sampled, st, scaffold)
        check(lib.gib_route_dlogits(self.B, self.apd, F._ptr(sampled), F._ptr(self.slots), F._ptr(b.coef),
                                    F._ptr(b.dlogits), F._ptr(self.lik), st), "gib_route_dlogits")
        check(lib.gib_model_backward(ctypes.byref(self.d), self.hdr, F._ptr(self.nodes), F._ptr(self.edges),
                                     F._ptr(self.gbuf), F._ptr(self.packed), F._ptr(self.ws), F._ptr(self.logits),
                                     F._ptr(b.dlogits), F._ptr_table(b.views), F._ptr(b.scratch), st),
              "gib_model_backward")
        check(lib.gib_rl_next_round(F._ptr(self.status[6:7]), st), "gib_rl_next_round")

    def _ensure_backward(self):
        """backward buffers and the captured backward batch, built by the first score() that needs gradients; the
        warm-up runs on a zeroed status (no state): zero rows, no likelihood, a bucket the backward zeroes first"""
        if self._bwd is not None:
            return
        dev = self.dev
        b = types.SimpleNamespace()
        b.scratch = torch.empty(lib.gib_model_bwd_scratch_bytes(ctypes.byref(self.d), self.hdr), dtype=_u8, device=dev)
        b.dlogits = torch.empty(self.B, self.apd, dtype=torch.float32, device=dev)
        b.coef = torch.zeros(self.lik.numel(), dtype=torch.float32, device=dev)
        b.gflat = torch.zeros(sum(p.numel() for p in self.params), dtype=torch.float32, device=dev)
        b.views = F._bucket_views(b.gflat, self.params)
        b.sgraph = None
        self._bwd = b
        self.status.zero_()
        b.graph, = _capture(dev, [self._enqueue_backward])

    def _ensure_backward_scaffold(self):
        """the captured conditional backward batch (captured again after set_scaffolds reallocates the table)"""
        self._ensure_backward()
        if self._bwd.sgraph is None:
            self.status.zero_()
            self._bwd.sgraph, = _capture(self.dev, [lambda: self._enqueue_backward(True)])

    def _backward_chunk(self, rec, c, lik, g_lik, g_nll, g_final, eager=False):
        """chunk c of a record: upload, plan, coefficients, its batches (`eager`: the same calls without the graph)"""
        pos, base, S = rec.chunks[c]
        n = min(pos + self.chunk, rec.nodes.shape[0]) - pos
        st = F._stream(self.dev)
        self.in_nodes[:n].copy_(rec.nodes[pos:pos + n])
        self.in_edges[:n].copy_(rec.edges[pos:pos + n])
        self._plan(n, rec.ids[pos:pos + n] if rec.ids is not None else None, st)
        part = lambda g, a, k: g[a:a + k] if g is not None else None
        check(lib.gib_route_grad_coef(n, F._ptr(self.offsets), F._ptr(lik[base:base + S]),
                                      F._ptr(part(g_lik, base, S)), F._ptr(part(g_nll, pos, n)),
                                      F._ptr(part(g_final, pos, n)), F._ptr(self._bwd.coef), st), "gib_route_grad_coef")
        scaffold = rec.ids is not None
        graph = self._bwd.sgraph if scaffold else self._bwd.graph
        for _ in range(-(-S // self.B)):
            if eager:
                self._enqueue_backward(scaffold)
            else:
                graph.replay()
        self.backward_replays += -(-S // self.B)

    @torch.no_grad()
    def _backward(self, rec, lik, params, g_lik, g_nll, g_final):
        """gradients of sum(g_lik * likelihoods + g_nll * nll + g_final * final) of one record w.r.t. `params` (None
        gradients count as zero), as views of a fresh bucket"""
        if rec.constraints_version != self.constraints_version:
            raise RuntimeError("set_constraints was called between RouteScorer.score() and its backward: the backward "
                               "would mask the recomputed states with other constraints")
        b = self._bwd
        if b is None:                               # M = 0: no state, no backward buffers
            return F._bucket_views(torch.zeros(sum(p.numel() for p in params), device=self.dev), params)
        if rec.ids is not None:
            if rec.scaffold_version != self.scaffold_version:
                raise RuntimeError("set_scaffolds was called between RouteScorer.score() and its backward: the "
                                   "backward would plan and mask the recomputed states with other scaffolds")
            self._ensure_backward_scaffold()
        g_lik, g_nll, g_final = (g.detach().contiguous().float() if g is not None else None
                                 for g in (g_lik, g_nll, g_final))
        self._pack(params)
        b.gflat.zero_()
        self._flags.zero_()
        self.backward_replays = 0
        for c in range(len(rec.chunks)):
            self._backward_chunk(rec, c, lik, g_lik, g_nll, g_final)
        self._packed_key = None                     # the next score() repacks the model's current parameters
        _check_flags(int(self._flags.item()), self.d, f"a batch of route states held more than {self.capacity} bond "
                     "entries: the static entry capacity is wrong, the gradients are invalid")
        return F._bucket_views(b.gflat.clone(), params)     # a fresh bucket: autograd may keep it as .grad

    def score(self, nodes, edges, scaffold_ids=None, requires_grad=False):
        """`RouteScores` of the molecules nodes [M, N, F] / edges [M, N, N, Ef]: int8 numpy arrays or torch tensors on
        the host or the device, padded graphs in decoding order (what `preprocess.stacks` makes of the reference's
        `PreprocessingGraph`s, or a generator's generated_nodes / generated_edges `.to(torch.int8)`).
        `scaffold_ids`: int [M] (numpy or torch, host or device) -- molecule m's conditional route from scaffold
        scaffold_ids[m] of the table, -1 for its whole route; None: every whole route.
        `requires_grad=True`, with grad enabled and a parameter that requires grad: likelihoods, nll and final are
        differentiable w.r.t. the model's parameters (offsets is not); otherwise plain tensors, as by default."""
        nodes, edges = _int8_stack(nodes, "nodes", 3), _int8_stack(edges, "edges", 4)
        M = nodes.shape[0]
        if tuple(nodes.shape[1:]) != (self.N, self.F) or tuple(edges.shape) != (M, self.N, self.N, self.Ef):
            raise ValueError(f"nodes {tuple(nodes.shape)} / edges {tuple(edges.shape)} do not fit the scorer's "
                             f"[M, {self.N}, {self.F}] / [M, {self.N}, {self.N}, {self.Ef}]")
        ids = self._scaffold_ids(scaffold_ids, M) if scaffold_ids is not None else None
        params = list(self.model.parameters())
        if not (requires_grad and torch.is_grad_enabled() and any(p.requires_grad for p in params)):
            with torch.no_grad():
                return self._score(nodes, edges, ids=ids)
        # the record: private copies of the molecules (and scaffold ids) where they came from, filled in with each
        # chunk's states
        rec = types.SimpleNamespace(nodes=nodes.clone(), edges=edges.clone(), chunks=[],
                                    ids=ids.clone() if ids is not None else None,
                                    scaffold_version=self.scaffold_version,
                                    constraints_version=self.constraints_version)
        return RouteScores(*_RouteLikelihoods.apply(self, rec.nodes, rec.edges, rec, *params))

    def _plan(self, n, ids, st):
        """the plan of the n molecules in in_nodes / in_edges: their whole routes, or (`ids`: the chunk's scaffold
        ids, uploaded to in_ids) their conditional routes"""
        pd = ctypes.byref(self.pp)
        if ids is None:
            check(lib.gib_route_plan(pd, F._ptr(self.in_nodes), F._ptr(self.in_edges), n, self.chunk,
                                     F._ptr(self.plan_ws), F._ptr(self.offsets), F._ptr(self.status), st),
                  "gib_route_plan")
        else:
            self.in_ids[:n].copy_(ids)
            self._sc = self.scaffolds.struct()
            check(lib.gib_route_plan_scaffold(pd, F._ptr(self.in_nodes), F._ptr(self.in_edges), n, self.chunk,
                                              ctypes.byref(self._sc), F._ptr(self.in_ids), F._ptr(self.plan_ws),
                                              F._ptr(self.offsets), F._ptr(self.status), st),
                  "gib_route_plan_scaffold")
        if self.action_mask is not None:
            m = self.action_mask
            check(lib.gib_route_check_actions(pd, F._ptr(self.in_nodes), F._ptr(self.in_edges), n, self.chunk,
                                              F._ptr(self.plan_ws), F._ptr(self.offsets), m.code,
                                              F._ptr(m.table) if m.table is not None else None,
                                              F._ptr(self.status[PP_STATUS_INTS:]), st), "gib_route_check_actions")
            if m.cons_table is not None:
                masked = ids is not None and self.masked
                m.check(self.in_nodes[:n], self.in_edges[:n], None, self.in_ids[:n] if masked else None,
                        sc=self.scaffolds.struct() if masked else None, out=self.cons_flags[:n], stream=st)

    def _score(self, nodes, edges, rec=None, ids=None):
        """the forward of score(); `rec`: the backward record whose chunk list (first molecule, first state,
        states) it fills, the backward graph captured; `ids`: the scaffold ids (conditional routes)"""
        from .preprocess import refuse_bad
        M = nodes.shape[0]
        dev, f32 = self.dev, torch.float32
        nll, final = torch.empty(M, dtype=f32, device=dev), torch.empty(M, dtype=f32, device=dev)
        pieces, offs, base = [], [], 0
        scaffold = ids is not None
        if M:
            self._pack()
            if scaffold and self._sgraph is None:
                self.capture(scaffold=True)
            elif not scaffold and self.graph is None:
                self.capture()
            if rec is not None:
                self._ensure_backward_scaffold() if scaffold else self._ensure_backward()
        graph = self._sgraph if scaffold else self.graph
        st = F._stream(self.dev)
        for pos in range(0, M, self.chunk):
            stop = min(pos + self.chunk, M)
            n = stop - pos
            self.in_nodes[:n].copy_(nodes[pos:stop])
            self.in_edges[:n].copy_(edges[pos:stop])
            self._plan(n, ids[pos:stop] if scaffold else None, st)
            status = self.status.cpu().numpy()
            refuse_bad(status, pos, stop)
            if scaffold:
                self._refuse_scaffold(status, ids, pos, stop)
            if self.action_mask is not None and status[PP_STATUS_INTS]:
                m = pos + int(status[PP_STATUS_INTS + 1])
                raise ValueError(f"molecule {m} (or a later one in molecules [{pos}, {stop})): "
                                 + dict(_ROUTE_REASONS)[ROUTE_ACTION])
            if self.action_mask is not None and self.action_mask.cons_table is not None:
                self._refuse_constraints(n, pos, stop)
            S = int(status[5])
            self._flags.zero_()
            for _ in range(-(-S // self.B)):
                graph.replay()
            self.replays += -(-S // self.B)
            check(lib.gib_route_reduce(n, F._ptr(self.offsets), F._ptr(self.lik), F._ptr(nll[pos:]),
                                       F._ptr(final[pos:]), st), "gib_route_reduce")
            pieces.append(self.lik[:S].clone())
            offs.append(self.offsets[:n].to(torch.int64) + base)
            if rec is not None:
                rec.chunks.append((pos, base, S))
            base += S
            _check_flags(int(self._flags.item()), self.d, f"a batch of route states held more than {self.capacity} "
                         "bond entries: the static entry capacity is wrong, the scores are invalid")
        offs.append(torch.full((1,), base, dtype=torch.int64, device=dev))
        lik = torch.cat(pieces) if pieces else torch.zeros(0, dtype=f32, device=dev)
        return RouteScores(lik, torch.cat(offs), nll, final)
