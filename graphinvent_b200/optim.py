"""
Flat-bucket Adam (SURVEY.md 8f rank 2).

Drop-in for the optimizer the reference builds at Workflow.py:191,221,245
(`torch.optim.Adam(params=model.parameters(), lr=init_lr)`) and steps at Workflow.py:795-796:

    optimizer = graphinvent_b200.optim.FlatAdam(model.parameters(), lr=init_lr)
    scheduler = torch.optim.lr_scheduler.OneCycleLR(optimizer, ...)      # unchanged (reads / writes lr and betas)

The parameters are re-pointed into ONE contiguous fp32 buffer (they stay the same `nn.Parameter` objects, so
`state_dict()`, `load_state_dict()`, `deepcopy` and the module protocol are unaffected); the moments live in two
more flat buffers.  The fused backward of this package already delivers the gradients as views of one flat
bucket, so `step()` is a single `gib_adam_step` launch over the four buffers instead of the per-tensor update
loop.  Same update rule as torch.optim.Adam (L2 weight decay, no amsgrad, bias corrections in Python floats).
There is no CPU path: CPU parameters raise.

`scaled_step(found_inf, scaler)` is `scaler.step(optimizer); scaler.update()` of a `torch.amp.GradScaler` entirely on
the device (the captured training step calls it, graphed.TrainStep(grad_scaler=)): the update is gated on a device
flag, the gradients are unscaled inside the Adam kernel and the step counts live in device memory, so no host read is
needed.  `state_dict()` reads the device counts (the only synchronisation); `load_state_dict()` writes them back.
"""
import ctypes

import torch

from . import functional as _F
from ._lib import check, lib


class FlatAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0):
        if lr < 0 or eps < 0 or weight_decay < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1):
            raise ValueError("FlatAdam: invalid hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))
        self.grad_scale = float(grad_scale)
        self._dsteps = None                    # device step counts (int64 [P]) once scaled_step() ran; else host only
        self.launches_last_step = 0
        self.grad_copies_last_step = 0
        self._flatten()

    # ---- layout ---------------------------------------------------------------------------------------------
    def _all(self):
        return [p for g in self.param_groups for p in g["params"]]

    def _flatten(self, moments=None):
        ps = self._all()
        if not ps:
            raise ValueError("FlatAdam: no parameters")
        dev = ps[0].device
        _F._require_cuda(*ps)                  # raises: there is no CPU fallback
        for p in ps:
            if p.device != dev or p.dtype != torch.float32:
                raise RuntimeError("FlatAdam: all parameters must be float32 tensors on one CUDA device")
        self._off, o = [], 0
        for p in ps:
            self._off.append(o)
            o += p.numel()                     # unpadded: the same layout as the fused backward's gradient bucket
        self._total = o
        flat = torch.zeros(o, dtype=torch.float32, device=dev)
        m, v = torch.zeros_like(flat), torch.zeros_like(flat)
        with torch.no_grad():
            for i, (p, off) in enumerate(zip(ps, self._off)):
                n = p.numel()
                flat[off:off + n].copy_(p.detach().reshape(-1))
                if moments is not None and moments[i] is not None:
                    m[off:off + n].copy_(moments[i][0].reshape(-1))
                    v[off:off + n].copy_(moments[i][1].reshape(-1))
                p.data = flat[off:off + n].view(p.shape)
        self._flat, self._m, self._v = flat, m, v
        self._gflat = None
        old = getattr(self, "_steps", None)
        self._steps = old if old is not None and len(old) == len(ps) else [0] * len(ps)
        for i, (p, off) in enumerate(zip(ps, self._off)):
            n = p.numel()
            self.state[p] = {"step": torch.tensor(float(self._steps[i])),
                             "exp_avg": m[off:off + n].view(p.shape), "exp_avg_sq": v[off:off + n].view(p.shape)}
        _F.invalidate_packed_weights()

    def _pull_steps(self):
        """the device step counts into the host list (a synchronising read); no-op when the host list is current"""
        if self._dsteps is not None:
            self._steps = [int(x) for x in self._dsteps.tolist()]

    def _push_steps(self):
        """the host step counts into device memory, from pinned memory: no synchronisation"""
        host = torch.tensor(self._steps, dtype=torch.int64).pin_memory()
        if self._dsteps is None or self._dsteps.numel() != len(self._steps):
            self._dsteps = torch.empty(len(self._steps), dtype=torch.int64, device=self._flat.device)
        self._dsteps.copy_(host, non_blocking=True)

    def device_step_counts(self):
        """the int64 [P] device tensor of the per-parameter step counts that scaled_step() reads and advances (created
        from the host counts on first use)"""
        if self._dsteps is None:
            self._push_steps()
        return self._dsteps

    def _in_place(self):
        base = self._flat.data_ptr()
        return all(p.data_ptr() == base + 4 * off for p, off in zip(self._all(), self._off))

    # ---- torch.optim.Optimizer protocol ---------------------------------------------------------------------
    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        if hasattr(self, "_flat"):            # a group added after construction: rebuild the bucket, keep the moments
            self._pull_steps()
            ps = self._all()
            known = {id(p): (self.state[p]["exp_avg"].clone(), self.state[p]["exp_avg_sq"].clone())
                     for p in ps if p in self.state and "exp_avg" in self.state[p]}
            steps = {id(p): int(self.state[p]["step"]) for p in ps if p in self.state and "step" in self.state[p]}
            self._steps = [steps.get(id(p), 0) for p in ps]
            self._flatten([known.get(id(p)) for p in ps])
            if self._dsteps is not None:
                self._push_steps()

    def state_dict(self):
        self._pull_steps()
        for i, p in enumerate(self._all()):
            self.state[p]["step"] = torch.tensor(float(self._steps[i]))
        return super().state_dict()

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)   # replaces self.state[p] by copies: move them back into the buckets
        ps = self._all()
        moments, steps = [], []
        for p in ps:
            st = self.state.get(p, {})
            moments.append((st["exp_avg"], st["exp_avg_sq"]) if "exp_avg" in st else None)
            steps.append(int(st["step"]) if "step" in st else 0)
        self._steps = steps
        self._flatten(moments)
        if self._dsteps is not None:
            self._push_steps()

    def _runs(self):
        """(i, j, lo, hi, grad address, group) of each launch: consecutive parameters [i, j) sharing group, step count
        and gradient bucket; scattered gradients are first copied into a private bucket"""
        ps = self._all()
        if not self._in_place():              # e.g. model.to(...) re-assigned .data after construction
            moments = [(self.state[p]["exp_avg"], self.state[p]["exp_avg_sq"]) for p in ps]
            self._flatten(moments)
        dev = self._flat.device
        # where does each gradient live relative to its slot in the bucket?  (equal deltas = one contiguous run)
        deltas = []
        for p, off in zip(ps, self._off):
            g = p.grad
            if g is None:
                deltas.append(None)
            elif (g.dtype != torch.float32 or g.device != dev or g.is_sparse or not g.is_contiguous()
                  or (g.data_ptr() - 4 * off - self._flat.data_ptr()) & 15):
                deltas.append("copy")         # the kernel wants the four buffers equally aligned modulo 16 bytes
            else:
                deltas.append(g.data_ptr() - 4 * off)
        n_runs = sum(1 for i, d in enumerate(deltas) if d is not None and (i == 0 or deltas[i - 1] != d))
        self.grad_copies_last_step = 0
        if n_runs > 8 or "copy" in deltas:    # scattered gradients (not produced by this package's fused backward)
            if self._gflat is None:
                self._gflat = torch.zeros_like(self._flat)
            dst, src = [], []
            for p, off, d in zip(ps, self._off, deltas):
                if d is not None:
                    dst.append(self._gflat[off:off + p.numel()].view(p.shape))
                    src.append(p.grad.to_dense() if p.grad.is_sparse else p.grad)
            torch._foreach_copy_(dst, src)
            self.grad_copies_last_step = len(dst)
            gdelta = self._gflat.data_ptr()
            deltas = [None if d is None else gdelta for d in deltas]
        # one launch per run of consecutive parameters sharing group, step count and gradient bucket
        group_of = [gi for gi, g in enumerate(self.param_groups) for _ in g["params"]]
        runs = []
        i, P = 0, len(ps)
        while i < P:
            if deltas[i] is None:             # no gradient: torch.optim.Adam skips the tensor, so do we
                i += 1
                continue
            j = i + 1
            while j < P and deltas[j] == deltas[i] and group_of[j] == group_of[i] and self._steps[j] == self._steps[i]:
                j += 1
            lo = self._off[i]
            hi = self._off[j - 1] + ps[j - 1].numel()
            runs.append((i, j, lo, hi, deltas[i] + 4 * lo, self.param_groups[group_of[i]]))
            i = j
        return runs

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._pull_steps()                    # after scaled steps: the device holds the counts
        st = ctypes.c_void_p(torch.cuda.current_stream(self._flat.device).cuda_stream)
        self.launches_last_step = 0
        for i, j, lo, hi, gptr, grp in self._runs():
            step = self._steps[i] + 1
            b1, b2 = grp["betas"]
            check(lib.gib_adam_step(ctypes.c_void_p(self._flat.data_ptr() + 4 * lo), ctypes.c_void_p(gptr),
                                    ctypes.c_void_p(self._m.data_ptr() + 4 * lo),
                                    ctypes.c_void_p(self._v.data_ptr() + 4 * lo), hi - lo, step, float(grp["lr"]),
                                    float(b1), float(b2), float(grp["eps"]), float(grp["weight_decay"]),
                                    self.grad_scale, st), "gib_adam_step")
            self.launches_last_step += 1
            for k in range(i, j):
                self._steps[k] = step
        if self._dsteps is not None:
            self._push_steps()
        _F.invalidate_packed_weights()        # the kernel wrote the weights behind autograd's version counters
        return loss

    @torch.no_grad()
    def scaled_step(self, found_inf, scaler):
        """`scaler.step(self); scaler.update()` on the device, for gradients already checked into `found_inf` (a 0-d
        float32 device tensor, non-zero when a gradient is inf or NaN): the Adam kernels write nothing when it is set
        and otherwise unscale the gradients by 1 / scale; then one launch applies torch's scale update to the scaler's
        `_scale` / `_growth_tracker` and advances the step counts of a step that was taken.  Every parameter must have
        a gradient (the captured training step's bucket).  No host synchronisation."""
        ps = self._all()
        if any(p.grad is None for p in ps):
            raise ValueError("FlatAdam.scaled_step: every parameter needs a gradient")
        scale, tracker = scaler._scale, scaler._growth_tracker
        dev = self._flat.device
        for t, dt in ((found_inf, torch.float32), (scale, torch.float32), (tracker, torch.int32)):
            if t is None or t.device != dev or t.dtype != dt or t.numel() != 1:
                raise ValueError("FlatAdam.scaled_step: found_inf, the scaler's scale and growth tracker must be "
                                 "one-element float32 / float32 / int32 tensors on the parameters' device")
        counts = self.device_step_counts()
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        self.launches_last_step = 0
        for i, j, lo, hi, gptr, grp in self._runs():
            b1, b2 = grp["betas"]
            check(lib.gib_adam_step_scaled(ctypes.c_void_p(self._flat.data_ptr() + 4 * lo), ctypes.c_void_p(gptr),
                                           ctypes.c_void_p(self._m.data_ptr() + 4 * lo),
                                           ctypes.c_void_p(self._v.data_ptr() + 4 * lo), hi - lo,
                                           ctypes.c_void_p(counts.data_ptr() + 8 * i), _F._ptr(found_inf),
                                           _F._ptr(scale), float(grp["lr"]), float(b1), float(b2), float(grp["eps"]),
                                           float(grp["weight_decay"]), self.grad_scale, st), "gib_adam_step_scaled")
            self.launches_last_step += 1
        check(lib.gib_amp_update_scale(_F._ptr(scale), _F._ptr(tracker), _F._ptr(found_inf),
                                       float(scaler._growth_factor), float(scaler._backoff_factor),
                                       int(scaler._growth_interval), _F._ptr(counts), counts.numel(), st),
              "gib_amp_update_scale")
        _F.invalidate_packed_weights()
