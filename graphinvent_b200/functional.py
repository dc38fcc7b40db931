"""
Host-side glue between the drop-in modules and the C-ABI: one `torch.autograd.Function` whose
forward/backward are `gib_model_forward` / `gib_model_backward`, plus the fused loss.

PyTorch is used for device memory (caching allocator), streams and autograd plumbing only.
No computation of the hot path happens in ATen, and there is no CPU path: CPU tensors raise.
"""
import ctypes
import math
from collections import namedtuple

import numpy as np
import torch

from ._lib import (Dims, FLAG_MULTITYPE, FLAG_OVERFLOW, HDR_E, HDR_FLAGS, HDR_INTS, HDR_P, MODEL_ID, check, lib)
from .config import dtype_of_code, matmul_code

_u8 = torch.uint8


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def make_dims(model, batch, in_dtype=0, tf32=None):
    """`in_dtype`: 0 = float32 batches (BlockDatasetLoader layout), 1 = int8 batches (the on-disk HDF5 type, read
    directly by K0 and the first-layer kernels).  `tf32`: precision of the tensor-core GEMMs of the model calls made
    with these dims (`gib_dims.tf32`), 0 = 3xTF32, 1 (or True) = single-pass TF32, 2 = bf16, 3 = fp16 operands;
    None = torch's current autocast / TF32 state (`config.matmul_code`)."""
    d = Dims()
    kw = model.dims()
    for name, _ in Dims._fields_:
        if name in ("model", "B", "big", "in_dtype", "tf32"):
            continue
        setattr(d, name, int(kw.get(name, 0)))
    d.model = MODEL_ID[kw["model"]]
    d.B = int(batch)
    d.big = float(kw.get("big", 1e6))
    d.in_dtype = int(in_dtype)
    d.tf32 = matmul_code() if tf32 is None else precision_code(tf32)
    return d


def precision_code(tf32):
    """a precision code from a code or a bool: 2 / 3 stay, any other value counts as a TF32 flag"""
    return int(tf32) if tf32 in (2, 3) and not isinstance(tf32, bool) else int(bool(tf32))


def autocast_dtype_of(d):
    """the autocast dtype whose precision dims `d` run in (None: the fp32-input modes)"""
    return dtype_of_code(d.tf32)


def dims_key(model, batch, in_dtype=0, tf32=None):
    """hashable copy of the `gib_dims` a model would be run with, its matmul precision included (two models with equal
    keys can share K0's output)"""
    return key_of(make_dims(model, batch, in_dtype, tf32))


def key_of(d):
    """the fields of a `Dims`, as a tuple"""
    return tuple(getattr(d, name) for name, _ in Dims._fields_)


def input_dtype_code(nodes, edges):
    """int8 batches stay int8 (K0 / the first-layer kernels widen them on the fly); anything else runs as float32"""
    return 1 if nodes.dtype == torch.int8 and edges.dtype == torch.int8 else 0


def as_input(t, code):
    t = t.contiguous()
    return t if (code == 1 and t.dtype == torch.int8) else t.float()


def _require_cuda(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError(
                "graphinvent_b200 runs only on CUDA tensors (sm_90a kernels); there is no CPU fallback. "
                "Move the model and the batch to the GPU.")


def _check_params(model, d, params):
    n = lib.gib_model_num_params(ctypes.byref(d))
    if n < 0:
        check(n, "gib_model_num_params")     # dims the library does not support: its message names the limit
    if n != len(params):
        raise RuntimeError(f"parameter table mismatch: library expects {n} tensors, module has {len(params)}")
    for i, p in enumerate(params):
        want = lib.gib_model_param_numel(ctypes.byref(d), i)
        if want != p.numel():
            raise RuntimeError(f"parameter {i} has {p.numel()} elements, library expects {want}")
        if p.dtype != torch.float32 or not p.is_contiguous():
            raise RuntimeError("parameters must be contiguous float32")


def _ptr_table(tensors):
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return arr


def _bucket_views(flat, shapes):
    """views of the flat gradient bucket `flat`, back to back in order, one per parameter or shape"""
    views, o = [], 0
    for s in shapes:
        s = getattr(s, "shape", s)
        n = math.prod(s)
        views.append(flat[o:o + n].view(s))
        o += n
    return views


_weights_epoch = [0]


def invalidate_packed_weights():
    """for writers that bypass autograd's version counters (the flat Adam kernel writes through raw pointers)"""
    _weights_epoch[0] += 1


def _weights_key(kind, *tables):
    """cache key of a packed arena: the invalidation epoch, the arena's kind, and the storage and in-place version of
    every parameter of the tables"""
    return (_weights_epoch[0], kind) + tuple((p.data_ptr(), p._version) for ps in tables for p in ps)


def packed_weights(model, d, params):
    """Zero-padded / transposed weight arena, rebuilt only when a parameter changed
    (keyed on data_ptr + in-place version counter, so generation re-uses it every round)."""
    # the arena of a 16-bit mode holds that mode's weight planes (gib_model_pack): it serves that mode only
    key = _weights_key(d.tf32 if d.tf32 >= 2 else 0, params)
    if model._packed is not None and model._packed_key == key:
        return model._packed
    if model._packed_key is None or len(model._packed_key) != len(key):
        _check_params(model, d, params)
    dev = params[0].device
    nbytes = lib.gib_model_packed_bytes(ctypes.byref(d))
    packed = torch.empty(nbytes, dtype=_u8, device=dev)
    check(lib.gib_model_pack(ctypes.byref(d), _ptr_table(params), _ptr(packed), _stream(dev)), "gib_model_pack")
    model._packed, model._packed_key = packed, key
    return packed


class GraphBatch:
    """Device-side bond-entry lists + CSR of one batch (output of K0) and its host header.
    It depends on the batch (B, N, Ef, the edges tensor) and on whether the model is the EMN, not on the weights:
    two models of one family can share it (`build_graph`, SURVEY.md 8f rank 4: agent + prior of the RL rollout).

    `capacity=None` (exact mode): one 64-byte device->host read sizes every buffer exactly.
    `capacity=n` (capacity mode): buffers are sized for n bond entries, the live counts stay on the
    device and the kernels read them there -- no host synchronisation; `overflowed()` / `flags()` read the device
    header when the caller chooses to (a batch with more entries is truncated and flagged, never written out of
    bounds).  `buffers=(cws, buf)` re-uses the allocations of an earlier GraphBatch of equal dims and capacity (static
    addresses: CUDA-graph capture)."""
    __slots__ = ("hdr", "hdr_np", "buf", "cws", "n_entries", "n_rows", "_flags", "key", "source", "capacity")

    def __init__(self, d, edges, capacity=None, buffers=None):
        dev = edges.device
        self.key = (d.B, d.N, d.Ef, d.model, d.in_dtype)
        self.source = (edges.data_ptr(), edges._version)
        self.capacity = capacity
        st = _stream(dev)
        cws_bytes = lib.gib_graph_count_ws_bytes(ctypes.byref(d))
        self.cws = buffers[0] if buffers is not None else torch.empty(cws_bytes, dtype=_u8, device=dev)
        check(lib.gib_graph_count(ctypes.byref(d), _ptr(edges), _ptr(self.cws), st), "gib_graph_count")
        if capacity is None:
            # the single device->host read of a forward: 16 ints (the reference syncs twice in nonzero())
            self.hdr_np = self.cws[: HDR_INTS * 4].view(torch.int32).cpu().numpy().copy()
            self._flags = int(self.hdr_np[HDR_FLAGS])
        else:
            self.hdr_np = np.zeros(HDR_INTS, dtype=np.int32)
            check(lib.gib_graph_header_capacity(ctypes.byref(d), int(capacity), _ptr(self.cws),
                                                self.hdr_np.ctypes.data_as(ctypes.c_void_p)),
                  "gib_graph_header_capacity")
            self._flags = None
        self.hdr = self.hdr_np.ctypes.data_as(ctypes.c_void_p)
        self.n_entries = int(self.hdr_np[HDR_E])
        self.n_rows = int(self.hdr_np[HDR_P])
        nbytes = max(256, lib.gib_graph_bytes(ctypes.byref(d), self.hdr))
        self.buf = buffers[1] if buffers is not None else torch.empty(nbytes, dtype=_u8, device=dev)
        if self.buf.numel() < nbytes or self.cws.numel() < cws_bytes:
            raise ValueError("GraphBatch: the supplied buffers are too small for these dims / capacity")
        check(lib.gib_graph_fill(ctypes.byref(d), _ptr(edges), _ptr(self.cws), self.hdr, _ptr(self.buf), st),
              "gib_graph_fill")

    def device_header(self):
        """synchronising read of the live 16-int header (capacity mode: counts, flags)"""
        return self.cws[: HDR_INTS * 4].view(torch.int32).cpu().numpy().copy()

    @property
    def flags(self):
        if self._flags is None:
            return int(self.device_header()[HDR_FLAGS])
        return self._flags

    def overflowed(self):
        return bool(self.flags & FLAG_OVERFLOW)

    def matches(self, d, edges):
        return (self.key == (d.B, d.N, d.Ef, d.model, d.in_dtype)
                and self.source == (edges.data_ptr(), edges._version))

    def array(self, d, which, count, dtype=torch.int32):
        """view of one internal array (tests): which = 0 ent_src .. 6 src_ent (include/gib200.h)"""
        addr = lib.gib_graph_array(ctypes.byref(d), self.hdr, _ptr(self.buf), which)
        off = addr - self.buf.data_ptr()
        return self.buf[off: off + count * 4].view(dtype)


def _workspace(d, hdr, dev):
    """the forward workspace of a model call with dims d on the graph of host header `hdr`"""
    nbytes = lib.gib_model_workspace_bytes(ctypes.byref(d), hdr)
    if nbytes == 0:
        check(-1, "gib_model_workspace_bytes")
    return torch.empty(nbytes, dtype=_u8, device=dev)


class _MPNNFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, nodes, edges, *params):
        dev = nodes.device
        B = nodes.shape[0]
        d = make_dims(model, B, input_dtype_code(nodes, edges))
        st = _stream(dev)
        graph = getattr(model, "_graph_in", None)       # a CSR shared between models (mpnn_forward(graph=...))
        if graph is None:
            graph = GraphBatch(d, edges, capacity=getattr(model, "entry_capacity", None))
        elif not graph.matches(d, edges):
            raise ValueError("the shared GraphBatch was built for another batch, model family or edges tensor")
        packed = packed_weights(model, d, params)
        ws = _workspace(d, graph.hdr, dev)
        apd = d.N * d.f_add + d.N * d.f_conn + 1
        out = torch.empty(B, apd, dtype=torch.float32, device=dev)
        check(lib.gib_model_forward(ctypes.byref(d), graph.hdr, _ptr(nodes), _ptr(edges), _ptr(graph.buf),
                                    _ptr(packed), _ptr(ws), _ptr(out), st), "gib_model_forward")
        model.last_stats = {"entries": graph.n_entries, "rows": graph.n_rows, "workspace_bytes": ws.numel(),
                            "flags": graph._flags, "capacity": graph.capacity}
        ctx.model, ctx.d, ctx.graph = model, d, graph
        ctx.save_for_backward(nodes, edges, packed, ws, out)
        ctx.shapes = [p.shape for p in params]
        return out

    @staticmethod
    def backward(ctx, dout):
        nodes, edges, packed, ws, out = ctx.saved_tensors
        d, graph, model = ctx.d, ctx.graph, ctx.model
        dev = nodes.device
        dout = dout.contiguous().float()
        flat = torch.zeros(sum(math.prod(s) for s in ctx.shapes), dtype=torch.float32, device=dev)
        views = _bucket_views(flat, ctx.shapes)        # one bucket: grads are views of it
        scratch = torch.empty(lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), graph.hdr), dtype=_u8, device=dev)
        # ctx.d carries the forward's precision, whatever torch's setting is by now
        check(lib.gib_model_backward(ctypes.byref(d), graph.hdr, _ptr(nodes), _ptr(edges), _ptr(graph.buf),
                                     _ptr(packed), _ptr(ws), _ptr(out), _ptr(dout), _ptr_table(views),
                                     _ptr(scratch), _stream(dev)), "gib_model_backward")
        if model._grad_hook is not None:
            model._grad_hook(flat)      # e.g. the single NCCL all-reduce of data-parallel training
        return (None, None, None, *views)


def build_graph(model, edges):
    """K0 once for several forward passes over the same batch (same model family): pass the result as
    `model(nodes, edges, graph=...)`.  `edges` must be the contiguous float32 tensor that is then fed to the models,
    unmodified in between."""
    _require_cuda(edges)
    if edges.dim() != 4 or edges.dtype not in (torch.float32, torch.int8) or not edges.is_contiguous():
        raise ValueError("build_graph expects a contiguous float32 (or int8) edges tensor [B,N,N,Ef]")
    return GraphBatch(make_dims(model, edges.shape[0], 1 if edges.dtype == torch.int8 else 0), edges,
                      capacity=getattr(model, "entry_capacity", None))


def mpnn_forward(model, nodes, edges, graph=None):
    _require_cuda(nodes, edges)
    params = list(model.parameters())
    _require_cuda(*params)
    if nodes.dim() != 3 or edges.dim() != 4:
        raise ValueError("expected nodes [B,N,F] and edges [B,N,N,Ef]")
    code = input_dtype_code(nodes, edges)
    nodes = as_input(nodes, code)
    edges = as_input(edges, code)
    model._graph_in = graph
    try:
        if torch.is_grad_enabled() and any(p.requires_grad for p in params):
            return _MPNNFunction.apply(model, nodes, edges, *params)
        with torch.no_grad():
            return _MPNNFunction.apply(model, nodes, edges, *[p.detach() for p in params])
    finally:
        model._graph_in = None


# ------------------------------------------------------------------------------------------
# Workflow.loss (Workflow.py:833-860): KLDivLoss(batchmean)(log_softmax(output), target/sum)
# ------------------------------------------------------------------------------------------
class _KLLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, target):
        B, apd = output.shape
        rows = torch.empty(B, dtype=torch.float32, device=output.device)
        dout = torch.empty_like(output)
        check(lib.gib_kl_loss_fwd_bwd(_ptr(output), _ptr(target), B, apd, 1.0 / B, _ptr(rows), _ptr(dout),
                                      _stream(output.device)), "gib_kl_loss_fwd_bwd")
        ctx.save_for_backward(dout)
        return rows.sum() / B

    @staticmethod
    def backward(ctx, g):
        (dout,) = ctx.saved_tensors
        return dout * g, None


def kl_loss(output, target):
    """Fused `Workflow.loss`: returns the scalar batch-mean KL divergence; its backward is the
    closed form (softmax(output) - target_hat) / B computed in the same kernel."""
    _require_cuda(output, target)
    return _KLLoss.apply(output.contiguous().float(), target.contiguous().float())


def validation_nll(output, target):
    """per-row NLL of the "correct" actions, the inner loop body of `Analyzer.get_validation_likelihood`
    (Analyzer.py:744-758): -log(sum(softmax(output) * target / sum(target))) in one kernel; NaN for all-zero target
    rows (filter with `nll[~torch.isnan(nll)]` as the reference does at :756).  No gradient (evaluation only)."""
    _require_cuda(output, target)
    B, apd = output.shape
    out = output.detach().contiguous().float()
    tgt = target.contiguous().float()
    nll = torch.empty(B, dtype=torch.float32, device=out.device)
    check(lib.gib_validation_nll(_ptr(out), _ptr(tgt), B, apd, _ptr(nll), _stream(out.device)), "gib_validation_nll")
    return nll


SamplingPolicy = namedtuple("SamplingPolicy", "temperature top_k top_p")
SamplingPolicy.__doc__ = """The sampling policy of `sample_actions` and the generators (include/gib200.h: gib_sampling_policy):
temperature >= 0 (0 = greedy), top_k >= 0 (0 = no cut), top_p in (0, 1] (1 = no cut)."""
SAMPLING_OFF = SamplingPolicy(1.0, 0, 1.0)


def sampling_policy(temperature=1.0, top_k=0, top_p=1.0):
    """the SamplingPolicy of these values as the device reads them (fp32 / int32); raises ValueError naming the
    argument that is out of range"""
    try:
        with np.errstate(over="ignore"):          # a value past the fp32 range becomes inf and is refused below
            t = float(np.float32(temperature))
            p = float(np.float32(top_p))
    except (TypeError, ValueError):
        raise ValueError(f"temperature and top_p must be numbers, got {temperature!r} and {top_p!r}") from None
    if not (math.isfinite(t) and t >= 0.0):
        raise ValueError(f"temperature must be finite and >= 0 (0 = greedy), got {temperature!r}")
    if isinstance(top_k, bool) or not isinstance(top_k, (int, np.integer)) or not 0 <= int(top_k) < 1 << 31:
        raise ValueError(f"top_k must be an integer in [0, 2**31) (0 = no top-k cut), got {top_k!r}")
    if not 0.0 < p <= 1.0:
        raise ValueError(f"top_p must lie in (0, 1] (1 = no nucleus cut), got {top_p!r}")
    return SamplingPolicy(t, int(top_k), p)


def set_policy(buf, policy):
    """`policy` (a SamplingPolicy) into the device struct `buf` (int32 [4]), in stream order"""
    check(lib.gib_sampling_policy_set(_ptr(buf), *policy, _stream(buf.device)), "gib_sampling_policy_set")


def sample_actions(output, uniforms=None, generator=None, temperature=1.0, top_k=0, top_p=1.0, return_policy=False):
    """softmax + one categorical draw per molecule from APD logits (GraphGenerator.py:121,535-542),
    inverse-CDF on uniforms in [0,1).  Returns (flat action index int32 [B], likelihood [B]).

    temperature / top_k / top_p: the sampling policy (`SamplingPolicy`, include/gib200.h), which changes only which
    action is drawn: the likelihood stays the model's softmax probability of that action.  return_policy=True also
    returns q [B], the policy's probability of the drawn action.  The default policy runs today's sampler."""
    _require_cuda(output)
    pol = sampling_policy(temperature, top_k, top_p)
    B, apd = output.shape
    if uniforms is None:
        uniforms = torch.rand(B, device=output.device, generator=generator)
    action = torch.empty(B, dtype=torch.int32, device=output.device)
    lik = torch.empty(B, dtype=torch.float32, device=output.device)
    if pol == SAMPLING_OFF and not return_policy:
        check(lib.gib_sample_actions(_ptr(output.contiguous()), B, apd, _ptr(uniforms.contiguous().float()),
                                     _ptr(action), _ptr(lik), _stream(output.device)), "gib_sample_actions")
        return action, lik
    buf = torch.empty(4, dtype=torch.int32, device=output.device)
    set_policy(buf, pol)
    q = torch.empty(B, dtype=torch.float32, device=output.device) if return_policy else None
    check(lib.gib_sample_actions_policy(_ptr(output.contiguous()), B, apd, _ptr(uniforms.contiguous().float()),
                                        _ptr(buf), _ptr(action), _ptr(lik), _ptr(q), _stream(output.device)),
          "gib_sample_actions_policy")
    return (action, lik, q) if return_policy else (action, lik)
