"""GPU: the captured training step (graphed.TrainStep) over a stream of different batches.

TrainStep captures K0 -> pack -> forward -> KL loss -> backward once, in capacity mode, and runs every later batch as a
replay of that graph.  So every extent that depends on the batch (K0's header, the per-type counts and bases, the
message-row table's counts, the EMN's live bond-row count, the GEMMs' device row counts) must come from device memory,
and every buffer the step keeps from one replay to the next (graph buffer, forward workspace, backward scratch, gradient
bucket, packed arena, Adam moments) must be rewritten or reset before it is read.  Replaying one batch cannot show a
miss: stale contents equal fresh ones.  The stream below changes the device-side extents at every step, with one batch
size and one entry capacity:

  1. a large batch near the capacity with every bond type: every static buffer holds valid indices afterwards;
  2. a small batch (the generator's corner graphs and three small molecules): the type bases move, P drops far below P_cap;
  3. bond type 0 absent (it was present in batch 2), type 1 dominant;
  4. no bond at all;
  5. exactly `capacity` entries, with type group 0 ending on a 128-row boundary (the capacity is a multiple of 128);
  6. GGNN / MNN only: hubs and complete graphs, bond value 1 and other values in one (source atom, bond type);
  7. more entries than the capacity: truncated and flagged;
  8. batch 1 again.

Against each replay k:
  a. the same step through the C-ABI on freshly allocated, guarded, 0xFF-poisoned buffers at the same capacity with the
     parameters as they were before step k (test_gpu_buffer_bounds.run_step): logits, loss rows, dlogits, loss and
     gradient bucket agree bit for bit, and the packed arena equals a fresh pack wherever a pack defines it.  The
     reference is not the module API: that allocates through the caching allocator and can get back the very blocks,
     stale contents included, that a stale read would then agree with;
  b. the device state the replay left behind against the numpy restatements: the whole count workspace
     (tests/k0_reference.py), every position of the graph buffer K0 defines (the pad rows of [P, P_cap) included), the
     GGNN / MNN message-row table (tests/msg_rows_reference.py); the overflow flag on the overflowing step only, whose
     surviving molecules keep, bit for bit, the logits of a fresh run at a capacity that fits;
  c. an eager twin in lockstep: the module API in capacity mode at the same capacity, Fn.kl_loss, FlatAdam and the same
     OneCycleLR schedule.  Logits, parameters and Adam moments are bit-identical after every step; the eager loss is
     torch's sum of the very loss rows the replay wrote, which gib_sum_scaled sums in another order, so the two losses
     are held to the float32 rounding bound of that sum (they differ by up to 2 ulps).  Mid-stream `opt.load_state_dict(opt.state_dict())` moves
     every parameter (the step re-captures), and a checkpoint taken after step 3 resumes into a fresh model, optimizer,
     scheduler and TrainStep; both stay bit-identical to the uninterrupted run;
  d. the two-graph (data-parallel) step on one GPU -- a world of 2 with an identity all-reduce -- equals the
     single-graph step bit for bit over the whole stream;
  e. two replays per model against fp64 (test_gpu_parity._fp64_anchored in capacity mode): the small batch right after
     the large one, and the repeated batch 1 with weights that Adam has moved.
"""
import copy
import ctypes

import numpy as np
import pytest
import torch

from tests.k0_reference import ceil_tile, k0_reference
from tests.test_gpu_buffer_bounds import _bits_equal, _model_case, run_step

pytestmark = pytest.mark.gpu

B = 48
LR = 1e-4
TOTAL_STEPS = 16            # OneCycleLR's length: more than one stream
RELOAD_BEFORE = 4           # opt.load_state_dict(opt.state_dict()) before this step (0-based)
CHECKPOINT_AFTER = 2        # the resumed run continues from this step's state

MODELS = ["small_GGNN", "small_MNN", "small_AttGGNN", "small_EMN", "row_A", "row_I"]
STREAMS = {m: (m, torch.float32) for m in MODELS}
STREAMS.update({"small_GGNN-int8": ("small_GGNN", torch.int8), "small_EMN-int8": ("small_EMN", torch.int8)})


# ---------------------------------------------------------------------------------------------------------------------
# the stream
# ---------------------------------------------------------------------------------------------------------------------
def _atoms(case):
    """atom types and formal charges of the model's node features"""
    if case.startswith("small_"):
        return 4, 2                 # tests/golden/make_golden.py
    from tests.test_model_dims_host import CONFIGS
    return CONFIGS[case[len("row_"):]][2:4]


def _entries(e, by_type):
    return int((e != 0).sum()) if by_type else int((e != 0).any(-1).sum())


def _set_count(e, t, want, by_type, rng):
    """add or remove type-t bonds (symmetric pairs, and one self-loop when the parity asks for it) until the group that
    holds them has `want` entries: type t with typed groups, every bonded cell with the EMN's one group"""
    N = e.shape[1]
    upper = np.triu(np.ones((N, N), bool), 1)

    def count():
        return int((e[..., t] != 0).sum()) if by_type else _entries(e, False)

    diff = want - count()
    if diff < 0:
        b, i, j = np.nonzero((e[..., t] != 0) & upper)
        k = rng.choice(b.size, (1 - diff) // 2, replace=False)
        e[b[k], i[k], j[k], t] = e[b[k], j[k], i[k], t] = 0
        diff = want - count()
    if diff > 0:
        empty = ~(e != 0).any(-1)
        b, i, j = np.nonzero(empty & upper)
        k = rng.choice(b.size, diff // 2, replace=False)
        e[b[k], i[k], j[k], t] = e[b[k], j[k], i[k], t] = 1
        if diff % 2:
            b, i = np.nonzero(empty[:, np.arange(N), np.arange(N)])
            k = rng.integers(b.size)
            e[b[k], i[k], i[k], t] = 1
    assert count() == want, (count(), want)


def _stream(case, C, int8=False, seed=0):
    """the batches (dicts of numpy nodes / edges / target, what, overflow) and the stream's entry capacity"""
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    N, F, Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
    A, CH = _atoms(case)
    by_type = C.model != "EMN"
    rng = np.random.default_rng(seed)
    upper = np.triu(np.ones((N, N), bool), 1)
    iu, ju = np.triu_indices(N, 1)

    def graphs(n, s, **kw):
        nodes, edges = S.random_graphs(n, N, A, CH, n_edge_features=Ef, seed=s, **kw)
        return nodes.astype(np.float32), edges.astype(np.float32)

    n1, e1 = graphs(B, seed + 1)                    # every molecule has all N atoms
    for t in range(1, Ef):                          # and every bond type occurs
        if not e1[..., t].any():
            b, i, j = np.argwhere((e1[..., 0] != 0) & upper)[t]
            e1[b, i, j] = e1[b, j, i] = 0
            e1[b, i, j, t] = e1[b, j, i, t] = 1
    cap = ceil_tile(_entries(e1, by_type) + 16)
    batches = [("large, every bond type", n1, e1)]

    n2, e2 = np.zeros_like(n1), np.zeros_like(e1)
    n2[:5], e2[:5] = S.corner_case_graphs(N, F, Ef)
    n2[[17, 30, B - 1]], e2[[17, 30, B - 1]] = graphs(3, seed + 2, n_atoms=min(N, 4))
    batches.append(("small: corner graphs and three small molecules", n2, e2))

    n3, e3 = graphs(B, seed + 3, min_atoms=0)
    e3[..., 1] = np.maximum(e3[..., 1], e3[..., 0])
    e3[..., 0] = 0
    batches.append(("bond type 0 absent, type 1 dominant", n3, e3))

    batches.append(("no bond", graphs(B, seed + 4)[0], np.zeros_like(e1)))

    n5, e5 = graphs(B, seed + 5)
    if by_type:
        c0 = int((e5[..., 0] != 0).sum())
        _set_count(e5, 0, max(128, c0 // 128 * 128), True, rng)
        rest = sum(int((e5[..., t] != 0).sum()) for t in range(Ef) if t != 1)
        _set_count(e5, 1, cap - rest, True, rng)
    else:
        _set_count(e5, 0, cap, False, rng)
    batches.append(("exactly the capacity, group 0 ends on a 128-row boundary", n5, e5))

    if C.model in ("GGNN", "MNN"):
        n6, e6 = graphs(B, seed + 6)
        vals = np.array([2.0, 3.0] if int8 else [0.5, 2.0, 3.0], np.float32)   # positive: no atom's values sum to 0
        e6[:4] = 0
        for b in (0, 1):                            # hubs: atom 0 bonds to all, values 1 and others in one (0, type 0)
            v = np.where(np.arange(N) % 2 == 1, 1.0, vals[np.arange(N) % vals.size])
            e6[b, 0, 1:, 0] = e6[b, 1:, 0, 0] = v[1:]
        for b in (2, 3):                            # complete graphs, a random type and value per bond
            t = rng.integers(0, Ef, iu.size)
            v = rng.choice(np.concatenate([[1.0, 1.0], vals]), iu.size)
            e6[b, iu, ju, t] = e6[b, ju, iu, t] = v
        b = B - 1
        while _entries(e6, by_type) > cap:
            e6[b] = 0
            b -= 1
        batches.append(("hubs and complete graphs, values 1 and others in one (source, type)", n6, e6))

    n7, e7 = n1.copy(), e1.copy()
    b = B - 1
    while _entries(e7, by_type) <= cap:             # complete graphs at the end: the first molecules still fit
        e7[b] = 0
        e7[b, iu, ju, 0] = e7[b, ju, iu, 0] = 1
        b -= 1
    batches.append(("overflowing: truncated and flagged", n7, e7))
    batches.append(("batch 1 again", n1, e1))

    dt = np.int8 if int8 else np.float32
    apd = apd_length(C)
    out = []
    for k, (what, n, e) in enumerate(batches):
        assert not np.isnan(e).any() and (e >= 0).all()
        tgt = S.random_targets(B, apd, seed=seed + 100 + (0 if k == len(batches) - 1 else k))
        ent = _entries(e, by_type)
        over = ent > cap
        assert over == (what.startswith("overflowing")), (what, ent, cap)
        out.append(dict(what=what, nodes=n.astype(dt), edges=e.astype(dt), target=tgt, entries=ent, overflow=over))
    hdrs = [k0_reference(x["edges"], by_type, cap).hdr for x in out]
    for k in range(1, len(out)):                    # every consecutive pair changes the device-side extents
        assert not np.array_equal(hdrs[k - 1][:11], hdrs[k][:11]), k
    return out, cap


def _device(bt):
    return (torch.from_numpy(bt["nodes"]).cuda(), torch.from_numpy(bt["edges"]).cuda(),
            torch.from_numpy(bt["target"]).cuda())


def _optimizer(net):
    from graphinvent_b200.optim import FlatAdam
    opt = FlatAdam(net.parameters(), lr=LR)
    return opt, torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=LR, total_steps=TOTAL_STEPS)


def _train_step(net, opt, cap, in_dtype, **kw):
    from graphinvent_b200.graphed import TrainStep
    return TrainStep(net, opt, batch_size=B, entry_capacity=cap, input_dtype=in_dtype, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# a. / b. a replay against a fresh run and against the numpy restatements
# ---------------------------------------------------------------------------------------------------------------------
class _Static:
    """a TrainStep buffer with the part of tests/guarded.Guarded's interface that test_gpu_message_rows._table_of reads"""

    def __init__(self, t):
        self.t = t

    def ptr(self):
        return self.t.data_ptr()

    def view(self, dtype):
        return self.t.view(dtype)


def _fresh_pack(net, code, fill):
    """gib_model_pack of the model's current parameters into a fresh buffer filled with `fill`"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import check, lib
    d = Fn.make_dims(net, B, code)
    params = [p.detach() for p in net.parameters()]
    packed = torch.full((lib.gib_model_packed_bytes(ctypes.byref(d)),), fill, dtype=torch.uint8, device="cuda")
    check(lib.gib_model_pack(ctypes.byref(d), Fn._ptr_table(params), Fn._ptr(packed),
                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "gib_model_pack")
    return packed


def _assert_equals_fresh(step, fresh, packs, what):
    g = fresh["g"]
    f32 = torch.float32
    assert _bits_equal(step.out, fresh["out"]), (what, "out")
    assert _bits_equal(step.rows, g["rows"].view(f32)), (what, "rows")
    assert _bits_equal(step.dout, g["dout"].view(f32).view(step.dout.shape)), (what, "dout")
    assert _bits_equal(step.loss.view(1), fresh["loss"].view(1)), (what, "loss")
    assert _bits_equal(step.gflat, fresh["grads"]), (what, "gflat", int((step.gflat != fresh["grads"]).sum()))
    # the captured pack read the parameters the optimizer wrote in place at the end of the previous step
    poisoned, zeroed = packs
    defined = poisoned == zeroed
    assert int(defined.sum()) >= 4 * sum(p.numel() for p in step.params), what
    bad = torch.nonzero(defined & (step.packed != poisoned)).flatten()
    assert bad.numel() == 0, (what, "packed", bad[:8].tolist())


def _assert_device_state(step, bt, net, C, cap, what):
    from tests.msg_rows_reference import TABLE_ARRAYS
    from tests.test_gpu_message_rows import _table_of
    by_type = C.model != "EMN"
    ref = k0_reference(bt["edges"], by_type, cap)
    cws = step.cws.view(torch.int32).cpu().numpy()
    assert np.array_equal(cws[:16], ref.hdr), (what, cws[:16], ref.hdr)
    assert np.array_equal(cws, ref.expected_cws), what
    # graph buffer: every position K0 defines (those where two different "unwritten" fills agree)
    want = ref.expected_buf
    defined = want == k0_reference(bt["edges"], by_type, cap, unwritten=-2).expected_buf
    buf = step.gbuf.view(torch.int32).cpu().numpy()[:want.size]
    bad = np.flatnonzero(defined & (buf != want))
    if bad.size:
        lay, first = ref.layout, int(bad[0])
        name = max((k for k in lay if lay[k] <= first), key=lambda k: lay[k])
        raise AssertionError(f"{what}: graph buffer differs first at int {first} ({name}[{first - lay[name]}]): "
                             f"{buf[first]} vs {want[first]}, {bad.size} ints differ")
    tail = slice(ref.layout["ent_src"] + ref.P, ref.layout["ent_src"] + ref.cap_P)
    assert ref.P >= ref.cap_P or (defined[tail].all() and (buf[tail] == -1).all()), what     # pad rows [P, P_cap)
    if C.model in ("GGNN", "MNN"):
        got = dict(hdr=step.hdr_np, g=dict(ws=_Static(step.ws), graph=_Static(step.gbuf), cws=_Static(step.cws)))
        table, mref = _table_of(got, net, B)
        for k in TABLE_ARRAYS:
            assert np.array_equal(table[k], mref[k]), (what, k, np.flatnonzero(table[k] != mref[k])[:8])
    return ref


def _state(step, opt):
    return dict(out=step.out.clone(), loss=step.loss.clone(), flat=opt._flat.clone(), m=opt._m.clone(),
                v=opt._v.clone())


@pytest.mark.parametrize("sid", list(STREAMS))
def test_replays_equal_fresh_runs_and_eager_steps(sid):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.gnn import mpnn
    case, in_dtype = STREAMS[sid]
    code = 1 if in_dtype == torch.int8 else 0
    C, net, *_ = _model_case(case)
    stream, cap = _stream(case, C, int8=bool(code))
    eager = copy.deepcopy(net)
    eager.entry_capacity = cap
    opt, sched = _optimizer(net)
    opt_e, sched_e = _optimizer(eager)
    step = _train_step(net, opt, cap, in_dtype)
    trail, ckpt = [], None
    for k, bt in enumerate(stream):
        what = f"{sid} step {k + 1}: {bt['what']}"
        nodes, edges, target = _device(bt)
        # references at the pre-step parameters
        fresh = run_step(net, nodes, edges, target, cap, "poison")
        packs = (fresh["g"]["packed"].t.clone(), _fresh_pack(net, code, 0))
        fit = run_step(net, nodes, edges, target, bt["entries"] + 128, "zero") if bt["overflow"] else None
        if k == RELOAD_BEFORE:
            graph = step.graph
            opt.load_state_dict(opt.state_dict())        # re-flattens: every parameter moves
        loss = step(nodes, edges, target)
        sched.step()
        if k == RELOAD_BEFORE:
            assert step.graph is not graph, "the moved parameters were not re-captured"
        out_e = eager(nodes, edges)
        loss_e = Fn.kl_loss(out_e, target)
        opt_e.zero_grad(set_to_none=True)
        loss_e.backward()
        opt_e.step()
        sched_e.step()
        torch.cuda.synchronize()
        # a.
        _assert_equals_fresh(step, fresh, packs, what)
        # b.
        ref = _assert_device_state(step, bt, net, C, cap, what)
        if bt["overflow"]:
            with pytest.raises(RuntimeError, match="entry_capacity"):
                step.check()
            keep = torch.from_numpy(ref.survivors).cuda()
            assert 0 < int(keep.sum()) < B, what
            assert _bits_equal(step.out[keep], fit["out"][keep]), what
        else:
            step.check()
        # c.
        assert _bits_equal(step.out, out_e.detach()), (what, "logits against the eager step")
        # the same loss rows, summed by torch (eager) and by gib_sum_scaled (captured) in different orders: each sum
        # within the float32 bound of its fp64 value; they differ by 2 ulps on the first batch of row I and AttGGNN
        assert _bits_equal((step.rows.sum() / B).view(1), loss_e.detach().view(1)), what
        rows = step.rows.double()
        exact = float(rows.sum()) / B
        bound = 2.0 ** -24 * ((B - 1) * float(rows.abs().sum()) / B + abs(exact))
        for side, val in (("captured", loss), ("eager", loss_e.detach())):
            assert abs(float(val) - exact) <= bound, (what, side, float(val), exact, bound)
        for name, a, b in (("parameters", opt._flat, opt_e._flat), ("exp_avg", opt._m, opt_e._m),
                           ("exp_avg_sq", opt._v, opt_e._v)):
            assert _bits_equal(a, b), (what, name, int((a != b).sum()))
        trail.append(_state(step, opt))
        if k == CHECKPOINT_AFTER:
            ckpt = ({n: v.detach().cpu().clone() for n, v in net.state_dict().items()},
                    copy.deepcopy(opt.state_dict()), copy.deepcopy(sched.state_dict()))
    del step
    # resume the checkpoint into a fresh model, optimizer, scheduler and TrainStep
    sd, osd, ssd = ckpt
    net_r = mpnn.create(C)
    net_r.load_state_dict(sd)
    net_r = net_r.cuda()
    opt_r, sched_r = _optimizer(net_r)
    opt_r.load_state_dict(osd)
    sched_r.load_state_dict(ssd)
    step_r = _train_step(net_r, opt_r, cap, in_dtype)
    for k in range(CHECKPOINT_AFTER + 1, len(stream)):
        step_r(*_device(stream[k]))
        sched_r.step()
        torch.cuda.synchronize()
        got = _state(step_r, opt_r)
        for name in got:
            assert _bits_equal(got[name], trail[k][name]), (f"{sid} resumed at step {k + 1}", name)


# ---------------------------------------------------------------------------------------------------------------------
# d. the two-graph (data-parallel) step on one GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sid", list(STREAMS))
def test_two_graph_step_equals_the_single_graph_step(sid, monkeypatch):
    case, in_dtype = STREAMS[sid]
    C, net, *_ = _model_case(case)
    stream, cap = _stream(case, C, int8=in_dtype == torch.int8)
    net2 = copy.deepcopy(net)
    opt, sched = _optimizer(net)
    opt2, sched2 = _optimizer(net2)
    one = _train_step(net, opt, cap, in_dtype, group=False)
    dist = torch.distributed
    # a world of 2 whose all-reduce is the identity: the step's arithmetic is one rank's, split into two graphs
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "all_reduce", lambda tensor, *a, **kw: None)
    two = _train_step(net2, opt2, cap, in_dtype)
    assert one.world == 1 and one.graph2 is None
    assert two.world == 2 and two.graph2 is not None and 0 < two.tail_off < two.gflat.numel()
    for k, bt in enumerate(stream):
        batch = _device(bt)
        one(*batch)
        sched.step()
        two(*batch)
        sched2.step()
        torch.cuda.synchronize()
        a, b = _state(one, opt), _state(two, opt2)
        for name in a:
            assert _bits_equal(a[name], b[name]), (f"{sid} step {k + 1}: {bt['what']}", name)
        assert _bits_equal(one.gflat, two.gflat), (f"{sid} step {k + 1}: {bt['what']}", "gflat")


# ---------------------------------------------------------------------------------------------------------------------
# e. two replays per model against fp64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", MODELS)
def test_replays_are_fp64_anchored(case, monkeypatch):
    from graphinvent_b200.gnn import mpnn
    from tests.test_gpu_parity import _fp64_anchored
    C, net, *_ = _model_case(case)
    stream, cap = _stream(case, C)
    opt, sched = _optimizer(net)
    step = _train_step(net, opt, cap, torch.float32)
    anchors = {1, len(stream) - 1}         # the small batch after the large one; batch 1 again, with moved weights
    runs = []
    for k, bt in enumerate(stream):
        if k in anchors:
            runs.append((k, {n: v.detach().cpu().clone() for n, v in net.state_dict().items()}, bt))
        step(*_device(bt))
        sched.step()
    torch.cuda.synchronize()
    step.check()
    create = mpnn.create

    def create_in_capacity_mode(c):
        m = create(c)
        m.entry_capacity = cap
        return m

    monkeypatch.setattr(mpnn, "create", create_in_capacity_mode)
    for k, sd, bt in runs:
        nodes, edges, target = (torch.from_numpy(bt[x]).float() for x in ("nodes", "edges", "target"))
        _fp64_anchored(C, sd, nodes, edges, target, f"{case} replay {k + 1}: {bt['what']}, capacity {cap}")
