"""GPU: capacity mode and the CUDA-graph training step for the EMN, whose message passing runs on bond rows -- each
against the exact-size eager path of the same library.

The batches hold more than 2048 bond entries, so that exact mode and capacity mode dispatch the same GEMM kernels
(exact mode sends forward GEMMs of M < 256 and weight gradients of M < 2048 to the fp32 SIMT kernels; capacity mode
always runs the tensor-core kernel)."""
import copy

import numpy as np
import pytest
import torch

from tests.test_gpu_capacity import _setup, _step_grads

pytestmark = pytest.mark.gpu

B = 256          # 3249 bond entries


def _entries(net, nodes, edges, target):
    net.entry_capacity = None
    out, loss, grads = _step_grads(net, nodes, edges, target)
    entries = net.last_stats["entries"]
    assert entries > 2048, entries
    return entries, out, loss, grads


@pytest.mark.parametrize("in_dtype,kw", [(torch.float32, {}), (torch.int8, {}),
                                         (torch.float32, dict(msg_depth=2, att_depth=3))],
                         ids=["float32", "int8", "msg_depth!=att_depth"])
def test_emn_capacity_mode_equals_exact_mode(in_dtype, kw):
    C, net, nodes, edges, target = _setup("EMN", B=B, **kw)
    nodes, edges = nodes.to(in_dtype), edges.to(in_dtype)
    entries, out0, loss0, g0 = _entries(net, nodes, edges, target)
    net.entry_capacity = int(entries * 1.3) + 64
    out1, loss1, g1 = _step_grads(net, nodes, edges, target)
    assert net.last_stats["capacity"] == net.entry_capacity
    # same tiles, same arithmetic on every live bond row: the logits agree to the last bit.  With msg_depth != att_depth
    # exact mode runs each sibling layer by layer (one tensor-core launch per layer) and capacity mode runs each as one
    # dependent-chain launch; both are the same tensor-core kernel with the same k-order per output tile.
    assert torch.equal(out0, out1)
    assert abs(loss0 - loss1) <= 1e-7
    # Weight gradients only differ by the split points of the fixed-order reductions (planned from the capacity
    # instead of the entry count, see test_emn_capacity_of_exactly_the_entries_is_bit_identical).  emb_msg_nn and
    # att_msg_nn run T + 1 times (every pass and the pass-independent branch), so their weight gradients add up T + 1
    # re-split grouped reductions: on this batch they differ by up to 1.43 x the single-reduction bound (an empirical
    # margin for this seed), hence twice that bound for them.
    names = [n for n, _ in net.named_parameters()]
    for n, a, b in zip(names, g0, g1):
        rel = 4e-6 if n.startswith(("emb_msg_nn.", "att_msg_nn.")) else 2e-6
        assert (a - b).abs().max().item() <= rel * max(1e-3, a.abs().max().item()), n


@pytest.mark.parametrize("in_dtype", [torch.float32, torch.int8])
def test_emn_capacity_of_exactly_the_entries_is_bit_identical(in_dtype):
    """with the capacity equal to the entry count, the weight-gradient reductions are planned from the same row counts
    as in exact mode: the whole step agrees to the last bit (siblings of equal depth)"""
    C, net, nodes, edges, target = _setup("EMN", B=B)
    nodes, edges = nodes.to(in_dtype), edges.to(in_dtype)
    entries, out0, loss0, g0 = _entries(net, nodes, edges, target)
    net.entry_capacity = entries
    out1, loss1, g1 = _step_grads(net, nodes, edges, target)
    assert torch.equal(out0, out1) and loss0 == loss1
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)


def _train_step(net, nodes, capacity, in_dtype=torch.float32):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    opt = FlatAdam(net.parameters(), lr=1e-4)
    return TrainStep(net, opt, batch_size=nodes.shape[0], entry_capacity=capacity, input_dtype=in_dtype, warmup=False)


def _run_eagerly(step):
    """forward + loss + backward of the step's launch sequence, without the optimizer"""
    step._enqueue_all()
    torch.cuda.synchronize()
    return step.out.clone(), step.loss.clone(), step.gflat.clone()


def test_emn_pad_rows_are_inert():
    """bond rows past the live count hold anything (here NaN) and no live result depends on them"""
    C, net, nodes, edges, target = _setup("EMN", B=B)
    entries = _entries(net, nodes, edges, target)[0]
    step = _train_step(net, nodes, 2 * entries + 128)
    step.load(nodes, edges, target)
    runs = []
    for fill in (0, 0xFF):
        step.ws.fill_(fill)
        step.scratch.fill_(fill)
        runs.append(_run_eagerly(step))
    assert int(step.cws[:64].view(torch.int32).cpu()[2]) == entries     # live count of the EMN's one group
    (o0, l0, g0), (o1, l1, g1) = runs
    assert torch.isfinite(o0).all() and torch.isfinite(g0).all()
    assert torch.equal(o0, o1) and torch.equal(l0, l1) and torch.equal(g0, g1)


def test_emn_capacity_mode_without_any_bond():
    C, net, nodes, edges, target = _setup("EMN", B=B)
    edges = torch.zeros_like(edges)
    out0, loss0, g0 = _step_grads(net, nodes, edges, target)
    assert net.last_stats["entries"] == 0
    net.entry_capacity = 256
    out1, loss1, g1 = _step_grads(net, nodes, edges, target)
    assert torch.isfinite(out1).all() and np.isfinite(loss1)
    assert torch.equal(out0, out1) and loss0 == loss1
    for a, b in zip(g0, g1):
        assert torch.isfinite(b).all() and torch.equal(a, b)


def test_emn_capacity_overflow_is_flagged_not_fatal():
    from graphinvent_b200 import functional as Fn
    C, net, nodes, edges, target = _setup("EMN", B=B)
    entries = _entries(net, nodes, edges, target)[0]
    net.entry_capacity = entries // 3
    graph = Fn.build_graph(net, edges)
    assert graph.overflowed()
    with torch.no_grad():
        out = net(nodes, edges, graph=graph)          # runs (truncated), must not fault
    torch.cuda.synchronize()
    assert out.shape[0] == nodes.shape[0]
    net.entry_capacity = None
    step = _train_step(net, nodes, entries // 3)       # forward + backward of a truncated batch
    step(nodes, edges, target)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="entry_capacity"):
        step.check()


@pytest.mark.parametrize("in_dtype", [torch.float32, torch.int8])
def test_emn_graphed_train_step_matches_eager_steps(in_dtype):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    C, net, nodes, edges, target = _setup("EMN", B=B)
    net2 = copy.deepcopy(net)
    opt = FlatAdam(net.parameters(), lr=1e-4)
    opt2 = FlatAdam(net2.parameters(), lr=1e-4)
    losses = []
    for _ in range(4):                                 # eager reference: the module API in exact mode
        out = net(nodes, edges)
        loss = Fn.kl_loss(out, target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    entries = net.last_stats["entries"]
    assert entries > 2048, entries
    step = TrainStep(net2, opt2, batch_size=B, entry_capacity=int(entries * 1.2) + 32, input_dtype=in_dtype)
    got = []
    for _ in range(4):
        got.append(float(step(nodes.to(in_dtype).cpu().pin_memory(), edges.to(in_dtype).cpu().pin_memory(), target)))
    assert step.check() & 4 == 0
    # the captured step differs from the eager one only in the split points of the weight-gradient reductions
    assert np.allclose(got, losses, rtol=0, atol=1e-5), (got, losses)
    for a, b in zip(net.parameters(), net2.parameters()):
        assert (a - b).abs().max().item() <= 1e-4


def test_emn_two_part_backward_equals_the_whole():
    """part 1 (readout) then part 2 (message passes) on the same scratch: the data-parallel split of TrainStep"""
    C, net, nodes, edges, target = _setup("EMN", B=B)
    entries = _entries(net, nodes, edges, target)[0]
    step = _train_step(net, nodes, int(entries * 1.3) + 64)
    step.load(nodes, edges, target)
    g_whole = _run_eagerly(step)[2]
    step.gflat.zero_()
    step._backward(1)
    step._backward(2)
    torch.cuda.synchronize()
    assert torch.count_nonzero(g_whole) > 0
    assert torch.equal(step.gflat, g_whole)
