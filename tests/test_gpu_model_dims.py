"""GPU: the four models across the reference's hyper-parameter range (tests/test_model_dims_host.py: one row per branch
of csrc/model.cu the default dims never reach) -- fp64-anchored forward + backward, capacity mode against exact mode,
the two-part backward against the whole, the CUDA-graph training step against eager steps, int8 against float batches,
and the refusals of unsupported dims through the module API."""
import copy
import functools

import numpy as np
import pytest
import torch

from tests.test_gpu_capacity import _step_grads
from tests.test_gpu_emn_capacity import _run_eagerly, _train_step
from tests.test_gpu_parity import _fp64_anchored
from tests.test_model_dims_host import CONFIGS, REFUSALS, constants

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _batch(cid):
    """about 50 seeded molecules of the row's dims plus the generator's corner graphs; every bond type occurs"""
    from graphinvent_b200 import synthetic as S
    from graphinvent_b200.config import apd_length
    C = constants(cid)
    _, _, n_atoms, n_charges, n_mol, _ = CONFIGS[cid]
    N, F, Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
    n, e = S.random_graphs(n_mol, N, n_atoms, n_charges, n_edge_features=Ef, seed=sum(map(ord, cid)), min_atoms=0)
    n2, e2 = S.corner_case_graphs(N, F, Ef)
    nodes = torch.from_numpy(np.concatenate([n2, n])).float()
    edges = torch.from_numpy(np.concatenate([e2, e])).float()
    target = torch.from_numpy(S.random_targets(nodes.shape[0], apd_length(C), seed=5))
    assert (edges.sum((0, 1, 2)) > 0).all(), f"row {cid}: a bond type never occurs"
    return C, nodes, edges, target


def _net(C, seed=0):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    net = mpnn.create(C)
    net.load_state_dict(O.init_state_dict(C, seed=seed))
    return net.cuda()


def _setup(cid):
    C, nodes, edges, target = _batch(cid)
    return C, _net(C), nodes.cuda(), edges.cuda(), target.cuda()


def _assert_every_type_group_is_live(C, net, edges):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import HDR_TYPE_COUNT
    if C.model == "EMN":
        return          # one untyped group of bond rows (the per-type check is _batch's)
    hdr = Fn.build_graph(net, edges).hdr_np
    assert all(hdr[HDR_TYPE_COUNT + t] > 0 for t in range(C.n_edge_features)), hdr


@pytest.mark.parametrize("cid,tensor_cores", [(c, 1) for c in CONFIGS] + [(c, 0) for c in ("F", "I", "M")])
def test_fp64_anchored(cid, tensor_cores):
    from oracle import mpnn_oracle as O
    C, nodes, edges, target = _batch(cid)
    _assert_every_type_group_is_live(C, _net(C), edges.cuda())
    _fp64_anchored(C, O.init_state_dict(C, seed=0), nodes, edges, target, f"row {cid}: {CONFIGS[cid][-1]}",
                   tensor_cores)


# Rows whose capacity-mode step runs the same kernels with the same reduction split as exact mode, up to the plan rows of
# the grouped weight gradients.  The others are held to fp64 instead (test_capacity_mode_is_fp64_anchored):
#   A, G  both modes run the message MLPs on the message-row table's device-side counts (the profiling records of
#         tests/test_gpu_message_rows_fp64.py show exact mode taking that branch for these rows) and their backward in
#         sub-groups of <= 16 layers, but the grouped weight gradients are planned with each mode's own entry-row count
#         (exact P, or the capacity's), so their split points differ;
#   I     exact mode sends GEMMs narrower than 48 columns to the fp32 SIMT kernel, capacity mode runs every bond-row
#         GEMM on the tensor-core kernel;
#   J     the re-split 640-wide grouped weight gradients differ by 2.03e-6 x max|g| (one element of msg_nns.2.seq.0),
#         just past the default-dims bound below.
SAME_KERNELS = [c for c in CONFIGS if c not in ("A", "G", "I", "J")]


@pytest.mark.parametrize("cid", SAME_KERNELS)
def test_capacity_mode_equals_exact_mode(cid):
    C, net, nodes, edges, target = _setup(cid)
    out0, loss0, g0 = _step_grads(net, nodes, edges, target)
    net.entry_capacity = int(net.last_stats["entries"] * 1.3) + 64
    out1, loss1, g1 = _step_grads(net, nodes, edges, target)
    assert net.last_stats["capacity"] == net.entry_capacity
    # same tiles, same arithmetic: the logits agree to the last bit; weight gradients only differ by the split points
    # of the fixed-order reductions
    assert torch.equal(out0, out1)
    assert abs(loss0 - loss1) <= 1e-7
    for (name, _), a, b in zip(net.named_parameters(), g0, g1):
        assert (a - b).abs().max().item() <= 2e-6 * max(1e-3, a.abs().max().item()), name


@pytest.mark.parametrize("cid", ["A", "D", "G", "I", "J"])
def test_capacity_mode_is_fp64_anchored(cid):
    """capacity mode against fp64 with _fp64_anchored's bounds: A and G run the message-MLP backward in sub-groups
    (their split points reorder the grouped dW sums), D's msg / att siblings have unequal depth, I runs the tensor-core
    kernel where exact mode runs the SIMT kernel, J's grouped weight gradients are re-split (SAME_KERNELS)"""
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C, nodes, edges, target = _batch(cid)
    entries = int((edges > 0).sum())
    create = mpnn.create

    def create_in_capacity_mode(c):
        net = create(c)
        net.entry_capacity = entries + 64
        return net

    mpnn.create = create_in_capacity_mode
    try:
        _fp64_anchored(C, O.init_state_dict(C, seed=0), nodes, edges, target, f"row {cid}, capacity mode")
    finally:
        mpnn.create = create


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_two_part_backward_equals_the_whole(cid):
    """part 1 (readout) then part 2 (message passes) on the same scratch: the data-parallel split of TrainStep"""
    C, net, nodes, edges, target = _setup(cid)
    _step_grads(net, nodes, edges, target)
    step = _train_step(net, nodes, int(net.last_stats["entries"] * 1.3) + 64)
    step.load(nodes, edges, target)
    g_whole = _run_eagerly(step)[2]
    step.gflat.zero_()
    step._backward(1)
    step._backward(2)
    torch.cuda.synchronize()
    assert torch.count_nonzero(g_whole) > 0
    assert torch.equal(step.gflat, g_whole)


@pytest.mark.parametrize("cid", ["A", "E", "G"])
def test_graphed_train_step_matches_eager_steps(cid):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    C, net, nodes, edges, target = _setup(cid)
    net2 = copy.deepcopy(net)
    opt = FlatAdam(net.parameters(), lr=1e-4)
    opt2 = FlatAdam(net2.parameters(), lr=1e-4)
    with torch.no_grad():
        net(nodes, edges)
    capacity = int(net.last_stats["entries"] * 1.2) + 32
    # eager reference: the module API in capacity mode with the same capacity, i.e. the same kernels and reduction
    # splits; capacity mode against exact mode is test_capacity_mode_equals_exact_mode / _is_fp64_anchored
    net.entry_capacity = capacity
    losses = []
    for _ in range(2):
        out = net(nodes, edges)
        loss = Fn.kl_loss(out, target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    step = TrainStep(net2, opt2, batch_size=nodes.shape[0], entry_capacity=capacity)
    got = [step(nodes, edges, target).clone() for _ in range(2)]
    assert step.check() & 4 == 0
    # the captured step replays the eager step's launches (K0, packing, forward, loss, backward) with the same capacity:
    # the parameters agree bit for bit.  The losses are float32 sums of the same non-negative loss rows in two orders
    # (torch's for the eager step, gib_sum_scaled's for the captured one): they agree to twice the rounding bound of
    # such a sum (tests/test_gpu_batch_stream.py compares the rows themselves)
    B = nodes.shape[0]
    for a, b in zip(got, losses):
        assert abs(float(a) - float(b)) <= 2 * B * 2.0 ** -24 * abs(float(b)), (got, losses)
    for a, b in zip(net.parameters(), net2.parameters()):
        assert torch.equal(a, b)


@pytest.mark.parametrize("cid", ["A", "M"])
def test_int8_batches_equal_float_batches(cid):
    C, net, nodes, edges, target = _setup(cid)
    out0, loss0, g0 = _step_grads(net, nodes, edges, target)
    out1, loss1, g1 = _step_grads(net, nodes.to(torch.int8), edges.to(torch.int8), target)
    assert torch.equal(out0, out1) and loss0 == loss1
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)


@pytest.mark.parametrize("rid", list(REFUSALS) + ["N91"])
def test_unsupported_dims_are_refused_through_the_module_api(rid):
    """a RuntimeError that names the limit, before any kernel runs on the unsupported dims, and no fault"""
    from oracle import mpnn_oracle as O
    if rid == "N91":        # 91 x 91 x 4 = 33124 > 32768 cells of K0's shared memory
        C, words = O.make_constants("GGNN", max_n_nodes=91, **CONFIGS["A"][1]), "N\\*N\\*groups<=32768"
    else:
        C, words = constants(rid), REFUSALS[rid][2]
    from graphinvent_b200.gnn import mpnn
    net = mpnn.create(C).cuda()
    nodes = torch.zeros(4, C.max_n_nodes, C.n_node_features, device="cuda")
    edges = torch.zeros(4, C.max_n_nodes, C.max_n_nodes, C.n_edge_features, device="cuda")
    edges[:, 0, 1, 0] = edges[:, 1, 0, 0] = 1
    with pytest.raises(RuntimeError, match=words):
        net(nodes, edges)
    torch.cuda.synchronize()
    assert float(torch.ones(8, device="cuda").sum()) == 8.0      # the context is intact
