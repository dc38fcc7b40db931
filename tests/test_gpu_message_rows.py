"""GPU: the GGNN / MNN message MLPs on message rows (one per source atom, bond type and -- for values other than 1 --
bond entry) against the per-entry path of gib_tc_debug bit 3.

  a. every array of the table the forward builds equals its numpy restatement (tests/msg_rows_reference.py) on K0's
     arrays, with every buffer poisoned and guard-banded: one-hot, multi-type and non-binary bonds, empty molecules and
     atoms without bonds, exact mode, a capacity that fits and one that truncates;
  b. the forward logits of both paths are bit-identical (the GEMMs compute a row from that row alone, K2 sums the same
     values in the same order), tensor cores on and off, exact and capacity mode, and through TrainStep;
  c. their gradients agree to a relative L2 of 1e-5 (duplicate entries are summed before the GEMMs instead of after).
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.msg_rows_reference import TABLE_ARRAYS, msg_rows_reference
from tests.test_gpu_buffer_bounds import _assert_intact, _bits_equal, _model_case, run_step

pytestmark = pytest.mark.gpu

MODELS = ["small_GGNN", "small_MNN"]


class _mode:
    """gib_tc_debug / tensor cores for one block, restored afterwards"""

    def __init__(self, debug=0, tc=True):
        self.debug, self.tc = debug, tc

    def __enter__(self):
        from graphinvent_b200._lib import lib
        lib.gib_tc_debug(self.debug)
        lib.gib_set_tensor_cores(1 if self.tc else 0)

    def __exit__(self, *exc):
        from graphinvent_b200._lib import lib
        lib.gib_tc_debug(0)
        lib.gib_set_tensor_cores(1)


def _edges(edges, kind, seed=0):
    """the fixture's bonds, or the same cells with non-binary values (some 1, a NaN) and extra bond types"""
    e = edges.clone()
    if kind == "onehot":
        return e
    rng = np.random.default_rng(seed)
    a = e.cpu().numpy()
    B, N, _, Ef = a.shape
    b, i, j = np.nonzero(rng.random((B, N, N)) < 0.03)
    a[b, i, j, rng.integers(0, Ef, b.size)] = 1.0                       # a second type on some cells
    if kind == "values":
        nz = np.nonzero(a)
        a[nz] = rng.choice(np.array([0.5, 2.0, 1.0, 1.0, -3.0], np.float32), nz[0].size)
    a[0] = 0.0                                                           # an empty molecule
    return torch.from_numpy(a).to(edges.device)


def _table_of(got, net, B):
    """the table the forward left in the workspace, and its restatement from the K0 arrays in the graph buffer"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import lib
    d = Fn.make_dims(net, B, 0)
    bd = ctypes.byref(d)
    hdr = got["hdr"]
    hp = hdr.ctypes.data_as(ctypes.c_void_p)
    E, P, S = int(hdr[0]), int(hdr[1]), B * d.N
    G = d.Ef
    ws, gb = got["g"]["ws"], got["g"]["graph"]

    def arr(buf, addr, n, dt=torch.int32):
        o = addr - buf.ptr()
        return buf.t[o:o + 4 * n].view(dt).cpu().numpy()

    def k0(which, n, dt=torch.int32):
        return arr(gb, lib.gib_graph_array(bd, hp, ctypes.c_void_p(gb.ptr()), which), n, dt)

    ent_src, ent_dst, ent_w = k0(0, P), k0(1, P), k0(2, P, torch.float32)
    dst_ptr, dst_ent, src_ptr, src_ent = k0(3, S + 1), k0(4, E), k0(5, S + 1), k0(6, E)
    tb = got["g"]["cws"].view(torch.int32)[6:11].cpu().numpy() if hdr[12] else hdr[6:11]
    ref = msg_rows_reference(ent_src, ent_dst, ent_w, dst_ptr, dst_ent, src_ptr, src_ent, tb, G, E)
    n = dict(u_src=P, u_w=P, u_ptr=P + 1, u_dst=E, ent_u=P, dst_u=E, s_ptr=S + 1, s_u=E, meta=16)
    table = {}
    for k, name in enumerate(TABLE_ARRAYS):
        addr = lib.gib_model_msg_rows(bd, hp, ctypes.c_void_p(ws.ptr()), k)
        assert addr, name
        table[name] = arr(ws, addr, n[name])
    ref["u_w"] = ref["u_w"].view(np.int32)
    return table, ref


@pytest.mark.parametrize("kind", ["onehot", "multitype", "values"])
@pytest.mark.parametrize("name", MODELS)
def test_table_matches_its_restatement(name, kind):
    C, net, nodes, edges, target = _model_case(name)
    e = _edges(edges, kind)
    B = nodes.shape[0]
    exact = run_step(net, nodes, e, target, None, "poison")
    E = int(exact["hdr"][0])
    for cap in (None, E + 300, int(E * 0.8)):
        got = exact if cap is None else run_step(net, nodes, e, target, cap, "poison")
        what = f"{name} {kind} capacity={cap}"
        _assert_intact(got["g"], what)
        table, ref = _table_of(got, net, B)
        for k in TABLE_ARRAYS:
            assert np.array_equal(table[k], ref[k]), (what, k, np.flatnonzero(table[k] != ref[k])[:8])


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("kind", ["onehot", "values"])
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "fp32"])
@pytest.mark.parametrize("name", MODELS)
def test_message_rows_match_the_per_entry_path(name, tc, kind):
    C, net, nodes, edges, target = _model_case(name)
    e = _edges(edges, kind)
    with _mode(0, tc):
        E = int(run_step(net, nodes, e, target, None, "zero")["hdr"][0])
    for cap in ((None, E + 300) if tc else (None,)):      # capacity mode needs the tensor-core call pattern
        with _mode(0, tc):
            new = run_step(net, nodes, e, target, cap, "poison")
        with _mode(8, tc):
            old = run_step(net, nodes, e, target, cap, "poison")
        what = f"{name} {kind} {'tc' if tc else 'fp32'} capacity={cap}"
        assert torch.isfinite(new["out"]).all(), what
        assert _bits_equal(new["out"], old["out"]), what
        assert _bits_equal(new["loss"], old["loss"]), what
        assert _rel(new["grads"], old["grads"]) <= 1e-5, (what, _rel(new["grads"], old["grads"]))


@pytest.mark.parametrize("name", MODELS)
def test_train_step_logits_match_the_per_entry_path(name):
    from graphinvent_b200.graphed import TrainStep
    from graphinvent_b200.optim import FlatAdam
    C, net, nodes, edges, target = _model_case(name)
    B = nodes.shape[0]
    cap = int((edges != 0).sum()) + 300
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    outs = {}
    for debug in (0, 8):          # the captured step: capacity mode, device-side row counts
        with _mode(debug):
            net.load_state_dict(sd)
            step = TrainStep(net, FlatAdam(net.parameters(), lr=1e-4), batch_size=B, entry_capacity=cap)
            loss = step(nodes, edges, target)
            torch.cuda.synchronize()
            outs[debug] = (step.out.clone(), loss.clone())
            del step
    assert _bits_equal(outs[0][0], outs[8][0]), name
    assert _bits_equal(outs[0][1], outs[8][1]), name
