"""CPU: the host-side plan and size queries (pure C++ host code, callable without a GPU) across the reference's
hyper-parameter range -- one row per branch of csrc/model.cu that the default dims never reach.  The same table drives
tests/test_gpu_model_dims.py, which runs every row on the device against fp64."""
import ctypes
import math

import numpy as np
import pytest

from graphinvent_b200.config import layout_dims

# aromatic bonds (the reference's use_aromatic_bonds, parameters/constants.py:161-166): 4 bond types, 5 atom types and
# 3 formal charges as in gdb13
EF4 = layout_dims(5, 3, 4)
SMALL = dict(hidden_node_features=64, message_size=64, enn_hidden_dim=64, gather_width=64, gather_att_hidden_dim=64,
             gather_emb_hidden_dim=64, mlp1_hidden_dim=64, mlp2_hidden_dim=64)
ALL_DEPTHS = ("enn_depth", "gather_att_depth", "gather_emb_depth", "mlp1_depth", "mlp2_depth")

# id -> (model, constants overrides, atom types, formal charges, molecules, what the row reaches)
CONFIGS = {
    "A": ("GGNN", dict(EF4), 5, 3, 50,
          "4 type groups; 5 x 4 = 20 > 16 message-MLP layers: the capacity-mode backward runs in sub-groups"),
    "B": ("GGNN", dict(EF4, enn_depth=3), 5, 3, 50, "exactly 16 problems in one chain and one dW group"),
    "C4": ("MNN", dict(EF4), 5, 3, 50, "strided message_weights slices [M, H, 4] and their dW"),
    "C1": ("MNN", layout_dims(5, 3, 1), 5, 3, 50, "one bond type: message_weights [M, H, 1]"),
    "D": ("AttGGNN", dict(EF4, msg_depth=1, att_depth=3, message_passes=1), 5, 3, 50,
          "msg / att of unequal depth; one pass, where the t == 0 skips are the whole backward"),
    "E": ("EMN", dict(EF4, edge_emb_depth=0, msg_depth=2, att_depth=5, message_passes=1), 5, 3, 50,
          "embedding_nn as one Linear with Ct = 0; siblings of unequal depth; emn_input with 2F + 4 columns"),
    "F": ("GGNN", {k: 0 for k in ALL_DEPTHS}, 5, 3, 50,
          "every MLP a single Linear; the APD heads write the logits from their first layer"),
    "G": ("GGNN", {k: 7 for k in ALL_DEPTHS}, 5, 3, 50,
          "8-layer chains; gather siblings fill 16 problems; the three heads (24) fall back"),
    "H": ("GGNN", dict(gather_att_depth=1, gather_emb_depth=3, mlp1_depth=2, mlp2_depth=0), 5, 3, 50,
          "readout siblings of unequal depth"),
    "I": ("GGNN", dict(hidden_node_features=17, message_size=33, enn_hidden_dim=1, gather_width=1, mlp1_hidden_dim=47,
                       mlp2_hidden_dim=129), 5, 3, 50, "widths < 48 and 1 padded to 16; 129 crosses a 128-row tile"),
    "J": ("GGNN", dict(hidden_node_features=300, message_size=300, enn_hidden_dim=640, gather_att_hidden_dim=640,
                       gather_emb_hidden_dim=640, mlp1_hidden_dim=640, mlp2_hidden_dim=700, gather_width=257),
          5, 3, 40, "K > 608 over several column tiles; gate-blocked GRU rows 3 x 304"),
    "K": ("GGNN", dict(SMALL, message_passes=16), 5, 3, 50, "the deepest layout (16 passes)"),
    "L": ("GGNN", dict(max_n_nodes=2), 5, 3, 50, "K0 and the graph gather at N = 2"),
    "M": ("GGNN", dict(SMALL, max_n_nodes=90, **layout_dims(2, 1, 4)), 2, 1, 8,
          "K0 at N^2 x 4 = 32400 cells (about 222 KB of shared memory); APD heads 90 x f_add wide"),
}

# dims every size query must refuse, and the words of the refusal
REFUSALS = {
    "depth8": ("GGNN", dict(enn_depth=8), "depth 8"),
    "T17": ("GGNN", dict(message_passes=17), "message_passes <= 16"),
    "Ef5": ("GGNN", dict(n_edge_features=5, len_f_conn_per_node=5), "n_edge_features <= 4"),
    "Linears97": ("AttGGNN", dict(EF4, msg_depth=6, att_depth=6, gather_att_depth=6, gather_emb_depth=6),
                  "97 Linears"),
}


def constants(cid):
    from oracle import mpnn_oracle as O
    model, kw, *_ = CONFIGS[cid] if cid in CONFIGS else REFUSALS[cid]
    return O.make_constants(model, **kw)


def _dims(C, B=64):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.gnn import mpnn
    return Fn.make_dims(mpnn.create(C), B)


def _exact_header(counts):
    """host header of K0's exact mode: per-type counts, each group padded to a multiple of 128 rows"""
    h = np.zeros(16, np.int32)
    base = 0
    for t, c in enumerate(counts):
        h[2 + t], h[6 + t] = c, base
        base += (c + 127) // 128 * 128
    h[6 + len(counts)] = base
    h[0], h[1] = sum(counts), base
    return h


def _capacity_header(lib, d, capacity):
    # gib_graph_header_capacity only records the device header's address; any non-null address serves the size queries
    dev_ws = ctypes.create_string_buffer(64)
    h = np.zeros(16, np.int32)
    assert lib.gib_graph_header_capacity(ctypes.byref(d), capacity, ctypes.addressof(dev_ws),
                                         h.ctypes.data_as(ctypes.c_void_p)) == 0
    return h, dev_ws


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_plan_matches_reference_parameter_schema(cid):
    from graphinvent_b200._lib import lib
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    C = constants(cid)
    shapes = O.param_shapes(C)
    sd = mpnn.create(C).state_dict()
    assert [k for k, _ in shapes] == list(sd.keys())
    assert all(tuple(sd[k].shape) == tuple(s) for k, s in shapes)
    d = _dims(C)
    assert lib.gib_model_num_params(ctypes.byref(d)) == len(shapes), lib.gib_last_error()
    for i, (k, s) in enumerate(shapes):
        assert lib.gib_model_param_numel(ctypes.byref(d), i) == math.prod(s), k
    assert lib.gib_model_packed_bytes(ctypes.byref(d)) >= 4 * sum(math.prod(s) for _, s in shapes)


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_plan_linear_offsets_are_disjoint_and_inside_the_packed_arena(cid):
    from graphinvent_b200._lib import PLAN_LINEAR_FIELDS, lib
    d = _dims(constants(cid))
    total = lib.gib_model_packed_bytes(ctypes.byref(d)) // 4
    out = (ctypes.c_longlong * len(PLAN_LINEAR_FIELDS))()
    n = lib.gib_test_plan_linear(ctypes.byref(d), 0, out)
    assert 0 < n <= 96
    ranges = []
    for i in range(n):
        assert lib.gib_test_plan_linear(ctypes.byref(d), i, out) == n
        f = dict(zip(PLAN_LINEAR_FIELDS, out))
        Rp = f["nblk"] * f["Rbp"]
        assert f["Rbp"] == (f["Rb"] + 15) // 16 * 16 and f["Cp"] == (f["C"] + 15) // 16 * 16
        assert f["Ctp"] == (f["Ct"] + 15) // 16 * 16 and 0 <= f["Ct"] <= f["C"]
        for name, size in (("ow", Rp * f["Cp"]), ("owt", f["Ctp"] * Rp), ("ob", Rp), ("ow_hi", Rp * f["Cp"]),
                           ("ow_lo", Rp * f["Cp"]), ("owt_hi", f["Ctp"] * Rp), ("owt_lo", f["Ctp"] * Rp)):
            if size:
                ranges.append((f[name], f[name] + size, i, name))
    ranges.sort()
    assert ranges[0][0] >= 0 and ranges[-1][1] <= total
    for a, b in zip(ranges, ranges[1:]):
        assert a[1] <= b[0], f"{a[2:]} overlaps {b[2:]}"


def test_the_rows_reach_their_layouts():
    """the plan facts the table's rows exist for"""
    from graphinvent_b200._lib import PLAN_LINEAR_FIELDS, lib

    def lins(cid):
        d = _dims(constants(cid))
        out = (ctypes.c_longlong * len(PLAN_LINEAR_FIELDS))()
        n = lib.gib_test_plan_linear(ctypes.byref(d), 0, out)
        rows = []
        for i in range(n):
            lib.gib_test_plan_linear(ctypes.byref(d), i, out)
            rows.append(dict(zip(PLAN_LINEAR_FIELDS, out)))
        return rows

    mnn = lins("C4")[:4]          # message_weights [M, H, 4]: four strided slices of one parameter
    H = constants("C4").hidden_node_features
    assert [(f["pw"], f["pb"], f["src_off"], f["rs"], f["cs"]) for f in mnn] == [(0, -1, t, H * 4, 4) for t in range(4)]
    assert lins("E")[0]["Ct"] == 0 and lins("E")[0]["C"] == 2 * 8 + 4   # embedding_nn: one Linear, no transposed copy
    assert len(lins("G")) == 3 * 8 + 2 + 2 * 8 + 5 * 8 == 82
    assert max(f["Cp"] for f in lins("J")) > 608


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_workspace_and_scratch_queries_for_exact_and_capacity_headers(cid):
    from graphinvent_b200._lib import lib
    C = constants(cid)
    d = _dims(C, 256)
    groups = 1 if C.model == "EMN" else C.n_edge_features
    sizes = []
    for counts in ([1000, 300, 20, 90][:groups], [4000, 1200, 80, 360][:groups]):
        h = _exact_header(counts).ctypes.data_as(ctypes.c_void_p)
        w = lib.gib_model_workspace_bytes(ctypes.byref(d), h)
        s = lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), h)
        assert w > 0 and s > 0, lib.gib_last_error()
        sizes.append((w, s))
    assert sizes[0][0] < sizes[1][0] and sizes[0][1] <= sizes[1][1]
    for cap in (2000, 8000):
        h, _keep = _capacity_header(lib, d, cap)
        hp = h.ctypes.data_as(ctypes.c_void_p)
        assert lib.gib_model_workspace_bytes(ctypes.byref(d), hp) > 0, lib.gib_last_error()
        assert lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), hp) > 0, lib.gib_last_error()


@pytest.mark.parametrize("rid", list(REFUSALS))
def test_size_queries_refuse_unsupported_dims(rid):
    from graphinvent_b200._lib import lib
    C = constants(rid)
    d = _dims(C)
    words = REFUSALS[rid][2]
    assert lib.gib_model_num_params(ctypes.byref(d)) < 0
    assert words in lib.gib_last_error().decode()
    assert lib.gib_model_packed_bytes(ctypes.byref(d)) == 0
    assert words in lib.gib_last_error().decode()
    h = _exact_header([100] * (1 if C.model == "EMN" else min(C.n_edge_features, 4)))
    assert lib.gib_model_workspace_bytes(ctypes.byref(d), h.ctypes.data_as(ctypes.c_void_p)) == 0
    assert words in lib.gib_last_error().decode()
    assert lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), h.ctypes.data_as(ctypes.c_void_p)) == 0


@pytest.mark.parametrize("N,Ef", [(91, 4), (182, 1), (13, 5)])
def test_graph_count_validates_dims_before_any_launch(N, Ef):
    """K0 keeps the N x N x groups cells of one molecule in shared memory (at most 32768; row M of CONFIGS runs
    N = 90, Ef = 4 on the device); the refusal comes before the first CUDA call, so it is host-testable"""
    from graphinvent_b200._lib import lib
    from oracle import mpnn_oracle as O
    d = _dims(O.make_constants("GGNN", max_n_nodes=N, n_edge_features=Ef, len_f_conn_per_node=Ef), 8)
    assert lib.gib_graph_count(ctypes.byref(d), None, None, None) < 0
    assert "N*N*groups<=32768" in lib.gib_last_error().decode()
