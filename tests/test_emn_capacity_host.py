"""CPU: capacity mode covers the EMN -- the host-side size queries of a capacity header (pure C++ host code, callable
without a GPU) size its bond-row buffers from the entry capacity."""
import ctypes

import numpy as np
import pytest


def _capacity_header(lib, d, capacity):
    # gib_graph_header_capacity only records the device header's address; any non-null address serves the size queries
    dev_ws = ctypes.create_string_buffer(64)
    h = np.zeros(16, np.int32)
    assert lib.gib_graph_header_capacity(ctypes.byref(d), capacity, ctypes.addressof(dev_ws),
                                         h.ctypes.data_as(ctypes.c_void_p)) == 0
    return h


@pytest.mark.parametrize("kw", [{}, dict(msg_depth=2, att_depth=4)], ids=["default", "unequal_depths"])
def test_emn_capacity_header_sizes_workspace_and_scratch(kw):
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import lib
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    net = mpnn.create(O.make_constants("EMN", **kw))
    d = Fn.make_dims(net, 1000)
    ws, scratch = [], []
    for cap in (10000, 30000, 60000):
        h = _capacity_header(lib, d, cap).ctypes.data_as(ctypes.c_void_p)
        w = lib.gib_model_workspace_bytes(ctypes.byref(d), h)
        assert w > 0, lib.gib_last_error()
        ws.append(w)
        scratch.append(lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), h))
    assert 0 < ws[0] < ws[1] < ws[2]
    assert 0 < scratch[0] < scratch[1] < scratch[2]
    # the EMN's message passing runs on bond rows: every extra entry of capacity costs at least one row of each of
    # the T+1 memories (edge_emb_size floats, padded to 16)
    Hp = (d.H + 15) // 16 * 16
    assert ws[2] - ws[1] >= 30000 * (d.T + 1) * Hp * 4
