"""CPU: the route scorer's C-ABI (symbols, size queries, argument refusals), RouteScorer's layout checks against
GraphedGenerator's, and the fp64 restatement (tests/route_nll_reference.py) against the live reference's route
likelihoods of gdb13 molecules under the pretrained GGNN (tests/golden/route_nll_gdb13.npz)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import preprocess_reference as P
from tests import route_nll_reference as R
from tests.conftest import GOLDEN, pretrained_path

NEW_SYMBOLS = ("gib_route_plan_ws_bytes", "gib_route_max_states", "gib_route_plan", "gib_route_fill",
               "gib_route_probs", "gib_route_reduce")


def _dims(**kw):
    from graphinvent_b200._lib import PPDims
    d = dict(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=100)
    d.update(kw)
    return PPDims(**d)


def test_symbols_are_exported_and_bound():
    from graphinvent_b200 import _lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    for name in NEW_SYMBOLS:
        assert getattr(_lib.lib, name).argtypes is not None
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "gib200.h")).read()
    assert all(f"{name}(" in header for name in NEW_SYMBOLS)


def test_size_queries():
    from graphinvent_b200._lib import lib
    d = _dims()
    s_max = 13 * 12 // 2 + 2
    assert lib.gib_route_max_states(ctypes.byref(d), 10) == 10 * s_max
    small, large = (lib.gib_route_plan_ws_bytes(ctypes.byref(d), m) for m in (10, 1000))
    assert 0 < small < large
    # the states of a chunk (hash, action, node count, molecule) and its bond steps fit
    assert large >= 1000 * s_max * (8 + 4 + 4 + 4) + 1000 * 13 * 13 * 2
    assert lib.gib_route_plan_ws_bytes(ctypes.byref(d), 0) == 0 and b"max_molecules" in lib.gib_last_error()
    assert lib.gib_route_max_states(ctypes.byref(d), 1 << 25) < 0
    for kw, msg in ((dict(N=105), b"N*N*Ef <= 32768"), (dict(F=9), b"sum of the layout"),
                    (dict(batch_size=0), b"batch_size")):
        d = _dims(**kw)
        assert lib.gib_route_plan_ws_bytes(ctypes.byref(d), 10) == 0 and msg in lib.gib_last_error()
        assert lib.gib_route_max_states(ctypes.byref(d), 10) < 0


def test_entry_points_refuse_bad_arguments():
    from graphinvent_b200._lib import lib
    d = _dims()
    p, a16 = ctypes.c_void_p(64), ctypes.c_void_p(64)
    bd = ctypes.byref(d)
    assert lib.gib_route_plan(bd, p, p, 0, 10, p, p, p, None) < 0 and b"n_molecules" in lib.gib_last_error()
    assert lib.gib_route_plan(bd, p, p, 11, 10, p, p, p, None) < 0 and b"n_molecules" in lib.gib_last_error()
    assert lib.gib_route_plan(bd, None, p, 5, 10, p, p, p, None) < 0 and b"null" in lib.gib_last_error()
    assert lib.gib_route_plan(bd, p, p, 5, 0, p, p, p, None) < 0 and b"max_molecules" in lib.gib_last_error()
    assert lib.gib_route_plan(ctypes.byref(_dims(F=9)), p, p, 5, 10, p, p, p, None) < 0
    fill = lambda *a: lib.gib_route_fill(bd, *a, None)
    assert fill(p, p, 10, p, p, p, p, None, p, p) < 0 and b"null" in lib.gib_last_error()
    assert fill(ctypes.c_void_p(65), p, 10, p, p, p, p, p, a16, a16) < 0 and b"16-byte" in lib.gib_last_error()
    assert fill(p, p, 10, p, p, p, p, p, a16, ctypes.c_void_p(72)) < 0 and b"16-byte" in lib.gib_last_error()
    assert fill(p, p, 0, p, p, p, p, p, a16, a16) < 0 and b"max_molecules" in lib.gib_last_error()
    assert lib.gib_route_probs(0, 625, p, p, p, None) < 0 and b"gib_route_probs" in lib.gib_last_error()
    assert lib.gib_route_probs(4, 625, p, None, p, None) < 0
    assert lib.gib_route_reduce(0, p, p, p, p, None) < 0 and b"gib_route_reduce" in lib.gib_last_error()
    assert lib.gib_route_reduce(3, p, p, None, p, None) < 0


def _model():
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    return mpnn.create(O.make_constants("GGNN"))


GDB13 = dict(n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0)


@pytest.mark.parametrize("kw", [dict(n_atom_types=4), dict(n_formal_charge=0), dict(n_imp_H=2),
                                dict(n_chirality=-1), dict(n_atom_types=300, n_formal_charge=3)])
def test_layout_checks_mirror_the_generators(kw):
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import RouteScorer
    net = _model()
    kw = {**GDB13, **kw}
    with pytest.raises(ValueError) as gen:
        GraphGenerator(net, 4, **kw)
    with pytest.raises(ValueError) as sc:
        RouteScorer(net, 4, **kw)
    assert str(sc.value) == str(gen.value) and "inconsistent action layout" in str(sc.value)


def test_foreign_models_are_refused():
    from graphinvent_b200.graphed import RouteScorer
    net = _model()

    class Foreign(torch.nn.Module):
        constants = net.constants

    with pytest.raises(TypeError, match="this package's models"):
        RouteScorer(Foreign(), 4, **GDB13)


def test_restatement_states_are_the_reference_route_reversed():
    """the states tests/preprocess_reference.route walks, reversed, are the build order: the first is empty with a
    first-atom action, the last is the full graph with terminate, n_edges + 2 per molecule"""
    z = np.load(os.path.join(GOLDEN, "route_nll_gdb13.npz"))
    X, E, acts, offsets = R.build_order_states(z["nodes"][:8], z["edges"][:8], P.segments(5, 3))
    for m in range(8):
        a, b = offsets[m], offsets[m + 1]
        assert b - a == int(z["edges"][m].sum()) // 2 + 2
        assert not X[a].any() and not E[a].any() and acts[a] < 5 * 3 * 3
        assert np.array_equal(X[b - 1], z["nodes"][m]) and np.array_equal(E[b - 1], z["edges"][m])
        assert acts[b - 1] == 624


def test_restatement_matches_the_live_reference():
    """fixture: the reference's get_decoding_route_state actions and Softmax(model) probabilities (fp32) of the
    pretrained GGNN; the restatement reproduces the actions exactly and the probabilities within the reference's
    own fp32 rounding (|d log p| <= 2 max |d logit|, logits within 1e-4)"""
    path = pretrained_path()
    if path is None:
        pytest.skip("oracle/_ref/pretrained_model.pth absent: run __graft_entry__.build() with a checkout of the reference")
    from oracle import mpnn_oracle as O
    z = np.load(os.path.join(GOLDEN, "route_nll_gdb13.npz"))
    sd = torch.load(path, map_location="cpu", weights_only=False)
    assert str(z["sha256"]) == __import__("hashlib").sha256(open(path, "rb").read()).hexdigest()
    X, E, acts, offsets = R.build_order_states(z["nodes"], z["edges"], P.segments(5, 3))
    assert np.array_equal(acts, z["actions"]) and np.array_equal(offsets, z["offsets"])
    C = O.make_constants("GGNN")
    p, logits = R.probabilities(sd, C, X, E, acts)
    b = R.log_p_bound(sd, C, X, E, acts, logits)
    ref = torch.from_numpy(z["likelihoods"])
    nll, final = R.reduce(ref.double(), offsets)
    R.assert_within(ref, nll.float(), final.float(), (p, offsets, *R.reduce(p, offsets), b), "live reference")
