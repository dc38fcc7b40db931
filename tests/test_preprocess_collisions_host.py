"""CPU: the restated state hash of the training-set construction (tests/preprocess_reference.py) against the collision
fixture (tests/golden/preprocess_collisions.npz, tests/golden/make_preprocess_collisions.py), and the C-ABI of the
hook that exposes the device's per-state hashes (gib_test_route_plan_offsets).

The GPU tests (tests/test_gpu_preprocess_collisions.py) rely on the fixture's states colliding under the device's
hash; here a change to the restated mix or to the fixture's molecules fails on its own, without a GPU."""
import ctypes
import os

import numpy as np
import pytest

from tests import preprocess_reference as P
from tests.conftest import GOLDEN

NEW_SYMBOLS = ("gib_test_route_plan_offsets",)
SEGS = P.segments(5, 3)
U = np.uint64


@pytest.fixture(scope="module")
def fx():
    return np.load(os.path.join(GOLDEN, "preprocess_collisions.npz"))


def _dims(**kw):
    from graphinvent_b200._lib import PPDims
    d = dict(N=13, F=8, Ef=3, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0, batch_size=100)
    d.update(kw)
    return PPDims(**d)


def _bytes(X, E):
    return [x.tobytes() + e.tobytes() for x, e, _ in P.route(X, E, SEGS)]


def test_mix64_is_splitmix64():
    """splitmix64's first output for seed 0, and the finaliser applied to (position << 8) | byte"""
    assert int(P.mix64(0)) == 0xE220A8397B1DCDAF
    assert int(P.byte_hash(3, 1)) == int(P.mix64((3 << 8) | 1)) and int(P.byte_hash(3, 0)) == 0
    assert int(P.byte_hash(2, -1)) == int(P.mix64((2 << 8) | 0xFF))          # a byte is mixed unsigned


def test_state_hash_is_additive_and_remapped():
    rng = np.random.default_rng(0)
    X = rng.integers(0, 2, (13, 8)).astype(np.int8)
    E = rng.integers(0, 2, (13, 13, 3)).astype(np.int8)
    nz = np.flatnonzero(np.concatenate([X.ravel(), E.ravel()]))
    with np.errstate(over="ignore"):
        want = U(0)
        for q in nz.tolist():
            want = want + P.mix64((q << 8) | 1)
    assert P.state_hash(X, E) == want
    assert P.state_hash(np.zeros_like(X), np.zeros_like(E)) == 0
    assert P.stored_hash(P.RESERVED) == P.RESERVED - U(1) and P.stored_hash(P.RESERVED - U(1)) == P.RESERVED - U(1)
    assert P.stored_hash(U(5)) == 5


def test_restated_hashes_reproduce_the_fixture(fx):
    nodes, edges, hashes = fx["nodes"], fx["edges"], fx["hashes"]
    assert nodes.shape[1:] == (13, 8) and edges.shape[1:] == (13, 13, 3) and hashes.dtype == np.uint64
    for m in range(nodes.shape[0]):
        assert np.array_equal(P.route_hashes(nodes[m], edges[m], SEGS), hashes[m]), m


def _removed(full, state):
    f, s = np.frombuffer(full, np.int8), np.frombuffer(state, np.int8)
    q = np.flatnonzero(f != s)
    return tuple(zip(q.tolist(), f[q].tolist()))


def test_colliding_states_differ_in_their_bytes(fx):
    """the first collide_states route states of the base (molecule 0) and its colliders share one hash each and have
    pairwise different bytes.  At every step, two of these routes' states share a hash exactly when their bytes are
    equal or the routes have removed the same bytes so far (the hash is additive and the full graphs collide)"""
    nodes, edges, hashes = fx["nodes"], fx["edges"], fx["hashes"]
    cls = np.concatenate([[0], fx["colliders"]])
    k_max = int(fx["collide_states"])
    assert cls.size >= 4 and k_max == 13
    states = {int(m): _bytes(nodes[m], edges[m]) for m in cls}
    for k in range(k_max):
        assert len({int(h) for h in hashes[cls, k]}) == 1, k
        assert len({states[int(m)][k] for m in cls}) == cls.size, k
    for k in range(hashes.shape[1]):
        b = [states[int(m)][k] for m in cls]
        rem = [_removed(states[int(m)][0], states[int(m)][k]) for m in cls]
        for i in range(cls.size):
            for j in range(i):
                same = hashes[cls[i], k] == hashes[cls[j], k]
                assert same == (b[i] == b[j] or rem[i] == rem[j]), (k, i, j)


def test_reserved_key_and_wrap_pairs(fx):
    hashes = fx["hashes"]
    r0, r1 = fx["reserved"]
    assert hashes[r0, 0] == P.RESERVED and hashes[r1, 0] == P.RESERVED - U(1)
    assert P.stored_hash(hashes[r0, 0]) == P.stored_hash(hashes[r1, 0])
    assert _bytes(fx["nodes"][r0], fx["edges"][r0])[0] != _bytes(fx["nodes"][r1], fx["edges"][r1])[0]
    w = hashes[fx["wrap"], 0]
    assert w[0] != w[1]
    for bits in range(10, 21):            # a table of 2^bits slots: both take its last slot
        mask = U((1 << bits) - 1)
        assert (w & mask == mask).all(), bits


def test_fixture_molecules_are_valid_routes(fx):
    """complete graphs of 13 atoms, one-hot nodes, symmetric single-type bonds: routes of N (N - 1) / 2 + 2 states"""
    for X, E in zip(fx["nodes"], fx["edges"]):
        assert (X[:, :5].sum(1) == 1).all() and (X[:, 5:].sum(1) == 1).all()
        assert np.array_equal(E, E.transpose(1, 0, 2)) and (E.sum(2) == 1 - np.eye(13, dtype=np.int64)).all()
        assert len(P.route(X, E, SEGS)) == 13 * 12 // 2 + 2


def test_hook_symbol_is_declared_and_bound():
    from graphinvent_b200 import _lib
    assert set(NEW_SYMBOLS) <= set(_lib.exported_symbols())
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "gib200.h")).read()
    for name in NEW_SYMBOLS:
        assert getattr(_lib.lib, name).argtypes is not None and f"{name}(" in header
    assert _lib.ABI_VERSION == 206 == _lib.lib.gib_version()     # a new symbol: existing entry points unchanged


@pytest.mark.parametrize("N,Ef,lay,M", [(13, 3, (5, 3, 0, 0), 1), (13, 3, (5, 3, 0, 0), 4096),
                                        (38, 4, (4, 3, 4, 3), 77), (181, 1, (5, 3, 0, 0), 3)])
def test_hook_offsets_lie_inside_the_workspace(N, Ef, lay, M):
    """hash (uint64), apd, nn, mol (int32): gib_route_max_states entries each, inside gib_route_plan_ws_bytes, apart"""
    from graphinvent_b200._lib import lib
    A, Fc, H, C = lay
    d = _dims(N=N, F=A + Fc + H + C, Ef=Ef, n_atom_types=A, n_formal_charge=Fc, n_imp_H=H, n_chirality=C)
    out = (ctypes.c_longlong * 4)()
    assert lib.gib_test_route_plan_offsets(ctypes.byref(d), M, out) == 0
    states = lib.gib_route_max_states(ctypes.byref(d), M)
    ws = lib.gib_route_plan_ws_bytes(ctypes.byref(d), M)
    assert states == M * (N * (N - 1) // 2 + 2) and ws > 0
    spans = sorted((o, o + size * states) for o, size in zip(out, (8, 4, 4, 4)))
    assert spans[0][0] >= 0 and spans[-1][1] <= ws
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    assert out[0] % 8 == 0 and all(o % 4 == 0 for o in out)


def test_hook_refuses_bad_dims():
    from graphinvent_b200._lib import lib
    out = (ctypes.c_longlong * 4)(-7, -7, -7, -7)
    for kw, msg in ((dict(N=105), b"N*N*Ef <= 32768"), (dict(F=9), b"sum of the layout"),
                    (dict(batch_size=0), b"batch_size")):
        assert lib.gib_test_route_plan_offsets(ctypes.byref(_dims(**kw)), 10, out) < 0
        assert msg in lib.gib_last_error()
    assert lib.gib_test_route_plan_offsets(ctypes.byref(_dims()), 0, out) < 0
    assert b"max_molecules" in lib.gib_last_error()
    assert lib.gib_test_route_plan_offsets(ctypes.byref(_dims()), 1 << 25, out) < 0
    assert lib.gib_test_route_plan_offsets(None, 10, out) < 0
    assert lib.gib_test_route_plan_offsets(ctypes.byref(_dims()), 10, None) < 0 and b"null" in lib.gib_last_error()
    assert list(out) == [-7] * 4
