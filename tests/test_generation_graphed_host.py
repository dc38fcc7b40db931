"""The captured-round generator (graphinvent_b200.graphed.GraphedGenerator) on CPU: the static entry capacity its
capacity-mode forward is sized for, the C-ABI of `gib_generation_sample_round`, and its argument checks.

The capacity rests on one claim about the round state machine: a round adds at most two `edges` non-zeros per slot
(dummy slot 0 included) and a batch runs at most 2N rounds.  The numpy oracle of the reference's generator checks it
after every round, on random action streams and on a scripted worst case."""
import numpy as np
import pytest

from tests.test_generation import _action_stream
from tests.test_generation_layouts import _constants

A, CH = 5, 3


def scripted_worst_case(st, rnd):
    """the longest-lived, most-bonded slots: rounds 0..N-1 add a chain of N atoms (each bonded to the previous one),
    rounds N..2N-3 connect the last atom to every atom it is not bonded to (0..N-3), and from round 2N-2 on every slot
    adds a first atom (bond_to 0): into a full graph that is invalid, so all slots end together one round before the
    2N-round limit with n_generated = B - 1"""
    N, Ef = st.N, st.Ef
    len_add = N * A * CH * Ef
    n = st.n_nodes.astype(np.int64)
    if N <= rnd < 2 * N - 2:
        return np.full(st.B, len_add + (rnd - N) * Ef, np.int32)
    bond_to = np.maximum(n - 1, 0) if rnd < N else np.zeros_like(n)
    return (bond_to * A * CH * Ef).astype(np.int32)          # atom 0, charge 0, bond type 0


def _bond_entries(st):
    return int(np.count_nonzero(st.edges))


@pytest.mark.parametrize("stream,seed,N,Ef,B", [
    ("random", 0, 13, 3, 200), ("random", 1, 5, 2, 64), ("random", 2, 38, 3, 48),
    ("scripted", 0, 5, 3, 32), ("scripted", 0, 13, 3, 40),
])
def test_bond_entries_stay_within_the_static_capacity(stream, seed, N, Ef, B):
    from graphinvent_b200.graphed import entry_capacity
    from oracle import generation_oracle as G
    rng = np.random.default_rng(seed)
    st = G.GenerationState(B, N, A, CH, Ef)
    len_add = N * A * CH * Ef
    apd = len_add + N * Ef + 1
    assert _bond_entries(st) == 1
    for rnd in range(2 * N):
        a = scripted_worst_case(st, rnd) if stream == "scripted" else _action_stream(rng, st, apd, len_add)
        G.generation_round(st, rnd, a, rng.random(B).astype(np.float32))
        assert _bond_entries(st) <= 1 + 2 * B * (rnd + 1), rnd
        if stream == "scripted" and rnd == 2 * N - 3:
            # every slot but the dummy one holds 2N - 3 bonds: two non-zeros per slot in every round but the first
            assert int(np.count_nonzero(st.edges[1:])) == 2 * (B - 1) * (2 * N - 3)
    if stream == "scripted":
        assert st.n_generated == B - 1          # the batch needs a round 2N: the generator raises
    assert entry_capacity(B, N, Ef) == min(1 + 4 * B * N, B * N * N * Ef) >= _bond_entries(st)
    assert entry_capacity(1000, 13, 3) == 52001 and entry_capacity(1000, 38, 3) == 152001
    assert entry_capacity(2, 2, 1) == 8                         # bounded by the size of `edges`


def test_sample_round_symbol_is_exported_bound_and_versioned():
    from graphinvent_b200 import _lib
    assert "gib_generation_sample_round" in _lib.exported_symbols()
    assert _lib.ABI_VERSION == 206 == _lib.lib.gib_version()
    assert _lib.lib.gib_generation_sample_round.restype is not None


def _call(B=8, N=13, F=15, Ef=3, H=4, C=3, apd=None):
    from graphinvent_b200._lib import lib
    if apd is None:
        apd = N * (A * CH * max(H, 1) * max(C, 1) * Ef + Ef) + 1
    return lib.gib_generation_sample_round(B, N, F, Ef, A, CH, H, C, None, apd, *([None] * 13), 16, None, None, None)


def test_sample_round_refuses_inconsistent_arguments_before_any_launch():
    """every refusal is a -1 with a message, decided on the host: the null device pointers are never touched"""
    from graphinvent_b200._lib import lib
    N = 13
    cases = [dict(F=14), dict(F=16), dict(C=4), dict(F=5 + 3 + 256 + 3, H=256), dict(F=5 + 3 + 4 - 1, C=-1),
             dict(B=0), dict(B=-3), dict(N=128, apd=128 * (540 * 3 + 3) + 1), dict(Ef=0),
             dict(apd=N * (540 + 3) + 2), dict(apd=N * (540 + 3)), dict(F=8, H=0, C=0, apd=N * (45 + 3) + 1 + 1)]
    for kw in cases:
        assert _call(**kw) == -1, kw
        assert b"gib_generation_round" in lib.gib_last_error(), kw
    assert b"apd" in (_call(apd=7) == -1 and lib.gib_last_error())


@pytest.mark.parametrize("overrides,kw", [
    (dict(n_node_features=14), {}),
    (dict(len_f_add_per_node=180), {}),
    (dict(n_chirality=0), {}),
    ({}, dict(n_imp_H=0)),
    ({}, dict(n_chirality=-3, n_imp_H=10)),
    (dict(n_atom_types=0, n_node_features=10, len_f_add_per_node=0), {}),
])
def test_graphed_generator_refuses_inconsistent_layout_dims_before_allocating(monkeypatch, overrides, kw):
    from graphinvent_b200.generation import GraphGenerator
    from graphinvent_b200.graphed import GraphedGenerator

    def no_allocation(self):
        raise AssertionError("allocated before validating the layout")
    monkeypatch.setattr(GraphGenerator, "_allocate", no_allocation)
    monkeypatch.setattr(GraphedGenerator, "_allocate", no_allocation)
    with pytest.raises(ValueError, match="inconsistent action layout"):
        GraphedGenerator(None, 8, constants=_constants("L3", **overrides), device="cpu", **kw)
