"""CPU: the scaffold oracle's start state, round-robin reset and mask rule on hand-made cases, the scaffold entry
capacity and record size, and the new C-ABI symbols' argument refusals (host code, no launch)."""
import ctypes

import numpy as np

from tests import scaffold_oracle as SO

N, A, CH, EF = 5, 2, 1, 2


def _scaffolds():
    """three scaffolds: one atom; two bonded atoms; a 4-atom chain (N - 1)"""
    F = A + CH
    nodes = np.zeros((3, N, F), np.int8)
    edges = np.zeros((3, N, N, EF), np.int8)
    for s, k in enumerate((1, 2, 4)):
        nodes[s, :k, 0] = 1
        nodes[s, :k, A] = 1
        for i in range(1, k):
            edges[s, i - 1, i, 0] = edges[s, i, i - 1, 0] = 1
    return nodes, edges


def _apd():
    return N * (A * CH * EF) + N * EF + 1


def test_start_state_and_round_robin_reset():
    nodes, edges = _scaffolds()
    B = 6
    st = SO.ScaffoldState(B, N, A, CH, EF, 0, 0, nodes, edges)
    assert st.slot_ids.tolist() == [-1, 0, 1, 2, 0, 1] and st.started == B - 1
    assert st.n_nodes.tolist() == [1, 1, 2, 4, 1, 2]
    term = _apd() - 1
    per_node = A * CH * EF
    # slot 5 terminates, slot 2 takes an invalid connect (self loop), slot 3 terminates; the rest add a bonded atom
    a = np.array([0] * B, np.int32)
    a[1] = 0 * per_node                        # add onto atom 0 of the single-atom scaffold
    a[4] = 0 * per_node + 1                    # add with bond type 1
    a[2] = N * per_node + 1 * EF               # connect bond_from = 1 -> bond_to = 1: a self loop, invalid
    a[3] = term
    a[5] = term
    lik = np.arange(1, B + 1, dtype=np.float32) / 10
    assert SO.generation_round(st, 0, a, lik) == 3
    # copy-out: terminate-sampled (3, 5) first, then invalid (2); restart in slot order 2, 3, 5 from started = 5
    assert st.generated_scaffolds[:3].tolist() == [2, 1, 1]
    assert st.generated_n_nodes[:3].tolist() == [4, 2, 2]
    assert st.slot_ids.tolist() == [-1, 0, (5 + 0) % 3, (5 + 1) % 3, 0, (5 + 2) % 3]
    assert st.started == 8
    assert st.n_nodes.tolist() == [1, 2, 4, 1, 2, 2]
    assert (st.likelihoods[[2, 3, 5]] == 0).all() and st.likelihoods[1, 0] == lik[1]
    assert (st.edges[2] == edges[2]).all() and (st.nodes[3] == nodes[0]).all()


def test_mask_rule():
    nodes, edges = _scaffolds()
    st = SO.ScaffoldState(4, N, A, CH, EF, 0, 0, nodes, edges)
    protect = SO.protect_of(st.k, [[0], [1], [0, 3]], N)
    assert protect.tolist()[2] == [False, True, True, False, False]
    per_node = A * CH * EF
    len_add = N * per_node
    assert not SO.forbidden(st, 0, protect).any()
    assert not SO.forbidden(st, 1, None).any()
    m = SO.forbidden(st, 2, protect)             # scaffold 1: atom 0 protected; n = k: every connect forbidden
    assert m[:per_node].all() and not m[per_node:len_add].any() and m[len_add:-1].all() and not m[-1]
    st.n_nodes[3] = 5                            # scaffold 2 after one add: connects onto atoms 1, 2 only forbidden
    m = SO.forbidden(st, 3, protect)
    assert not m[:per_node].any() and m[per_node:3 * per_node].all() and not m[3 * per_node:len_add].any()
    conn = m[len_add:-1].reshape(N, EF)
    assert conn.all(1).tolist() == [False, True, True, False, False] and not m[-1]


def test_scaffold_entry_capacity_and_record_bytes():
    from graphinvent_b200.graphed import entry_capacity, rl_record_bytes, scaffold_entry_capacity
    assert scaffold_entry_capacity(1000, 13, 3, 0) == entry_capacity(1000, 13, 3)
    assert scaffold_entry_capacity(1000, 13, 3, 12) == 1 + 4 * 1000 * 13 + 2 * 999 * 12
    assert scaffold_entry_capacity(2, 3, 1, 100) == 2 * 9
    assert rl_record_bytes(100, 13, 8, 3, masked=True) - rl_record_bytes(100, 13, 8, 3) == 2 * 13 * 100 * 8


def test_scaffold_entry_points_refuse_bad_arguments():
    from graphinvent_b200._lib import Scaffolds, lib
    sc = Scaffolds()
    assert lib.gib_generation_scaffold_init(4, N, 3, EF, ctypes.byref(sc), None, None, None, None, None) < 0
    assert b"scaffold table" in lib.gib_last_error()
    assert lib.gib_generation_mask_logits(4, N, EF, _apd() + 1, ctypes.byref(sc), None, None, None, None, None,
                                          None, None) < 0
    assert lib.gib_rl_snapshot_scaffold(4, N, None, None, None, None, None, None, None) < 0


# ---- the reference generator decorating scaffolds (tests/golden/generation_scaffold_traces.npz) --------------------
TRACES = ("L0", "L0_attach", "L3", "L3_attach")


def scaffold_trace(name):
    import os
    from tests.conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "generation_scaffold_traces.npz"))
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def replay_oracle(z):
    """the scaffold oracle on the trace's draws and stored likelihoods"""
    from tests.test_generation_layouts import A as A13, CH as CH13, EF as EF13, N as N13
    st = SO.ScaffoldState(int(z["batch"]), N13, A13, CH13, EF13, int(z["n_imp_H"]), int(z["n_chirality"]),
                          z["scaffold_nodes"], z["scaffold_edges"])
    for rnd, (a, lik) in enumerate(zip(z["actions"], z["likelihoods"])):
        SO.generation_round(st, rnd, a, lik)
    return st


def assert_oracle_matches(z, st):
    from tests.test_generation_layouts import assert_matches_trace
    assert st.n_generated == int(z["n_generated"])
    assert_matches_trace(z, st.generated_nodes, st.generated_edges, st.generated_n_nodes, st.generated_likelihoods,
                         st.properly_terminated, st.nodes, st.edges, st.n_nodes, st.likelihoods)
    assert (st.generated_scaffolds == z["generated_scaffolds"]).all()
    assert (st.slot_ids == z["final_slot_ids"]).all() and st.started == int(z["started"])


def test_scaffold_oracle_replays_the_reference_traces_bit_exactly():
    for name in TRACES:
        z = scaffold_trace(name)
        assert int(z["rounds"]) == z["actions"].shape[0] and int(z["n_generated"]) >= int(z["batch"])
        st = replay_oracle(z)
        assert_oracle_matches(z, st)
        if bool(z["attachment"]):               # the recorded draws never take an action the rule forbids
            again = SO.ScaffoldState(int(z["batch"]), st.N, st.A, st.CH, st.Ef, st.H, st.C, z["scaffold_nodes"],
                                     z["scaffold_edges"])
            for rnd, (a, lik) in enumerate(zip(z["actions"], z["likelihoods"])):
                assert not any(SO.forbidden(again, b, z["protect"])[a[b]] for b in range(1, again.B)), rnd
                SO.generation_round(again, rnd, a, lik)


def _maker():
    import importlib.util
    import os
    from tests.conftest import GOLDEN
    spec = importlib.util.spec_from_file_location("_make_scaffold_traces",
                                                  os.path.join(GOLDEN, "make_generation_scaffold_traces.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_live_reference_sweep_matches_the_scaffold_oracle(monkeypatch):
    """the unmodified reference generator with the fixture maker's wrappers, over a few seeds, layouts and batch
    sizes: the oracle replays each run bit for bit"""
    from tests.test_generation_layouts import _reference_generator_module
    maker = _maker()
    GG = _reference_generator_module(monkeypatch, maker.layout_constants(4, 3))
    for seed, (h, c, attach), batch in ((0, (0, 0, True), 24), (1, (4, 3, True), 17), (2, (0, 0, False), 40),
                                        (3, (4, 0, True), 31)):
        z = maker.record(GG, "sweep", h, c, attach, batch, seed)
        assert_oracle_matches(z, replay_oracle(z))
