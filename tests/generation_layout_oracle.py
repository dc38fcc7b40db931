"""
CPU oracle for one generation round in any of the reference's four action layouts  --  TEST INFRASTRUCTURE.

`oracle/generation_oracle.py` restates the reference generator's round for the gdb13 layout (node features = atom
type + formal charge).  This module restates the same round (reference GraphGenerator.py:118-157, 236-305, 556-657;
RL twin GraphGeneratorRL.py:283-320, 618-629, 665-711) with the two optional node-feature segments of
`parameters/constants.py:23-95`: implicit-H counts (H > 0) and chirality (C > 0), 0 = absent.  The add segment of the
APD is laid out as f_add[bond_to, atom, charge, (imp_h,) (chirality,) bond_type].  With H = C = 0 it is the gdb13
oracle, which the tests check on the reference traces of both.

The reference's quirks, kept here:
  * element 5 of the reference's add tuple (`f_add_idc[5]`) is bond_from only when H = C = 0.  It is bond_type when
    one segment is present and chirality when both are.  Its "max nodes" rule (element 5 >= max_n_nodes -> invalid,
    :618) and its reset to 0 (:568, for such adds and every add into an empty graph) act on that element, so with both
    segments the first atom of every molecule is stored with chirality index 0;
  * deliberate deviation: the reference has no result for an add into a graph that already holds max_n_nodes atoms
    when a segment is present (it indexes nodes[b, N] and raises IndexError).  Here the slot terminates as invalid,
    with bond_from = 0, in every layout -- the reference's outcome for the gdb13 layout.

Pinned by tests/golden/generation_layout_traces.npz (made by tests/golden/make_generation_layout_traces.py from the
unmodified reference); the CUDA round kernels are checked against it on random action streams.
"""
import numpy as np

from oracle import generation_oracle as G


class LayoutState(G.GenerationState):
    """`GenerationState` with F = A + CH + H + C node features"""

    def __init__(self, batch, N, A, CH, Ef, H=0, C=0, rl=False):
        super().__init__(batch, N, A, CH, Ef, rl=rl)
        self.H, self.C, self.F = H, C, A + CH + H + C
        self.nodes = np.zeros((batch, N, self.F), np.float32)
        self.nodes[0] = 1                       # the dummy graph covers all F features (:418-423)
        self.generated_nodes = np.zeros((2 * batch, N, self.F), np.float32)


def add_dims(state):
    """the shape of f_add: [N, A, CH, (H,) (C,) Ef]"""
    return (state.N, state.A, state.CH) + ((state.H,) if state.H else ()) + ((state.C,) if state.C else ()) + (state.Ef,)


def decode(state, b, a):
    """flat APD index -> (kind, bond_to, bond_from, atom, charge, imp_h, chirality, bond_type, invalid)
    kind: 0 add, 1 connect, 2 terminate"""
    N, H, C, Ef = state.N, state.H, state.C, state.Ef
    n = int(state.n_nodes[b])
    dims = add_dims(state)
    len_add, len_conn = int(np.prod(dims)), N * Ef
    if a < len_add:
        idx = [int(i) for i in np.unravel_index(a, dims)]
        bt, at, ch = idx[0], idx[1], idx[2]
        ih = idx[3] if H else 0
        cy = idx[-2] if C else 0
        ty = idx[-1]
        bf = n                                                # :557
        empty = n == 0
        invalid = ((not empty) and bt >= n) or (empty and bt != 0)      # :602-615
        # the reference's add tuple is (batch, bond_to, atom, charge, [imp_h], [chirality], bond_type, bond_from)
        tup = [b, bt, at, ch] + ([ih] if H else []) + ([cy] if C else []) + [ty, bf]
        madd = tup[5] >= N                                    # :618
        invalid = invalid or madd
        if madd or empty:                                     # :568 `f_add_idc[5][max_node_idc] = 0`
            tup[5] = 0
        bt, at, ch = tup[1:4]
        ih = tup[4] if H else 0
        cy = tup[-3] if C else 0
        ty, bf = tup[-2], tup[-1]
        if n >= N:                                            # full graph: invalid in every layout (deviation)
            invalid, bf = True, 0
        return 0, bt, bf, at, ch, ih, cy, ty, bool(invalid)
    if a < len_add + len_conn:                                # f_conn[bond_to, bond_type]
        bt, ty = np.unravel_index(a - len_add, (N, Ef))
        bf = n - 1                                            # :561
        bfw = bf + N if bf < 0 else bf                        # Python negative indexing of the reference tensors
        invalid = bt >= n or n == 0 or bt == bf or state.edges[b, bt, bfw].sum() == 1   # :621-634
        return 1, int(bt), int(bfw), 0, 0, 0, 0, int(ty), bool(invalid)
    return 2, 0, 0, 0, 0, 0, 0, 0, False


def generation_round(state, rnd, actions, likelihoods, prior_likelihoods=None):
    """one pass of the `while` body of build_graphs (:118-157; RL: GraphGeneratorRL.py:127-168); returns the number
    of graphs written this round"""
    B, A, CH, H = state.B, state.A, state.CH, state.H
    rl = prior_likelihoods is not None
    assert rl == state.rl
    rec = [decode(state, b, int(actions[b])) for b in range(B)]
    term = [b for b in range(B) if rec[b][0] == 2]
    invalid = [b for b in range(B) if rec[b][8]]
    k = state.n_generated
    cap = state.properly_terminated.shape[0]
    state.properly_terminated[k:min(cap, k + len(term))] = 1                        # :127 (counts slot 0 too)
    order = [b for b in term if b != 0] + [b for b in invalid if b != 0]          # :130-133
    for i, b in enumerate(order):                                                 # copy_terminated_graphs
        state.likelihoods[b, rnd] = likelihoods[b]
        if rl:
            state.prior_likelihoods[b, rnd] = prior_likelihoods[b]
        p = k + i
        if p < cap:
            state.generated_nodes[p] = state.nodes[b]
            state.generated_edges[p] = state.edges[b]
            state.generated_n_nodes[p] = state.n_nodes[b]
            state.generated_likelihoods[p] = state.likelihoods[b]
            if rl:
                state.generated_prior_likelihoods[p] = state.prior_likelihoods[b]
    state.n_generated = k + len(order)
    gone = set(order)
    for b in range(B):                                                            # apply_actions on every slot
        kind, bt, bf, at, ch, ih, cy, ty, _ = rec[b]
        if b in gone:
            continue                                                              # reset below anyway
        if kind == 0:                                                             # _add_nodes :257-306
            state.nodes[b, bf, at] = 1
            state.nodes[b, bf, A + ch] = 1
            if state.H:
                state.nodes[b, bf, A + CH + ih] = 1
            if state.C:
                state.nodes[b, bf, A + CH + H + cy] = 1
            if state.n_nodes[b] != 0:
                state.edges[b, bt, bf, ty] = 1
                state.edges[b, bf, bt, ty] = 1
            state.n_nodes[b] += 1
        elif kind == 1:
            state.edges[b, bf, bt, ty] = 1
            state.edges[b, bt, bf, ty] = 1
        if kind in (0, 1):
            state.likelihoods[b, rnd] = likelihoods[b]
            if rl:
                state.prior_likelihoods[b, rnd] = prior_likelihoods[b]
    for b in order:                                                               # reset_graphs
        state.nodes[b] = 0
        state.edges[b] = 0
        state.n_nodes[b] = 0
        state.likelihoods[b] = 0
        if rl:
            state.prior_likelihoods[b] = 0
    state.nodes[0] = 1                                                            # dummy graph re-stamped (:462-465)
    state.edges[0, 0, 0, 0] = 1
    state.n_nodes[0] = 1
    return len(order)
