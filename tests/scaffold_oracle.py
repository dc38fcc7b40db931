"""
CPU oracle for generation rounds that decorate scaffolds  --  TEST INFRASTRUCTURE.

Extends the layout oracle (tests/generation_layout_oracle.py) with the scaffold semantics of `gib_scaffolds`
(include/gib200.h):
  * start: slot 0 is the dummy graph as before; slot b >= 1 holds scaffold (b - 1) mod S, n_nodes = k_s, a zero
    likelihood row; started = B - 1;
  * reset: the slots that terminate in a round (terminate-sampled and invalid alike), in ascending slot order, restart
    from scaffolds (started + j) mod S, j = 0, 1, ...; started then grows by their number;
  * generated_scaffolds[p]: the scaffold of the molecule copied out to row p (copy-out order unchanged);
  * mask (`forbidden`): with attachment points, an add or a connect whose bond_to is a protected scaffold atom, and
    every connect while bond_from = n_nodes - 1 is still a scaffold atom, is forbidden; terminate never is.  Slot 0 is
    never masked.
"""
import numpy as np

from tests import generation_layout_oracle as L


class ScaffoldState(L.LayoutState):
    """`LayoutState` whose slots grow from the scaffolds nodes [S, N, F] / edges [S, N, N, Ef] (0/1)"""

    def __init__(self, batch, N, A, CH, Ef, H, C, sc_nodes, sc_edges, rl=False):
        super().__init__(batch, N, A, CH, Ef, H, C, rl=rl)
        self.sc_nodes = np.asarray(sc_nodes, np.float32)
        self.sc_edges = np.asarray(sc_edges, np.float32)
        self.S = self.sc_nodes.shape[0]
        self.k = (self.sc_nodes != 0).any(-1).sum(-1)
        self.slot_ids = np.full(batch, -1, np.int64)
        self.started = batch - 1
        self.generated_scaffolds = np.full(2 * batch, -1, np.int32)
        for b in range(1, batch):
            self.load(b, (b - 1) % self.S)

    def load(self, b, s):
        self.nodes[b] = self.sc_nodes[s]
        self.edges[b] = self.sc_edges[s]
        self.n_nodes[b] = self.k[s]
        self.likelihoods[b] = 0
        if self.rl:
            self.prior_likelihoods[b] = 0
        self.slot_ids[b] = s


def generation_round(state, rnd, actions, likelihoods, prior_likelihoods=None):
    """the layout oracle's round, then the scaffold reset and the output's scaffold ids"""
    B = state.B
    rec = [L.decode(state, b, int(actions[b])) for b in range(B)]
    order = [b for b in range(1, B) if rec[b][0] == 2] + [b for b in range(1, B) if rec[b][8]]
    k = state.n_generated
    cap = state.generated_scaffolds.shape[0]
    for i, b in enumerate(order):
        if k + i < cap:
            state.generated_scaffolds[k + i] = state.slot_ids[b]
    n = L.generation_round(state, rnd, actions, likelihoods, prior_likelihoods)
    for j, b in enumerate(sorted(order)):
        state.load(b, (state.started + j) % state.S)
    state.started += len(order)
    return n


def add_len(state):
    return int(np.prod(L.add_dims(state)[1:]))


def forbidden(state, b, protect):
    """bool [apd]: the actions slot b may not take; protect bool [S, N] (True: a scaffold atom that is not an
    attachment point) or None"""
    N, Ef = state.N, state.Ef
    per_node = add_len(state)
    len_add = N * per_node
    m = np.zeros(len_add + N * Ef + 1, bool)
    s = int(state.slot_ids[b])
    if b == 0 or s < 0 or protect is None:
        return m
    k, n = int(state.k[s]), int(state.n_nodes[b])
    for i in range(k):
        if protect[s, i]:
            m[i * per_node:(i + 1) * per_node] = True
            m[len_add + i * Ef:len_add + (i + 1) * Ef] = True
    if n - 1 < k:
        m[len_add:len_add + N * Ef] = True
    return m


def protect_of(k, attachment, N):
    """bool [S, N] protected atoms of scaffolds with k[s] atoms and attachment-point lists `attachment`"""
    p = np.arange(N)[None] < np.asarray(k)[:, None]
    for s, idx in enumerate(attachment):
        p[s, list(idx)] = False
    return p
