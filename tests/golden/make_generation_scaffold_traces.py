"""
Records golden traces of the reference's batched graph generator (`GraphGenerator.build_graphs`, reference
GraphGenerator.py:99-161) decorating scaffolds, in the gdb13 layout (L0) and with both optional node-feature segments
(L3), each without and with attachment points:

    python tests/golden/make_generation_scaffold_traces.py

The unmodified reference `GraphGenerator` is imported with the stubs of make_generation_trace.py, and the seeded
scripted policy of make_generation_layout_traces.py gives the logits.  Three methods are wrapped, the module itself is
not changed:
  * `initialize_graph_batch`: after the reference's start state, slot b >= 1 is loaded with scaffold (b - 1) mod S
    (nodes, edges, n_nodes = k_s), and `started` = B - 1;
  * `copy_terminated_graphs`: records the scaffold of each graph copied out, at its output row;
  * `reset_graphs`: after the reference's reset, the reset slots, in ascending slot order, are loaded with scaffolds
    (started + j) mod S, and `started` grows by their number.
With attachment points the policy's logits are masked by the attachment rule (an add or a connect whose bond_to is a
protected scaffold atom, and every connect while the newest atom is still a scaffold atom, get -inf) before the
reference's softmax, so the reference's Multinomial draws from the renormalised distribution and stores its
probabilities.  `record(GG, ...)` is shared with the host test's live-reference sweep.

Scaffolds: decoding-route states of gdb13_1K (tests/golden/gdb13_train_head256.h5) with 1, 2, 4, 6, 9 and 12 atoms
(12 = max_n_nodes - 1), widened to L3 with implicit-H and chirality index 0 on every atom; attachment points: the
last atom of each scaffold and a seeded third of the others.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_generation_layout_traces import A, CH, EF, N, ScriptedPolicy, layout_constants   # noqa: E402
from make_generation_trace import install_stubs                                            # noqa: E402
from tests import refimpl                                                                  # noqa: E402

TRACES = {"L0": (0, 0, False), "L0_attach": (0, 0, True), "L3": (4, 3, False), "L3_attach": (4, 3, True)}
SIZES = (1, 2, 4, 6, 9, 12)


def scaffolds(h, c):
    """int8 nodes [S, N, A + CH + h + c], edges [S, N, N, EF] and the bool protected-atom mask [S, N] of the seeded
    attachment points"""
    from graphinvent_b200 import data
    nodes, edges, _ = data.read_hdf5_raw(os.path.join(HERE, "gdb13_train_head256.h5"), N, A + CH, EF, 625)
    k_all = (nodes != 0).any(-1).sum(-1)
    rows = [int(np.flatnonzero(k_all == s)[0]) for s in SIZES]
    nodes, edges = nodes[rows].copy(), edges[rows].copy()
    atoms = (nodes != 0).any(-1, keepdims=True)
    extra = [np.concatenate([atoms, np.zeros(atoms.shape[:-1] + (w - 1,), bool)], -1) for w in (h, c) if w]
    nodes = np.concatenate([nodes] + [e.astype(np.int8) for e in extra], -1)
    rng = np.random.default_rng(0)
    k = np.array(SIZES)
    protect = np.arange(N)[None] < k[:, None]
    for s, n in enumerate(k):
        protect[s, n - 1] = False
        protect[s, np.flatnonzero(rng.random(n) < 0.3)] = False
    return nodes, edges, protect


def forbidden(n_nodes, slot_ids, k, protect, per_node):
    """bool [B, apd] of the attachment rule (slot 0 and slots without a scaffold: nothing)"""
    B = n_nodes.shape[0]
    len_add = N * per_node
    m = torch.zeros(B, len_add + N * EF + 1, dtype=torch.bool)
    for b in range(1, B):
        s = int(slot_ids[b])
        if s < 0:
            continue
        for i in np.flatnonzero(protect[s, :k[s]]):
            m[b, i * per_node:(i + 1) * per_node] = True
            m[b, len_add + i * EF:len_add + (i + 1) * EF] = True
        if int(n_nodes[b]) - 1 < k[s]:
            m[b, len_add:len_add + N * EF] = True
    return m


class MaskedPolicy(torch.nn.Module):
    """the scripted policy's logits with the attachment rule applied from the generator's live state"""

    def __init__(self, net, k, protect):
        super().__init__()
        self.net, self.k, self.protect, self.gen = net, k, protect, None

    def forward(self, nodes, edges):
        out = self.net(nodes, edges)
        if self.protect is None:
            return out
        m = forbidden(self.gen.n_nodes, self.gen.slot_ids, self.k, self.protect, self.net.per_node)
        return out.masked_fill(m, -float("inf"))


def record(GG, name, h, c, attach, batch, seed, sc=None):
    """one trace of the reference generator decorating scaffolds `sc` = (nodes, edges, protect) (default: the
    gdb13 sets above); returns the dict saved under `name/`"""
    C = layout_constants(h, c)
    GG.constants = C
    nodes_s, edges_s, protect = sc if sc is not None else scaffolds(h, c)
    if not attach:
        protect = None
    S = nodes_s.shape[0]
    k = (nodes_s != 0).any(-1).sum(-1)
    torch.manual_seed(seed)
    net = MaskedPolicy(ScriptedPolicy(h, c, seed), k, protect)
    draws, liks, masked = [], [], []
    Gen = GG.GraphGenerator
    orig = {f: getattr(Gen, f) for f in ("initialize_graph_batch", "copy_terminated_graphs", "reset_graphs",
                                           "get_actions")}
    orig_sample = torch.distributions.Multinomial.sample

    def load(self, b, s):
        self.nodes[b] = torch.from_numpy(nodes_s[s]).float()
        self.edges[b] = torch.from_numpy(edges_s[s]).float()
        self.n_nodes[b] = int(k[s])
        self.slot_ids[b] = s

    def initialize_graph_batch(self):
        orig["initialize_graph_batch"](self)
        self.slot_ids = np.full(self.batch_size, -1, np.int64)
        self.generated_scaffolds = np.full(2 * self.batch_size, -1, np.int32)
        for b in range(1, self.batch_size):
            load(self, b, (b - 1) % S)
        self.started = self.batch_size - 1

    def copy_terminated_graphs(self, idc, n_generated, generation_round, likelihoods):
        for i, b in enumerate(idc.tolist()):
            if n_generated + i < self.generated_scaffolds.shape[0]:
                self.generated_scaffolds[n_generated + i] = self.slot_ids[b]
        return orig["copy_terminated_graphs"](self, idc, n_generated, generation_round, likelihoods)

    def reset_graphs(self, idc):
        orig["reset_graphs"](self, idc)
        order = sorted(idc.tolist())
        for j, b in enumerate(order):
            load(self, b, (self.started + j) % S)
        self.started += len(order)

    def get_actions(self, apds):
        if protect is not None:
            masked.append(forbidden(self.n_nodes, self.slot_ids, k, protect, net.net.per_node).numpy())
        res = orig["get_actions"](self, apds)
        liks.append(res[4].numpy().copy())
        return res

    def recording_sample(self, sample_shape=torch.Size()):
        one_hot = orig_sample(self, sample_shape)
        draws.append(one_hot.argmax(1).to(torch.int32).numpy().copy())
        return one_hot

    for f, fn in (("initialize_graph_batch", initialize_graph_batch), ("copy_terminated_graphs", copy_terminated_graphs),
                  ("reset_graphs", reset_graphs), ("get_actions", get_actions)):
        setattr(Gen, f, fn)
    torch.distributions.Multinomial.sample = recording_sample
    try:
        with torch.no_grad():
            gen = Gen(model=net, batch_size=batch)
            net.gen = gen
            n_generated = gen.build_graphs()
    finally:
        torch.distributions.Multinomial.sample = orig_sample
        for f, fn in orig.items():
            setattr(Gen, f, fn)
    actions = np.stack(draws)
    if protect is not None:
        m = np.stack(masked)
        hit = m[np.arange(len(draws))[:, None], np.arange(batch)[None, 1:], actions[:, 1:]]
        assert not hit.any(), (name, "a forbidden action was drawn")
        assert m[:, 1:].any(), (name, "the mask never applied")
    out = dict(batch=np.int32(batch), n_generated=np.int32(n_generated), rounds=np.int32(len(draws)),
               n_imp_H=np.int32(h), n_chirality=np.int32(c), scaffold_nodes=nodes_s.astype(np.int8),
               scaffold_edges=edges_s.astype(np.int8),
               protect=(protect if protect is not None else np.zeros((S, N), bool)), attachment=np.bool_(attach),
               actions=actions.astype(np.int16), likelihoods=np.stack(liks),
               generated_nodes=gen.generated_nodes.numpy().astype(np.int8),
               generated_edges=gen.generated_edges.numpy().astype(np.int8),
               generated_n_nodes=gen.generated_n_nodes.numpy(), generated_likelihoods=gen.generated_likelihoods.numpy(),
               properly_terminated=gen.properly_terminated.numpy(), generated_scaffolds=gen.generated_scaffolds,
               final_nodes=gen.nodes.numpy().astype(np.int8), final_edges=gen.edges.numpy().astype(np.int8),
               final_n_nodes=gen.n_nodes.numpy(), final_likelihoods=gen.likelihoods.numpy(),
               final_slot_ids=gen.slot_ids.astype(np.int32), started=np.int32(gen.started))
    return out


def main(batch=80, seed=23):
    assert refimpl.available()
    install_stubs(layout_constants(4, 3))
    refimpl.load()
    import GraphGenerator as GG     # the unmodified reference module
    out = {}
    for i, (name, (h, c, attach)) in enumerate(TRACES.items()):
        z = record(GG, name, h, c, attach, batch, seed + i)
        n_gen = int(z["n_generated"])
        ids = z["generated_scaffolds"][:n_gen]
        print(f"{name}: rounds {int(z['rounds'])}, generated {n_gen}, scaffolds used {sorted(set(ids.tolist()))}, "
              f"restarts {int(z['started']) - batch + 1}, mean atoms {z['generated_n_nodes'][:n_gen].mean():.2f}")
        assert len(set(ids.tolist())) == len(SIZES), (name, "not every scaffold finished a molecule")
        out.update({f"{name}/{k}": v for k, v in z.items()})
    np.savez_compressed(os.path.join(HERE, "generation_scaffold_traces.npz"), **out)


if __name__ == "__main__":
    main()
