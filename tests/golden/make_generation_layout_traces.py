"""
Records golden traces of the reference's batched graph generator (`GraphGenerator.build_graphs`, reference
GraphGenerator.py:99-161) in the three action layouts beyond gdb13's (parameters/constants.py:23-95):

    L1  implicit H   (ignore_H=False, use_explicit_H=False)        node features A + CH + H
    L2  chirality    (use_chirality=True, ignore_H=True)           node features A + CH + C
    L3  both         (use_chirality=True, ignore_H=False)          node features A + CH + H + C

Run in the build container after __graft_entry__.build():

    python tests/golden/make_generation_layout_traces.py

The unmodified reference `GraphGenerator` is imported with the stubs of make_generation_trace.py, and its
`Multinomial.sample` / `get_actions` are wrapped the same way to record every round's draws and stored likelihoods.
No checkpoint exists for these dims, so the model is a seeded scripted policy (`ScriptedPolicy`) that computes logits
from (nodes, edges): most mass on valid-looking adds, on connects and on terminate (growing with the atom count), a
uniform floor so that every validity rule fires, and zero mass on adds into a full graph -- the reference has no
result for those outside gdb13's layout (it raises IndexError).  The script checks that each trace covers what the
tests rely on and prints the counts.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_generation_trace import generator_constants, install_stubs   # noqa: E402
from tests import refimpl                                              # noqa: E402

N, A, CH, H, C, EF = 13, 5, 3, 4, 3, 3
LAYOUTS = {"L1": (H, 0), "L2": (0, C), "L3": (H, C)}


def layout_constants(h, c):
    F = A + CH + h + c
    f_add = [N, A, CH] + ([h] if h else []) + ([c] if c else []) + [EF]
    return generator_constants(dim_nodes=[N, F], dim_f_add=f_add, n_imp_H=h, n_chirality=c, ignore_H=not h,
                               use_explicit_H=False, use_chirality=bool(c), n_node_features=F,
                               len_f_add_per_node=int(np.prod(f_add[1:])))


class ScriptedPolicy(torch.nn.Module):
    """logits [B, apd] = log of an explicit action distribution of the atom count n (non-zero node rows; the dummy
    slot 0 reads as full).  Per graph, masses go to: valid-looking adds (bond_to < n, or 0 into an empty graph),
    connects among existing atoms, self loops, terminate (growing with n), and a floor spread uniformly over all adds
    and over all connects; an add into a full graph gets exactly zero.  A fixed seeded factor exp(0.5 z) per action
    keeps the draws from being uniform inside a segment."""

    def __init__(self, h, c, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.add_dims = [N, A, CH] + ([h] if h else []) + ([c] if c else []) + [EF]
        self.per_node = int(np.prod(self.add_dims[1:]))
        self.noise = torch.exp(0.5 * torch.randn(N * self.per_node + N * EF + 1, generator=g))

    def forward(self, nodes, edges):
        B = nodes.shape[0]
        n = (nodes.sum(-1) > 0).sum(-1)[:, None].float()                         # [B, 1]
        pos = torch.arange(N, dtype=torch.float32)[None]
        full, empty = n >= N, n == 0
        z = torch.zeros_like(n)
        m_term = torch.where(full, z + 0.9, torch.where(empty, z + 0.005, 0.002 + 0.001 * n))
        m_conn = torch.where(n >= 2, torch.where(full, z + 0.08, z + 0.025), z)
        m_loop = torch.where(empty | full, z, z + 0.006)
        m_floor_conn = torch.where(empty, z + 0.04, torch.where(full, z + 0.02, z + 0.006))
        m_floor_add = torch.where(empty, z + 0.04, torch.where(full, z, z + 0.006))
        m_add = 1 - m_term - m_conn - m_loop - m_floor_conn - m_floor_add
        to_ok = ((pos < n) | (empty & (pos == 0))).float()                          # [B, N]
        add = m_add * to_ok / to_ok.sum(1, keepdim=True) + m_floor_add / N
        add = (add * ~full / self.per_node)[:, :, None].expand(B, N, self.per_node).reshape(B, -1)
        among = (pos < n - 1).float()
        conn = m_conn * among / among.sum(1, keepdim=True).clamp(min=1) + m_loop * (pos == n - 1) + m_floor_conn / N
        conn = (conn / EF)[:, :, None].expand(B, N, EF).reshape(B, -1)
        p = torch.cat([add, conn, m_term], dim=1) * self.noise
        return torch.log(p)                                  # log 0 = -inf: exactly zero probability after softmax


def classify(h, c, n_nodes, edges, actions):
    """per (round, slot != 0): which validity rule an action hits, and whether a first-atom add sampled a non-zero
    chirality (recomputed from the pre-action state the reference held)"""
    dims = [N, A, CH] + ([h] if h else []) + ([c] if c else []) + [EF]
    len_add = int(np.prod(dims))
    hits = dict(add_bond_to_missing=0, first_add_off_slot0=0, conn_to_missing=0, conn_in_empty=0, conn_self_loop=0,
                conn_double=0, add_into_full=0, terminate=0, quirk1=0)
    for r in range(actions.shape[0]):
        for b in range(1, actions.shape[1]):
            a, n = int(actions[r, b]), int(n_nodes[r][b])
            if a < len_add:
                idx = np.unravel_index(a, dims)
                bt = int(idx[0])
                hits["add_into_full"] += n >= N
                hits["add_bond_to_missing"] += n > 0 and bt >= n
                hits["first_add_off_slot0"] += n == 0 and bt != 0
                hits["quirk1"] += bool(h and c and n == 0 and bt == 0 and int(idx[-2]) != 0)
            elif a < len_add + N * EF:
                bt = (a - len_add) // EF
                hits["conn_to_missing"] += bt >= n
                hits["conn_in_empty"] += n == 0
                hits["conn_self_loop"] += bt == n - 1
                hits["conn_double"] += 0 <= n - 1 and bt < n and edges[r][b, bt, n - 1].sum() == 1
            else:
                hits["terminate"] += 1
    return hits


def record(GG, name, h, c, batch, seed):
    C = layout_constants(h, c)
    GG.constants = C                      # the module bound `from parameters.constants import constants` at import
    torch.manual_seed(seed)
    net = ScriptedPolicy(h, c, seed)
    draws, liks, n_pre, e_pre = [], [], [], []
    orig_sample = torch.distributions.Multinomial.sample
    orig_get_actions = GG.GraphGenerator.get_actions

    def recording_sample(self, sample_shape=torch.Size()):
        one_hot = orig_sample(self, sample_shape)
        draws.append(one_hot.argmax(1).to(torch.int32).numpy().copy())
        return one_hot

    def recording_get_actions(self, apds):
        n_pre.append(self.n_nodes.numpy().copy())
        e_pre.append(self.edges.numpy().astype(np.int8))
        res = orig_get_actions(self, apds)
        liks.append(res[4].numpy().copy())
        return res

    GG.GraphGenerator.get_actions = recording_get_actions
    torch.distributions.Multinomial.sample = recording_sample
    try:
        with torch.no_grad():
            gen = GG.GraphGenerator(model=net, batch_size=batch)
            n_generated = gen.build_graphs()
    finally:
        torch.distributions.Multinomial.sample = orig_sample
        GG.GraphGenerator.get_actions = orig_get_actions
    actions = np.stack(draws)
    hits = classify(h, c, n_pre, e_pre, actions)
    nn = gen.generated_n_nodes[:n_generated].numpy()
    gnodes = gen.generated_nodes.numpy()
    print(f"{name}: rounds {len(draws)}, actions {actions.size}, generated {n_generated}, properly terminated "
          f"{int(gen.properly_terminated[:n_generated].sum())}, mean atoms {nn.mean():.2f}, "
          f"molecules with {N} atoms {int((nn == N).sum())}, rule hits {hits}")
    assert int(nn.max()) == N, (name, "no molecule reached max_n_nodes")
    assert hits["add_into_full"] == 0
    for k in ("add_bond_to_missing", "first_add_off_slot0", "conn_to_missing", "conn_in_empty", "conn_self_loop",
              "conn_double", "terminate"):
        assert hits[k] > 0, (name, k, hits)
    if h and c:
        assert hits["quirk1"] > 0
        first = gnodes[:n_generated][nn > 0, 0, A + CH + h:]
        assert (first[:, 0] == 1).all() and (first[:, 1:] == 0).all()     # every first atom stored with chirality 0
    out = {f"{name}/{k}": v for k, v in dict(
        batch=np.int32(batch), n_generated=np.int32(n_generated), rounds=np.int32(len(draws)), n_imp_H=np.int32(h),
        n_chirality=np.int32(c), actions=actions.astype(np.int16), likelihoods=np.stack(liks),
        generated_nodes=gnodes.astype(np.int8), generated_edges=gen.generated_edges.numpy().astype(np.int8),
        generated_n_nodes=gen.generated_n_nodes.numpy(), generated_likelihoods=gen.generated_likelihoods.numpy(),
        properly_terminated=gen.properly_terminated.numpy(), final_nodes=gen.nodes.numpy().astype(np.int8),
        final_edges=gen.edges.numpy().astype(np.int8), final_n_nodes=gen.n_nodes.numpy(),
        final_likelihoods=gen.likelihoods.numpy()).items()}
    return out


def main(batch=80, seed=11):
    assert refimpl.available()
    install_stubs(layout_constants(H, C))
    refimpl.load()
    import GraphGenerator as GG     # the unmodified reference module
    out = {}
    for i, (name, (h, c)) in enumerate(LAYOUTS.items()):
        out.update(record(GG, name, h, c, batch, seed + i))
    np.savez_compressed(os.path.join(HERE, "generation_layout_traces.npz"), **out)


if __name__ == "__main__":
    main()
