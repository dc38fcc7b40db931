"""
Records the reference's verdict on every action of many generator states, for the action mask
(graphinvent_b200/csrc/action_mask.cuh, tests/action_mask_reference.py).  Run in the build container:

    python tests/golden/make_action_mask_fixture.py

The unmodified reference `GraphGenerator.get_invalid_actions` (GraphGenerator.py:573-657) is imported under the
stubs of make_generation_trace.py.  For each state (atom count n, edges [N, N, Ef]) it is called once on a batch that
holds the state once per add / connect index of the action space, each row with its own action, in the tuples
`get_actions` builds (GraphGenerator.py:559-566); the invalid rows it returns are the verdicts.  Cases cover the four
action layouts, N small enough for the element-5 rule to fire on bond types / chiralities (N = 1, 2), Ef 1-4, empty,
single-atom and full graphs, and states with bonds (including states whose bond rows hold several types, as the
dummy slot accumulates them).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from tests import refimpl                                               # noqa: E402
from make_generation_trace import generator_constants, install_stubs    # noqa: E402

# (N, A, CH, H, C, Ef)
CASES = [
    (13, 5, 3, 0, 0, 3), (13, 2, 2, 4, 0, 3), (13, 2, 2, 0, 3, 3), (13, 2, 1, 4, 3, 3),
    (1, 2, 2, 0, 0, 3), (1, 2, 1, 2, 0, 3), (2, 2, 1, 0, 3, 4), (2, 1, 2, 3, 3, 2), (2, 1, 1, 2, 0, 4),
    (6, 3, 3, 0, 0, 1), (6, 2, 3, 2, 0, 2), (6, 2, 2, 0, 2, 4), (6, 1, 2, 3, 2, 1), (9, 2, 2, 0, 0, 4),
]


def random_state(rng, N, Ef, n, p_bond=0.5, multi=False):
    e = np.zeros((N, N, Ef), np.int8)
    for i in range(1, n):
        nb = [int(rng.integers(0, i))]                       # every atom bonded to an earlier one
        nb += [j for j in range(i) if j != nb[0] and rng.random() < p_bond * 0.3]
        for j in nb:
            t = int(rng.integers(0, Ef))
            e[i, j, t] = e[j, i, t] = 1
            if multi and Ef > 1 and rng.random() < 0.3:      # a second type on the same pair: sum 2
                t2 = (t + 1) % Ef
                e[i, j, t2] = e[j, i, t2] = 1
    return e


def states(rng, N, Ef):
    out = [(0, np.zeros((N, N, Ef), np.int8)), (N, random_state(rng, N, Ef, N))]
    if N > 1:
        out.append((1, np.zeros((N, N, Ef), np.int8)))
    for _ in range(4):
        n = int(rng.integers(0, N + 1))
        out.append((n, random_state(rng, N, Ef, n, multi=bool(rng.random() < 0.3))))
    return out


def verdict(GG, N, A, CH, H, C, Ef, n, edges):
    dim_f_add = [N, A, CH] + ([H] if H else []) + ([C] if C else []) + [Ef]
    GG.constants = generator_constants(dim_nodes=[N, A + CH + H + C], dim_edges=[N, N, Ef], dim_f_add=dim_f_add,
                                       dim_f_conn=[N, Ef], max_n_nodes=N)
    len_add = int(np.prod(dim_f_add))
    n_act = len_add + N * Ef
    gen = GG.GraphGenerator.__new__(GG.GraphGenerator)
    gen.n_nodes = torch.full((n_act,), n, dtype=torch.int64)
    gen.edges = torch.from_numpy(np.broadcast_to(edges, (n_act, N, N, Ef)).astype(np.float32).copy())
    rows = torch.arange(n_act)
    add = torch.zeros((n_act, *dim_f_add))
    add.view(n_act, -1)[rows[:len_add], rows[:len_add]] = 1
    conn = torch.zeros((n_act, N, Ef))
    conn.view(n_act, -1)[rows[len_add:], rows[len_add:] - len_add] = 1
    f_add_idc = torch.nonzero(add, as_tuple=True)               # as get_actions builds them (:559-566)
    f_add_idc = (*f_add_idc, gen.n_nodes[f_add_idc[0]])
    f_conn_idc = torch.nonzero(conn, as_tuple=True)
    f_conn_idc = (*f_conn_idc, gen.n_nodes[f_conn_idc[0]] - 1)
    invalid, _ = GG.GraphGenerator.get_invalid_actions(gen, f_add_idc, f_conn_idc)
    v = np.zeros(n_act + 1, bool)
    v[invalid.numpy()] = True
    return v


def main(seed=5):
    assert refimpl.available()
    install_stubs(generator_constants())
    refimpl.load()
    import GraphGenerator as GG     # the unmodified reference module
    rng = np.random.default_rng(seed)
    out = {"cases": np.array(CASES, np.int32)}
    for k, (N, A, CH, H, C, Ef) in enumerate(CASES):
        ns, es, vs = [], [], []
        for n, e in states(rng, N, Ef):
            ns.append(n)
            es.append(e)
            vs.append(verdict(GG, N, A, CH, H, C, Ef, n, e))
        out[f"n_{k}"], out[f"edges_{k}"], out[f"invalid_{k}"] = np.array(ns, np.int32), np.stack(es), np.stack(vs)
    np.savez_compressed(os.path.join(HERE, "action_mask_invalid.npz"), **out)
    print(f"{len(CASES)} layouts, {sum(out[f'n_{k}'].size for k in range(len(CASES)))} states, "
          f"{sum(out[f'invalid_{k}'].size for k in range(len(CASES)))} verdicts")


if __name__ == "__main__":
    main()
