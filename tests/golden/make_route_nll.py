"""Writes tests/golden/route_nll_gdb13.npz: the decoding-route likelihoods of gdb13 molecules under the reference's
pretrained GGNN, from the live reference.

    python tests/golden/make_route_nll.py

Needs oracle/_ref as __graft_entry__.build() installs it.  The molecules are the first MOLECULES full graphs of
gdb13_1K/train in tests/golden/preprocess_gdb13.npz.  Each one's states come from the reference's own
`PreprocessingGraph.get_decoding_route_state(k)`, k = 0 .. n_edges + 1 (stub rdkit, the graph built from the stacks
as tests/test_preprocess_host.py builds it), its action from the one-hot APD that call returns; the probabilities are
`Softmax(dim=1)(model(nodes, edges))[action]` of the reference GGNN with the pretrained checkpoint, in float32.  Stored
in build order (k = n_edges + 1 first): nodes / edges (the molecules, int8), offsets, actions, likelihoods."""
import hashlib
import os
import sys
from collections import namedtuple

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import mpnn_oracle as O  # noqa: E402
from tests import molecules_reference as MR  # noqa: E402
from tests import preprocess_reference as P  # noqa: E402
from tests import refimpl  # noqa: E402
from tests.conftest import pretrained_path  # noqa: E402

MOLECULES = 96
N, EF, SEGS = 13, 3, [5, 3]


def route_constants(B=1000):
    fields = dict(max_n_nodes=N, n_edge_features=EF, n_atom_types=5, n_formal_charge=3, n_imp_H=0, n_chirality=0,
                  use_explicit_H=False, ignore_H=True, use_chirality=False, batch_size=B, dim_f_add=[N] + SEGS + [EF],
                  dim_f_conn=[N, EF], n_node_features=8, atom_types=["X"] * 5, formal_charge=[0] * 3, imp_H=[],
                  chirality=[], device="cpu")
    return namedtuple("constants", sorted(fields))(**fields)


def live_states(nodes, edges):
    ref = MR.load_reference(route_constants())
    G = ref.MolecularGraph.PreprocessingGraph
    Xs, Es, acts, offsets = [], [], [], [0]
    for m in range(nodes.shape[0]):
        g = G.__new__(G)
        g.constants = route_constants()
        g.node_features, g.edge_features = nodes[m].astype(np.float64), edges[m].astype(np.float64)
        g.n_nodes = P.n_atoms(nodes[m])
        states = []
        for k in range(g.get_decoding_route_length()):
            (X, E), apd = g.get_decoding_route_state(k)
            flat = np.asarray(apd).ravel()
            assert flat.sum() == 1
            states.append((np.asarray(X).astype(np.int8), np.asarray(E).astype(np.int8), int(np.argmax(flat))))
        for X, E, a in states[::-1]:
            Xs.append(X)
            Es.append(E)
            acts.append(a)
        offsets.append(offsets[-1] + len(states))
    return np.stack(Xs), np.stack(Es), np.array(acts, np.int64), np.array(offsets, np.int64)


def main():
    path = pretrained_path()
    assert refimpl.available() and path, "needs the reference installed by __graft_entry__.build()"
    z = np.load(os.path.join(HERE, "preprocess_gdb13.npz"))
    nodes, edges = z["gdb13_1K_train/nodes"][:MOLECULES], z["gdb13_1K_train/edges"][:MOLECULES]
    X, E, acts, offsets = live_states(nodes, edges)
    net = refimpl.build(O.make_constants("GGNN"))
    net.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    net.eval()
    with torch.no_grad():
        probs = torch.nn.Softmax(dim=1)(net(torch.from_numpy(X).float(), torch.from_numpy(E).float()))
    lik = probs.gather(1, torch.from_numpy(acts).view(-1, 1)).view(-1).numpy()
    sha = hashlib.sha256(open(path, "rb").read()).hexdigest()
    np.savez_compressed(os.path.join(HERE, "route_nll_gdb13.npz"), nodes=nodes, edges=edges, offsets=offsets,
                        actions=acts, likelihoods=lik, sha256=np.array(sha))
    print(f"{MOLECULES} molecules, {X.shape[0]} route states, mean log p {np.log(lik).mean():.4f}")


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
