"""Python restatement of the molecule set (graphinvent_b200.molecules.MoleculeSet, `gib_molset_identify` in
csrc/preprocess.cu), the oracle of its tests.  Written from the rule in include/gib200.h:

  * a molecule's canonical form: its atoms breadth-first from atom 0, each layer in increasing index
    (`murcko_reference.canonical_order` with every atom kept);
  * identity: graph isomorphism (node rows and edge cells preserved), decided by `scaffold_match_reference.search`
    embedding an entry in the molecule between graphs of equal atom and bond counts, after the 1-WL hash
    (`murcko_reference.wl_hash`) matched; two empty graphs are the same molecule;
  * a call processes the batch in order: each valid molecule joins the entry it is isomorphic to, else (add) it opens
    the next entry; `new` = its class was not in the set before the call, `first` = the first molecule of its class in
    the call.  `find` is the same call on a copy of the set, with ids -1 for classes that were not in it.
"""
import copy
import itertools

import numpy as np

from tests import murcko_reference as MR
from tests import scaffold_match_reference as SM


def canonical(nodes, edges):
    """(nodes, edges) of the molecule in canonical order"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    n = SM.n_atoms(nodes)
    keep = np.zeros(nodes.shape[0], bool)
    keep[:n] = True
    return SM.reorder(nodes, edges, MR.canonical_order(edges, keep))


class MoleculeSet:
    """entries (canonical nodes, edges), hashes, atom and bond counts, counts"""

    def __init__(self):
        self.nodes, self.edges, self.hash, self.k, self.bonds, self.counts = [], [], [], [], [], []

    def __len__(self):
        return len(self.nodes)

    def lookup(self, X, E, budget=1 << 20):
        """the entry the canonical molecule (X, E) is, None when none, "budget" when a search runs out"""
        h, k = MR.wl_hash(X, E), SM.n_atoms(X)
        b = MR.n_bonds(E, k)
        for s in range(len(self)):
            if self.hash[s] != h or self.k[s] != k or self.bonds[s] != b:
                continue
            if k == 0:
                return s
            res, _ = SM.search(X, E, self.nodes[s], self.edges[s], None, budget)
            if res == "budget":
                return "budget"
            if res == "found":
                return s
        return None

    def _append(self, X, E):
        k = SM.n_atoms(X)
        self.nodes.append(X)
        self.edges.append(E)
        self.hash.append(MR.wl_hash(X, E))
        self.k.append(k)
        self.bonds.append(MR.n_bonds(E, k))
        self.counts.append(0)
        return len(self) - 1

    def add(self, nodes, edges, valid=None, budget=1 << 20):
        """(ids, new, first) of the batch, inserting it"""
        M = len(nodes)
        before = len(self)
        ids = np.full(M, -1, np.int32)
        new = np.zeros(M, bool)
        first = np.zeros(M, bool)
        seen = set()
        for m in range(M):
            if valid is not None and not valid[m]:
                continue
            X, E = canonical(nodes[m], edges[m])
            s = self.lookup(X, E, budget)
            if s == "budget":
                raise ValueError(f"molecule {m}: budget")
            if s is None:
                s = self._append(X, E)
            self.counts[s] += 1
            ids[m] = s
            new[m] = s >= before
            first[m] = s not in seen
            seen.add(s)
        return ids, new, first

    def find(self, nodes, edges, valid=None, budget=1 << 20):
        """(ids, new, first) of the batch, the set unchanged"""
        before = len(self)
        ids, new, first = copy.deepcopy(self).add(nodes, edges, valid, budget)
        ids[ids >= before] = -1
        return ids, new, first

    def arrays(self, N, F, Ef):
        if not len(self):
            return np.zeros((0, N, F), np.int8), np.zeros((0, N, N, Ef), np.int8), np.zeros(0, np.int64)
        return np.stack(self.nodes), np.stack(self.edges), np.array(self.counts, np.int64)


def brute_isomorphic(n1, e1, n2, e2):
    """the identity rule stated directly: some renumbering of molecule 1's atoms gives molecule 2, byte for byte"""
    n1, e1, n2, e2 = map(np.asarray, (n1, e1, n2, e2))
    k = SM.n_atoms(n1)
    if SM.n_atoms(n2) != k:
        return False
    for perm in itertools.permutations(range(k)):
        X, E = SM.reorder(n1, e1, list(perm))
        if np.array_equal(X, n2) and np.array_equal(E, e2):
            return True
    return False


def write_molecules_uniqueness(keys, valid):
    """util.write_molecules' uniqueness tensor (util.py:549-585) over hashable molecule keys: 1 for an invalid molecule
    or the first occurrence of a key among the valid ones, 0 for a later one"""
    out, seen = [], []
    for key, ok in zip(keys, valid):
        if not ok:
            out.append(1.0)
            continue
        out.append(0.0 if key in seen else 1.0)
        seen.append(key)
    return np.array(out, np.float32)
