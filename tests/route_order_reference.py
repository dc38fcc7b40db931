"""
Python restatement of the reference's decoding-route choice, `PreprocessingGraph.node_remap` (MolecularGraph.py:
435-461): `breadth_first_search` / `depth_first_search` (MolecularGraph.py:328-433) from atom `ranking[0]`, then
`reorder_nodes` (MolecularGraph.py:592-614).  Written from the reference's rules with an explicit model of CPython
3.12's set table (`PySet`), the same algorithm as `reorder_kernel` in csrc/preprocess.cu: the reference's BFS orders
each layer as `set(...)` of the layer's atoms iterates, and that order depends on the table's probing and resizing.
"""
import numpy as np

LINEAR_PROBES, PERTURB_SHIFT, MIN_SIZE = 9, 5, 8          # Objects/setobject.c


class PySet:
    """CPython 3.12's set table for small non-negative ints (hash(i) == i), insertions only"""

    def __init__(self):
        self.table = [None] * MIN_SIZE
        self.used = 0

    @property
    def mask(self):
        return len(self.table) - 1

    def _find(self, table, key):
        """set_add_entry's probe (set_insert_clean's for a key not present): the slot holding key or the empty one"""
        mask = len(table) - 1
        i, perturb = key & mask, key
        while True:
            probes = LINEAR_PROBES if i + LINEAR_PROBES <= mask else 0
            for j in range(i, i + probes + 1):
                if table[j] is None or table[j] == key:
                    return j
            perturb >>= PERTURB_SHIFT
            i = (i * 5 + 1 + perturb) & mask

    def add(self, key):
        s = self._find(self.table, key)
        if self.table[s] == key:
            return
        self.table[s] = key
        self.used += 1                     # fill == used: nothing is deleted
        if self.used * 5 < self.mask * 3:
            return
        size = MIN_SIZE                    # set_table_resize(so, used * 4)
        while size <= self.used * 4:
            size <<= 1
        old, self.table = self.table, [None] * size
        for k in old:
            if k is not None:
                self.table[self._find(self.table, k)] = k

    def __iter__(self):
        return (k for k in self.table if k is not None)


def set_order(keys):
    """list(set(keys)) as CPython 3.12 iterates it, for small non-negative ints"""
    s = PySet()
    for k in keys:
        s.add(int(k))
    return list(s)


def n_atoms(nodes):
    """rows up to the last non-zero one (graphinvent_b200.preprocess's atom count)"""
    nz = np.flatnonzero(np.asarray(nodes).any(1))
    return int(nz[-1]) + 1 if nz.size else 0


def _adjacency(edges, n):
    return [set(np.flatnonzero(np.asarray(edges)[i, :n].any(1)).tolist()) for i in range(n)]


def bfs(edges, ranking, n):
    """breadth_first_search(node_ranking=ranking, node_init=ranking[0]) over the molecule's first n atoms"""
    adj = _adjacency(edges, n)
    start = int(ranking[0])
    visited, layer = [start], [start]
    while len(visited) < n:
        seen = set(visited)
        s = PySet()
        for a in layer:
            for b in sorted(adj[a] - seen, key=lambda v: -ranking[v]):
                s.add(b)
        layer = list(s)
        if not layer:
            raise ValueError("disconnected graph: the reference's search does not terminate")
        visited += layer
    return visited


def dfs(edges, ranking, n):
    """depth_first_search(node_ranking=ranking, node_init=ranking[0]) over the molecule's first n atoms"""
    adj = _adjacency(edges, n)
    start = int(ranking[0])
    visited, last, stuck = [start], start, 0
    while len(visited) < n:
        new = adj[last] - set(visited)
        if not new:
            stuck += 1
            if stuck > len(visited):
                raise ValueError("disconnected graph: the reference's search does not terminate")
            last = visited[visited.index(last) - 1]
            continue
        stuck = 0
        last = max(new, key=lambda v: ranking[v])
        visited.append(last)
    return visited


def reorder(nodes, edges, order):
    """reorder_nodes, padded back to N: node rows and edge rows / columns in `order`, zero past len(order)"""
    nodes, edges = np.asarray(nodes), np.asarray(edges)
    X, E = np.zeros_like(nodes), np.zeros_like(edges)
    o = np.asarray(order, np.int64)
    X[:o.size] = nodes[o]
    E[:o.size, :o.size] = edges[o][:, o]
    return X, E


def node_remap(nodes, edges, ranking, route):
    """(order padded with -1 to N, reordered nodes, reordered edges) of one padded molecule"""
    n = n_atoms(nodes)
    order = (bfs if route == "bfs" else dfs)(edges, ranking, n)
    X, E = reorder(nodes, edges, order)
    out = np.full(nodes.shape[0], -1, np.int32)
    out[:n] = order
    return out, X, E
