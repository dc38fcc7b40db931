"""CPU: the restatement of the reference's decoding-route choice (tests/route_order_reference.py) against the reference's
own BFS / DFS orders (tests/golden/route_orders.npz), and its model of CPython's set table against the interpreter."""
import hashlib
import itertools
import os
import random
import sys

import numpy as np
import pytest

from tests import route_order_reference as RO
from tests.conftest import GOLDEN

FIXTURE = os.path.join(GOLDEN, "route_orders.npz")
CPYTHON_312 = sys.version_info[:2] == (3, 12)


def test_fixture_records_its_python():
    z = np.load(FIXTURE)
    assert str(z["python_version"]).startswith("3.12.")


@pytest.mark.parametrize("name", ["gdb13", "synthetic38"])
@pytest.mark.parametrize("route", ["bfs", "dfs"])
def test_restatement_matches_the_reference_orders(name, route):
    z = np.load(FIXTURE)
    nodes, edges = z[f"{name}/nodes"], z[f"{name}/edges"]
    rankings, orders = z[f"{name}/rankings"], z[f"{name}/orders"][:, :, 0 if route == "bfs" else 1]
    M, R, N = rankings.shape
    out_n = np.zeros((M, R) + nodes.shape[1:], np.int8)
    out_e = np.zeros((M, R) + edges.shape[1:], np.int8)
    for m in range(M):
        n = RO.n_atoms(nodes[m])
        for k in range(R):
            order, out_n[m, k], out_e[m, k] = RO.node_remap(nodes[m], edges[m], rankings[m, k, :n].tolist(), route)
            assert np.array_equal(order, orders[m, k]), (m, k)
    assert hashlib.sha256(out_n.tobytes() + out_e.tobytes()).hexdigest() == str(z[f"{name}/sha256_{route}"])


def test_fixture_exercises_set_order_quirks():
    """the N = 38 BFS orders include layers whose order is not ascending atom index"""
    z = np.load(FIXTURE)
    nodes, edges, rankings = z["synthetic38/nodes"], z["synthetic38/edges"], z["synthetic38/rankings"]
    quirks = 0
    for m in range(nodes.shape[0]):
        n = RO.n_atoms(nodes[m])
        for k in range(rankings.shape[1]):
            r = rankings[m, k, :n].tolist()
            for layer in _layers(edges[m], r, n):
                quirks += layer != sorted(layer)
    assert quirks > 0


def _layers(edges, ranking, n):
    order = RO.bfs(edges, ranking, n)
    adj = RO._adjacency(edges, n)
    depth = {order[0]: 0}
    for a in order[1:]:
        depth[a] = 1 + min(depth[b] for b in adj[a] if b in depth)
    out = {}
    for a in order:
        out.setdefault(depth[a], []).append(a)
    return list(out.values())


@pytest.mark.skipif(not CPYTHON_312, reason="models CPython 3.12's set table")
@pytest.mark.parametrize("values", [range(6), [0, 8, 16, 24, 32, 40], [9, 1, 17, 33, 25, 41], [5, 13, 21, 29, 37, 2],
                                    [0, 32, 64, 96, 128, 160], [7, 15, 23, 31, 39, 47]])
def test_set_order_every_insertion_order(values):
    for k in range(1, 7):
        for sub in itertools.combinations(values, k):
            for p in itertools.permutations(sub):
                assert RO.set_order(p) == list(set(p)), p
    assert RO.set_order([9, 1]) == [9, 1] and RO.set_order([1, 9]) == [1, 9]


@pytest.mark.skipif(not CPYTHON_312, reason="models CPython 3.12's set table")
def test_set_order_random_lists():
    rng = random.Random(5)
    for _ in range(5000):
        xs = [rng.randint(0, 180) for _ in range(rng.randint(1, 400))]
        assert RO.set_order(xs) == list(set(xs))
        xs = [np.int64(x) for x in xs]
        assert RO.set_order(xs) == [int(x) for x in set(xs)]


def test_disconnected_is_an_error():
    E = np.zeros((4, 4, 1), np.int8)
    E[0, 1, 0] = E[1, 0, 0] = 1
    E[2, 3, 0] = E[3, 2, 0] = 1
    for search in (RO.bfs, RO.dfs):
        with pytest.raises(ValueError, match="disconnected"):
            search(E, [0, 1, 2, 3], 4)
