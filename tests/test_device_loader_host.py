"""Host tests of graphinvent_b200.loader.DeviceBlockLoader (no GPU): its batch order and its draws from torch's default
generator against tests/golden/loader_order.npz (the reference BlockDataLoader's, made by
tests/golden/make_loader_order.py) and, when oracle/_ref/ holds the reference, against the live reference over a
further sweep; the reference's one-row-block behaviour; the constructor's refusals; the gib_gather_rows binding."""
import os
import types

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN
from tests.golden.make_loader_order import indexed_rows, reference_loader, reference_module, row_index, run_reference

FIXTURE = np.load(os.path.join(GOLDEN, "loader_order.npz"))
N_CASES = len([k for k in FIXTURE.files if k.endswith("/params")])


def _dataset(nodes, edges, apds):
    return types.SimpleNamespace(nodes=nodes, edges=edges, apds=apds)


def replica(rows, batch, block, shuffle, n_workers, seed, stop):
    """DeviceBlockLoader's order for one case, as make_loader_order.run_reference records the reference's: (sizes with
    -1 for the one-row last block's batch, global row indices of the other batches, len, torch.rand(4) after)"""
    from graphinvent_b200.loader import DeviceBlockLoader
    loader = DeviceBlockLoader(_dataset(*indexed_rows(rows)), batch_size=batch, block_size=block, shuffle=shuffle,
                               n_workers=n_workers)
    torch.manual_seed(seed)
    sizes, indices = [], []
    for idx, (k, ix) in enumerate(loader.order()):
        if idx == stop:
            break
        lo, hi = loader._block_range(k)
        if hi - lo == 1:
            sizes.append(-1)
        else:
            sizes.append(ix.numel())
            indices.append(ix + lo)
    rand = torch.rand(4)
    idx = torch.cat(indices).numpy() if indices else np.zeros(0, np.int64)
    return np.array(sizes, np.int64), idx, len(loader), rand.numpy()


@pytest.mark.parametrize("i", range(N_CASES))
def test_order_matches_the_reference_fixture(i):
    case = [int(v) for v in FIXTURE[f"case{i}/params"]]
    sizes, idx, n, rand = replica(*case)
    assert np.array_equal(sizes, FIXTURE[f"case{i}/sizes"])
    assert np.array_equal(idx, FIXTURE[f"case{i}/indices"])
    assert n == int(FIXTURE[f"case{i}/len"])
    assert np.array_equal(rand, FIXTURE[f"case{i}/rand"])        # the generator state after the (broken) pass


SWEEP = [(777, 50, 200, True, 0), (777, 50, 200, False, 2), (5000, 7, 100, True, 0), (1500, 100, 100, True, 1),
         (9, 2, 3, True, 2), (64, 64, 64, True, 0), (65, 64, 64, True, 0), (130, 64, 64, False, 0),
         (3000, 3, 10, True, 0), (2201, 100, 1100, True, 2)]


@pytest.mark.parametrize("rows,batch,block,shuffle,n_workers", SWEEP)
def test_order_matches_the_live_reference(rows, batch, block, shuffle, n_workers):
    mod = reference_module()
    if mod is None:
        pytest.skip("the reference's BlockDatasetLoader.py is not installed in oracle/_ref/")
    n_batches = None
    for seed, stop in ((21, -1), (22, 3), (23, None)):
        if stop is None:                                  # break inside the last block
            stop = max(n_batches - 2, 0)
        ref = run_reference(mod, rows, batch, block, shuffle, n_workers, seed, stop)
        got = replica(rows, batch, block, shuffle, n_workers, seed, stop)
        for a, b in zip(got, ref):
            assert np.array_equal(np.asarray(a), np.asarray(b))
        n_batches = len(ref[0]) if n_batches is None else n_batches


def test_reference_one_row_block_drops_the_batch_dimension():
    """the reference's torch.squeeze on a one-row block: 1001 gdb13-sized rows, block 1000, batch 100 -- its last batch
    indexes the atoms of that one molecule.  DeviceBlockLoader yields that block as one batch of one molecule."""
    from graphinvent_b200.loader import DeviceBlockLoader
    mod = reference_module()
    if mod is None:
        pytest.skip("the reference's BlockDatasetLoader.py is not installed in oracle/_ref/")
    nodes, edges, apds = np.zeros((1001, 13, 8), np.int8), np.zeros((1001, 13, 13, 3), np.int8), np.zeros(
        (1001, 625), np.int8)
    torch.manual_seed(0)
    shapes = [tuple(tuple(t.shape) for t in b) for b in reference_loader(mod, nodes, edges, apds, batch_size=100,
                                                                         block_size=1000, pin_memory=False)]
    odd = [s for s in shapes if len(s[0]) != 3]
    assert odd == [((13, 8), (13, 13, 3), (13,))]
    loader = DeviceBlockLoader(_dataset(nodes, edges, apds), batch_size=100, block_size=1000)
    torch.manual_seed(0)
    ours = [(k, ix.numel()) for k, ix in loader.order()]
    assert ours[-1] == (1, 1) and len(ours) == len(shapes) == len(loader) == 11


def test_drop_last_is_the_reference_expression():
    from graphinvent_b200.loader import DeviceBlockLoader
    for rows, block, expect in ((9, 3, True), (30, 3, False), (12, 3, False), (2000, 100, False),
                                (100 * 100 * 2, 100, True), (100 * 100 + 1, 100, False)):
        loader = DeviceBlockLoader(_dataset(*indexed_rows(rows)), batch_size=2, block_size=block)
        n = loader.n_blocks
        assert loader.drop_last == bool(int(n / block) > 1 & n % block < block / 10) == expect, (rows, block)


def test_refusals():
    from graphinvent_b200.loader import DeviceBlockLoader
    nodes, edges, apds = indexed_rows(10)
    with pytest.raises(ValueError, match="block_size"):
        DeviceBlockLoader(_dataset(nodes, edges, apds), batch_size=8, block_size=4)
    with pytest.raises(ValueError, match="rows"):
        DeviceBlockLoader(_dataset(nodes, edges, apds[:9]), batch_size=2, block_size=4)
    with pytest.raises(ValueError, match="rows"):
        DeviceBlockLoader(_dataset(nodes[:9], edges, apds), batch_size=2, block_size=4)
    with pytest.raises(ValueError, match="do not match"):
        DeviceBlockLoader(_dataset(nodes, np.zeros((10, 3, 3, 1), np.int8), apds), batch_size=2, block_size=4)
    with pytest.raises(ValueError, match=r"\[n, N, F\]"):
        DeviceBlockLoader(_dataset(nodes[:, 0], edges, apds), batch_size=2, block_size=4)
    with pytest.raises(ValueError, match="int8"):
        DeviceBlockLoader(_dataset(nodes.astype(np.float32), edges, apds), batch_size=2, block_size=4)
    with pytest.raises(ValueError, match="no rows"):
        DeviceBlockLoader(_dataset(nodes[:0], edges[:0], apds[:0]), batch_size=2, block_size=4)


def test_indexed_rows_round_trip():
    nodes, _, _ = indexed_rows(70000)
    assert torch.equal(row_index(torch.from_numpy(nodes).float()), torch.arange(70000))


def test_gather_rows_symbol_is_bound():
    import ctypes
    from graphinvent_b200 import _lib
    assert "gib_gather_rows" in _lib.exported_symbols()
    fn = _lib.lib.gib_gather_rows
    assert fn.restype is ctypes.c_int and len(fn.argtypes) == 15
    # refusals that need no device: b > B, non-positive dims, an unknown out_dtype, null pointers
    p = ctypes.c_void_p(16)
    for args, what in (((p, p, p, p, 5, 4, 8, 8, 8, p, p, 0, p, None, None), "b <= B"),
                       ((p, p, p, p, 1, 4, 0, 8, 8, p, p, 0, p, None, None), "row_nodes"),
                       ((p, p, p, p, 1, 4, 8, 8, 8, p, p, 2, p, None, None), "out_dtype"),
                       ((p, None, p, p, 1, 4, 8, 8, 8, p, p, 0, p, None, None), "null"),
                       ((p, p, p, None, 1, 4, 8, 8, 8, p, p, 0, p, None, None), "null"),
                       ((ctypes.c_void_p(17), p, p, p, 1, 4, 8, 8, 8, p, p, 0, p, None, None), "aligned")):
        assert fn(*args) < 0
        assert what in _lib.lib.gib_last_error().decode()
