"""
Fixture of tests/test_device_loader_host.py and tests/test_gpu_device_loader.py: the batch order of the unmodified
reference BlockDataLoader (BlockDatasetLoader.py, with `h5py.File` replaced by in-memory int8 arrays) and the state of
torch's default generator after a pass, for a table of cases.  Each row's nodes carry the row's own index, so a batch's
indices are read back from the batch itself.

    python tests/golden/make_loader_order.py        # needs the reference installed by __graft_entry__.build()

Per case i: case{i}/params = (rows, batch, block, shuffle, n_workers, seed, stop): torch.manual_seed(seed), one pass,
broken off after `stop` batches when stop >= 0; case{i}/sizes: the batch sizes (-1 marks a batch of the one-row last
block, whose batch dimension the reference's torch.squeeze dropped), case{i}/indices: the row indices of the other
batches, concatenated; case{i}/len: len(loader); case{i}/rand: torch.rand(4) drawn after the pass.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SRC = os.path.join(ROOT, "oracle", "_ref", "graphinvent", "BlockDatasetLoader.py")
# (rows, batch, block, shuffle, n_workers, seed, stop)
CASES = [
    (1234, 100, 500, True, 0, 0, -1),
    (1234, 100, 500, True, 2, 1, -1),
    (2100, 100, 1000, True, 2, 2, -1),
    (2350, 64, 1000, True, 0, 3, -1),
    (1234, 100, 500, False, 0, 4, -1),
    (1234, 100, 500, True, 0, 5, 7),
    (2350, 64, 1000, True, 0, 6, 17),
    (2350, 64, 1000, True, 0, 6, 0),
    (9, 2, 3, True, 0, 8, -1),           # the reference's drop_last expression is True
    (30, 2, 3, True, 0, 9, -1),          # ... and False
    (1001, 100, 1000, True, 0, 10, -1),  # a one-row last block
    (256, 32, 100, True, 0, 11, -1),     # tests/golden/gdb13_train_head256.h5 at block 100, batch 32
    (256, 32, 100, True, 0, 11, 4),
    (301, 32, 100, True, 0, 12, -1),     # the GPU tests' 4-block set with a one-row last block
    (301, 32, 100, True, 0, 12, 5),
]
DIMS = (2, 4, 1, 3)                      # N, F, Ef, apd of the index-carrying rows


def reference_module():
    """the reference's BlockDatasetLoader module, its `import h5py` stubbed (`h5py.File` set by `reference_loader`)"""
    if not os.path.exists(SRC):
        return None
    saved = sys.modules.get("h5py")
    sys.modules["h5py"] = types.ModuleType("h5py")
    try:
        spec = importlib.util.spec_from_file_location("_ref_BlockDatasetLoader", SRC)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            del sys.modules["h5py"]
        else:
            sys.modules["h5py"] = saved
    return mod


def reference_loader(mod, nodes, edges, apds, **kw):
    """the unmodified BlockDataLoader over an unmodified HDFDataset whose file is the in-memory int8 arrays"""
    arrays = {"nodes": nodes, "edges": edges, "APDs": apds}
    mod.h5py.File = lambda path, mode="r", swmr=False: arrays
    return mod.BlockDataLoader(mod.HDFDataset("<memory>"), **kw)


def indexed_rows(n, dims=DIMS):
    """n int8 rows whose nodes[i, 0, :4] hold i in base 128"""
    N, F, Ef, apd = dims
    nodes = np.zeros((n, N, F), np.int8)
    for j in range(4):
        nodes[:, 0, j] = (np.arange(n) >> (7 * j)) & 127
    edges = np.zeros((n, N, N, Ef), np.int8)
    apds = np.zeros((n, apd), np.int8)
    return nodes, edges, apds


def row_index(nodes):
    """the indices carried by a float32 batch of indexed_rows"""
    v = nodes[:, 0, :4].to(torch.int64)
    return sum(v[:, j] << (7 * j) for j in range(4))


def run_reference(mod, rows, batch, block, shuffle, n_workers, seed, stop):
    """one pass of the reference loader: (sizes, indices, len, rand)"""
    nodes, edges, apds = indexed_rows(rows)
    loader = reference_loader(mod, nodes, edges, apds, batch_size=batch, block_size=block, shuffle=shuffle,
                              n_workers=n_workers, pin_memory=False)
    torch.manual_seed(seed)
    sizes, indices = [], []
    for idx, (n, _, _) in enumerate(loader):
        if idx == stop:
            break
        if n.dim() == 3:
            sizes.append(n.shape[0])
            indices.append(row_index(n))
        else:
            sizes.append(-1)
    rand = torch.rand(4)
    idx = torch.cat(indices).numpy() if indices else np.zeros(0, np.int64)
    return np.array(sizes, np.int64), idx, len(loader), rand.numpy()


def main():
    mod = reference_module()
    assert mod is not None, f"{SRC} is missing: run __graft_entry__.build() with the reference checkout present"
    out = {}
    for i, case in enumerate(CASES):
        sizes, idx, n, rand = run_reference(mod, *case)
        out[f"case{i}/params"] = np.array([int(v) for v in case], np.int64)
        out[f"case{i}/sizes"], out[f"case{i}/indices"] = sizes, idx
        out[f"case{i}/len"], out[f"case{i}/rand"] = np.int64(n), rand
    np.savez_compressed(os.path.join(HERE, "loader_order.npz"), **out)


if __name__ == "__main__":
    main()
