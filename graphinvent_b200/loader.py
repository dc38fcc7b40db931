"""
The training and validation sets on the device: `DeviceBlockLoader`, a drop-in for the reference's `BlockDataLoader`
(BlockDatasetLoader.py) in `Workflow.get_dataloader`.

    loader = graphinvent_b200.loader.DeviceBlockLoader(HDFDataset(path), batch_size=B, block_size=K)
    for nodes, edges, target in loader:          # float32 device tensors
        ...
    loss = step.train_epoch(loader, scheduler)   # graphed.TrainStep: one gather launch per batch, no host copies

Order.  The batches are the reference's, in its order, and the pass takes the same draws from torch's default
generator at the same points: the order comes from torch's own DataLoader run over index ranges -- an outer loader over
range(n_blocks) and, when block k starts, an inner loader over range(len(block k)) -- built with the arguments the
reference gives its loaders (num_workers=0: the main process makes the same draws either way).  A pass broken off
early leaves the generator where the reference's pass leaves it.

Streaming.  The int8 rows stay int8 on the device, one block per slot, two slots.  While block k is consumed, block
k + 1 is read on a background thread into one of two pinned staging buffers and copied to the other slot on a side
stream; the slot is refilled only after an event recorded behind its last gather, and the first gather of a block
waits on its copy's event.  A block still resident from an earlier pass is not uploaded again, so a one-block set is
uploaded once (`uploads` counts block uploads).  Each batch is one `gib_gather_rows` launch on the current stream.

Deviation: when the last block holds one row, the reference's `torch.squeeze` drops that block's batch dimension and
its ShuffleBlockWrapper then indexes atoms as molecules; here that block is a batch of one molecule (INTEGRATION.md
section 2).  Its draws are the reference's.
"""
import ctypes
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import functional as F
from ._lib import check, lib

__all__ = ["DeviceBlockLoader", "RandomRouteLoader"]


class _Batch:
    """one batch of a pass: b rows of block slot `slot`, listed in the device int32 tensor `rows`"""
    __slots__ = ("slot", "rows", "b")

    def __init__(self, slot, rows, b):
        self.slot, self.rows, self.b = slot, rows, b


class DeviceBlockLoader:
    def __init__(self, dataset, batch_size=100, block_size=10000, shuffle=True, n_workers=0, pin_memory=True,
                 device=None):
        """the reference's BlockDataLoader arguments; n_workers and pin_memory are accepted and have no effect.
        `dataset`: the reference's HDFDataset or any object with int8 `nodes` [n, N, F], `edges` [n, N, N, Ef] and
        `apds` [n, apd] array-likes that can be sliced by rows (h5py datasets, numpy arrays), or three contiguous int8
        tensors on the loader's device, whose rows are gathered in place."""
        self.batch_size, self.block_size = int(batch_size), int(block_size)
        self.shuffle, self.n_workers, self.pin_memory = bool(shuffle), n_workers, pin_memory
        if self.batch_size < 1:
            raise ValueError(f"batch_size must be >= 1, got {batch_size}")
        if self.block_size < self.batch_size:
            raise ValueError(f"block_size ({self.block_size}) must be >= batch_size ({self.batch_size}), as the "
                             "reference's BlockDataset asserts")
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._bind(dataset)

    def _bind(self, dataset):
        """takes `dataset`'s rows: checks them and sets up the pass state.  Rows held as int8 device tensors on the
        loader's device are gathered in place (both slots are the whole set, a batch's rows are indices into it): no
        staging or uploads."""
        self.dataset = dataset
        arrays = (dataset.nodes, dataset.edges, dataset.apds)
        shapes = [tuple(a.shape) for a in arrays]
        if len(shapes[0]) != 3 or len(shapes[1]) != 4 or len(shapes[2]) != 2:
            raise ValueError(f"nodes / edges / apds must be [n, N, F] / [n, N, N, Ef] / [n, apd], got {shapes}")
        if not shapes[0][0] == shapes[1][0] == shapes[2][0]:
            raise ValueError(f"nodes, edges and apds hold {shapes[0][0]}, {shapes[1][0]} and {shapes[2][0]} rows")
        if shapes[1][1] != shapes[0][1] or shapes[1][2] != shapes[0][1]:
            raise ValueError(f"edges {shapes[1]} do not match nodes {shapes[0]}: need [n, N, N, Ef] with N = "
                             f"{shapes[0][1]}")
        self._on_device = all(isinstance(a, torch.Tensor) and a.is_cuda for a in arrays)
        for name, a in zip(("nodes", "edges", "apds"), arrays):
            if isinstance(a, torch.Tensor):
                if a.dtype != torch.int8 or not a.is_contiguous() or (a.is_cuda and (not self._on_device
                                                                                     or a.device != self.device)):
                    raise ValueError(f"{name}: a tensor must be contiguous int8 on {self.device} (device rows) or a "
                                     f"host array, got {a.dtype} on {a.device}")
            elif np.dtype(a.dtype) != np.int8:
                raise ValueError(f"{name} must be int8 (the reference's preprocessed HDF5 layout), got {a.dtype}")
        self.n_rows = shapes[0][0]
        if self.n_rows < 1:
            raise ValueError("the dataset holds no rows")
        _, self.N, self.F = shapes[0]
        self.Ef, self.apd = shapes[1][3], shapes[2][1]
        self.row_bytes = (self.N * self.F, self.N * self.N * self.Ef, self.apd)
        self.n_blocks = -(-self.n_rows // self.block_size)
        # the reference's drop_last expression, evaluated as Python does (with its precedence it is False unless there
        # are about block_size blocks or more)
        n_blocks, block_size = self.n_blocks, self.block_size
        self.drop_last = bool(int(n_blocks / block_size) > 1 & n_blocks % block_size < block_size / 10)
        self.uploads = 0
        self._slot_rows = min(self.block_size, self.n_rows)
        self._slots = [None, None]          # per slot: (nodes, edges, apds) int8 device tensors
        self._staging = [None, None]        # per slot: pinned host tensors of the same shapes
        self._resident = [None, None]       # per slot: the block it holds (or is being loaded with)
        self._ready = [None, None]          # per slot: event after its upload
        self._free = [None, None]           # per slot: event after its last gather
        self._staged = [None, None]         # per staging buffer: event after its last upload read it
        self._pending = {}                  # slot -> future of its upload
        self._side = None
        self._reader = None

    # ---- the reference's BlockDataLoader protocol --------------------------------------------------------------
    def __len__(self):
        """the reference's BlockDataLoader.__len__"""
        return self._count(self.n_rows)

    def _count(self, n_rows):
        n_blocks, n_rem = divmod(n_rows, self.block_size)
        return -(-self.block_size // self.batch_size) * n_blocks + -(-n_rem // self.batch_size)

    def __iter__(self):
        """(nodes, edges, target): fresh float32 device tensors, one gather launch per batch"""
        for item in self.batches():
            b = item.b
            nodes = torch.empty(b, self.N, self.F, dtype=torch.float32, device=self.device)
            edges = torch.empty(b, self.N, self.N, self.Ef, dtype=torch.float32, device=self.device)
            target = torch.empty(b, self.apd, dtype=torch.float32, device=self.device)
            self.gather(item, nodes, edges, target)
            yield nodes, edges, target

    # ---- the order -------------------------------------------------------------------------------------------
    def _block_range(self, k):
        return k * self.block_size, min((k + 1) * self.block_size, self.n_rows)

    def _blocks(self):
        """(block, next block or None, inner index loader) per block of a pass.  Taking the next block from the outer
        loader draws nothing from the default generator, so its upload can start before this block's order is drawn."""
        outer = iter(torch.utils.data.DataLoader(range(self.n_blocks), shuffle=self.shuffle, num_workers=0))
        nxt = next(outer, None)
        while nxt is not None:
            k = int(nxt)
            nxt = next(outer, None)
            lo, hi = self._block_range(k)
            inner = torch.utils.data.DataLoader(range(hi - lo), shuffle=self.shuffle, batch_size=self.batch_size,
                                                num_workers=0, drop_last=self.drop_last)
            yield k, None if nxt is None else int(nxt), inner

    def order(self):
        """the pass's batches as (block, int64 row indices within the block), drawn lazily as the reference draws;
        needs no device"""
        for k, _, inner in self._blocks():
            for idx in inner:
                yield k, idx

    # ---- streaming -------------------------------------------------------------------------------------------
    def _read(self, k, slot):
        """background thread: block k into staging buffer `slot`, then its upload into device slot `slot`"""
        lo, hi = self._block_range(k)
        m = hi - lo
        if self._staged[slot] is not None:
            self._staged[slot].synchronize()             # the previous upload from this buffer has read it
        for a, host in zip((self.dataset.nodes, self.dataset.edges, self.dataset.apds), self._staging[slot]):
            host.numpy()[:m] = a[lo:hi]
        with torch.cuda.device(self.device), torch.cuda.stream(self._side):
            self._side.wait_event(self._free[slot])       # the slot's last gather has run
            for dev, host in zip(self._slots[slot], self._staging[slot]):
                dev[:m].copy_(host[:m], non_blocking=True)
            self._ready[slot].record(self._side)
            self._staged[slot].record(self._side)

    def _allocate(self, slot):
        if self._slots[slot] is not None:
            return
        R, N, F_, Ef = self._slot_rows, self.N, self.F, self.Ef
        shapes = ((R, N, F_), (R, N, N, Ef), (R, self.apd))
        self._slots[slot] = tuple(torch.empty(s, dtype=torch.int8, device=self.device) for s in shapes)
        self._staging[slot] = tuple(torch.empty(s, dtype=torch.int8, pin_memory=True) for s in shapes)
        self._ready[slot], self._free[slot], self._staged[slot] = (torch.cuda.Event(), torch.cuda.Event(),
                                                                   torch.cuda.Event())
        self._free[slot].record(torch.cuda.current_stream(self.device))
        if self._side is None:
            self._side = torch.cuda.Stream(self.device)
            self._reader = ThreadPoolExecutor(max_workers=1, thread_name_prefix="DeviceBlockLoader")

    def _load(self, k, avoid=None):
        """the slot that holds or will hold block k, starting its upload if needed; `avoid`: the slot in use"""
        for slot in (0, 1):
            if self._resident[slot] == k:
                return slot
        slot = 1 - avoid if avoid is not None else (0 if self._resident[0] is None else 1)
        self._wait(slot)
        if self._on_device:        # device rows: the slot is the whole set (16-byte aligned), its rows offset by block
            self._slots[slot] = (self.dataset.nodes, self.dataset.edges, self.dataset.apds)
            self._resident[slot] = k
            if self._ready[slot] is None:
                self._ready[slot], self._free[slot] = torch.cuda.Event(), torch.cuda.Event()
                self._ready[slot].record(torch.cuda.current_stream(self.device))
            return slot
        self._allocate(slot)
        self._resident[slot] = k
        self._pending[slot] = self._reader.submit(self._read, k, slot)
        self.uploads += 1
        return slot

    def _wait(self, slot):
        fut = self._pending.pop(slot, None)
        if fut is not None:
            try:
                fut.result()
            except BaseException:
                self._resident[slot] = None
                raise

    def batches(self):
        """the pass as `_Batch` items (slot, device int32 rows, b) without materialising any batch: hand each to
        `gather`.  The draws are those of the reference's pass (see `order`)."""
        cur = torch.cuda.current_stream(self.device)
        for slot in (0, 1):                               # an earlier pass may have stopped with an upload queued
            self._wait(slot)
        slot = None
        for k, nxt, inner in self._blocks():
            slot = self._load(k, avoid=slot)
            if nxt is not None:
                self._load(nxt, avoid=slot)
            # the block's whole order at its start: the inner sampler draws its seed at its first batch and nothing after
            order = list(inner)
            if not order:
                continue
            self._wait(slot)
            cur.wait_event(self._ready[slot])
            rows = torch.cat(order)
            if self._on_device:
                rows += self._block_range(k)[0]
            rows = rows.to(torch.int32).pin_memory().to(self.device, non_blocking=True)
            off = 0
            for idx in order:
                b = idx.numel()
                yield _Batch(slot, rows[off:off + b], b)
                off += b

    def gather(self, item, nodes, edges, target, ctl=None):
        """`gib_gather_rows` of one batch into [B, ...] outputs (B >= item.b; rows past b are zeroed): nodes / edges
        float32 or int8, target float32; `ctl`: a gib_batch_ctl to set to {b, 1/b}, or None"""
        B = nodes.shape[0]
        if edges.shape[0] != B or target.shape[0] != B:
            raise ValueError(f"nodes, edges and target hold {B}, {edges.shape[0]} and {target.shape[0]} rows")
        if (nodes[0].numel(), edges[0].numel(), target[0].numel()) != self.row_bytes:
            raise ValueError(f"outputs of row sizes {(nodes[0].numel(), edges[0].numel(), target[0].numel())} for a "
                             f"loader of row sizes {self.row_bytes}")
        if nodes.dtype != edges.dtype or nodes.dtype not in (torch.float32, torch.int8):
            raise ValueError(f"nodes / edges must both be float32 or both int8, got {nodes.dtype} / {edges.dtype}")
        if target.dtype != torch.float32:
            raise ValueError(f"target must be float32, got {target.dtype}")
        for t in (nodes, edges, target):
            if t.device != self.device or not t.is_contiguous():
                raise ValueError(f"outputs must be contiguous tensors on {self.device}")
        src = self._slots[item.slot]
        check(lib.gib_gather_rows(F._ptr(src[0]), F._ptr(src[1]), F._ptr(src[2]), F._ptr(item.rows), item.b, B,
                                  *self.row_bytes, F._ptr(nodes), F._ptr(edges), int(nodes.dtype == torch.int8),
                                  F._ptr(target), F._ptr(ctl),
                                  F._stream(self.device)), "gib_gather_rows")
        self._free[item.slot].record(torch.cuda.current_stream(self.device))


class RandomRouteLoader(DeviceBlockLoader):
    """Training passes over fresh random decoding routes: pass e is exactly `DeviceBlockLoader(ds_e, batch_size,
    block_size, shuffle)`, where ds_e is the int8 file the reference's preprocessing writes for the molecules reordered
    by `preprocess.reorder(nodes, edges, route, seed=seed, epoch=e)` -- the same batches and the same draws from
    torch's default generator.  The reordering and the construction run on the device; the ranking draws depend on
    (seed, e, molecule) only and take nothing from torch's generators.

        loader = RandomRouteLoader(nodes, edges, batch_size=B, block_size=K, route="bfs", seed=0, constants=C)
        scheduler = OneCycleLR(optimizer, ..., total_steps=loader.total_batches(start_epoch, n_epochs))
        loader.set_epoch(start_epoch)                 # a restarted job
        loss = step.train_epoch(loader, scheduler)    # graphed.TrainStep; one call per pass

    `epoch` is the epoch of the upcoming pass: it starts at 0 (or `set_epoch`) and advances by one when a pass starts,
    so `len(loader)` before a pass counts that pass's batches.  A pass's rows are built when the pass or its `len` is
    first needed and stay on the device until the next pass's are built: about
    `preprocess.file_rows`' sum over molecules of (bonds + 2) rows at N*F + N*N*Ef + apd bytes each (6.5 KB at N = 38
    with gdb13's layout).  A set whose rows do not fit raises torch's out-of-memory error.  The molecule stacks stay on
    the device too.  Building the next pass's rows (its `len`) while a pass is being consumed ends that pass."""

    def __init__(self, nodes, edges, batch_size=100, block_size=10000, route="bfs", seed=0, n_atom_types=None,
                 n_formal_charge=None, n_imp_H=0, n_chirality=0, constants=None, shuffle=True, chunk_molecules=4096,
                 device=None):
        """`nodes` [M, N, F] / `edges` [M, N, N, Ef]: int8 padded molecules (numpy or torch), in any atom order.  The
        layout: `constants` (the reference's, through `preprocess.layout_of`) or the segment widths."""
        from . import preprocess
        if route not in ("bfs", "dfs"):
            raise ValueError(f"route must be 'bfs' or 'dfs', got {route!r}")
        if constants is not None:
            self.layout = preprocess.layout_of(constants)
        elif n_atom_types is None or n_formal_charge is None:
            raise ValueError("give constants= or n_atom_types and n_formal_charge")
        else:
            self.layout = (int(n_atom_types), int(n_formal_charge), int(n_imp_H), int(n_chirality))
        self.route, self.seed, self.chunk_molecules = route, int(seed), int(chunk_molecules)
        self.batch_size, self.block_size, self.shuffle = int(batch_size), int(block_size), bool(shuffle)
        if self.batch_size < 1 or self.block_size < self.batch_size:
            raise ValueError(f"need 1 <= batch_size <= block_size, got {batch_size} and {block_size}")
        self.n_workers, self.pin_memory = 0, False
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.M, self.N, self.F, self.Ef = preprocess._check_stacks(nodes, edges)
        if self.M < 1:
            raise ValueError("no molecules")
        self.nodes = preprocess._on_device(nodes, self.device)
        self.edges = preprocess._on_device(edges, self.device)
        d = preprocess._pp_dims(self.N, self.F, self.Ef, self.layout, self.batch_size)
        self.apd = preprocess.lib.gib_preprocess_apd_length(ctypes.byref(d))
        self.row_bytes = (self.N * self.F, self.N * self.N * self.Ef, self.apd)
        self.epoch = 0
        self._built = None                  # the epoch whose rows are bound

    def set_epoch(self, epoch):
        """the next pass (and `len`) is epoch `epoch`: resumes a job or repeats a pass"""
        self.epoch = int(epoch)

    def _rows(self, epoch, keep):
        from . import preprocess
        nodes, edges, _ = preprocess.reorder(self.nodes, self.edges, self.route, seed=self.seed, epoch=epoch,
                                             layout=self.layout, device=self.device)
        return preprocess.file_rows(nodes, edges, self.batch_size, *self.layout, chunk_molecules=self.chunk_molecules,
                                    keep=keep, device=self.device)

    def _build(self):
        if self._built == self.epoch:
            return
        self._built = None
        self.dataset = self._slots = None                     # the last pass's rows go before the next pass's come
        rows, _ = self._rows(self.epoch, keep=True)
        self._bind(types.SimpleNamespace(nodes=rows[0], edges=rows[1], apds=rows[2]))
        self._built = self.epoch

    def __len__(self):
        """batches of the upcoming pass (epoch `epoch`), building its rows"""
        self._build()
        return super().__len__()

    def total_batches(self, first_epoch, n_epochs):
        """sum of len() over passes first_epoch .. first_epoch + n_epochs - 1, counted without keeping their rows:
        the total_steps of a OneCycleLR over those passes"""
        return sum(self._count(self.n_rows if e == self._built else self._rows(e, keep=False)[1])
                   for e in range(int(first_epoch), int(first_epoch) + int(n_epochs)))

    def batches(self):
        """the pass of epoch `epoch` (DeviceBlockLoader.batches over its rows); the epoch advances as it starts"""
        self._build()
        self.epoch += 1
        yield from super().batches()
