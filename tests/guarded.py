"""Guarded buffers for memory-discipline tests: one allocation of `guard + n + guard` bytes whose interior is handed to
the library as an ordinary buffer and whose two bands must come back untouched.

The bands (and, on request, the interior) are filled with 0xFF bytes.  Read as float32 that is NaN, so a kernel that
reads bytes no kernel of the call wrote turns a finite result into NaN; read as int32 it is -1, which the index kernels
treat as a pad row, so a stray index read stays inside the allocation.  `intact()` compares both bands byte for byte.
"""
import torch

POISON = 0xFF
MIB = 1 << 20
ALIGN = 512          # the caching allocator's block alignment: interiors keep it


class Guarded:
    def __init__(self, nbytes, device="cuda", guard=MIB, fill="poison"):
        """fill: "poison" (0xFF), "zero", or None (the interior is filled by the caller)"""
        self.n = int(nbytes)
        guard = -(-max(int(guard), MIB) // ALIGN) * ALIGN
        self.raw = torch.full((guard + self.n + guard + ALIGN,), POISON, dtype=torch.uint8, device=device)
        self.start = guard + (-(self.raw.data_ptr() + guard) % ALIGN)   # host allocations are less aligned than CUDA's
        self.t = self.raw[self.start: self.start + self.n]                # the interior (uint8)
        if fill == "zero":
            self.t.zero_()

    @classmethod
    def like(cls, src, device="cuda", guard=MIB):
        """a guarded copy of a tensor (inputs, targets); view() gives it back with src's dtype and shape"""
        g = cls(src.numel() * src.element_size(), device=device, guard=guard, fill=None)
        g.src_meta = (src.dtype, tuple(src.shape))
        g.view(src.dtype, src.shape).copy_(src)
        return g

    def view(self, dtype=None, shape=None):
        if dtype is None:
            dtype, shape = self.src_meta
        v = self.t.view(dtype)
        return v if shape is None else v.view(shape)

    def ptr(self):
        return self.t.data_ptr()

    def intact(self):
        lo, hi = self.raw[: self.start], self.raw[self.start + self.n:]
        return bool((lo == POISON).all()) and bool((hi == POISON).all())

    def damage(self):
        """byte offsets, relative to the interior's start, of the first and last changed band byte (None if intact)"""
        bad = torch.nonzero(self.raw != POISON).flatten()
        bad = bad[(bad < self.start) | (bad >= self.start + self.n)]
        if bad.numel() == 0:
            return None
        return int(bad[0]) - self.start, int(bad[-1]) - self.start
