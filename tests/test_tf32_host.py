"""CPU: the matmul precision -- torch's setting read by `config.tf32_enabled`, carried by `make_dims` / `dims_key` in
`gib_dims.tf32` to every call -- and the C-ABI pieces that do not need a GPU."""
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT


@pytest.fixture(autouse=True)
def _restore_precision():
    m, g = torch.backends.cuda.matmul.fp32_precision, torch.backends.fp32_precision
    yield
    torch.backends.fp32_precision = g
    torch.backends.cuda.matmul.fp32_precision = m


def test_default_is_3xtf32():
    from graphinvent_b200.config import tf32_enabled
    assert torch.backends.cuda.matmul.fp32_precision in ("none", "ieee")
    assert tf32_enabled() is False


@pytest.mark.parametrize("level,want", [("highest", False), ("high", True), ("medium", True)])
def test_legacy_setter_levels(level, want):
    from graphinvent_b200.config import tf32_enabled
    torch.set_float32_matmul_precision(level)
    assert tf32_enabled() is want


@pytest.mark.parametrize("matmul,glob,want", [
    ("tf32", "ieee", True), ("ieee", "tf32", False), ("tf32", "tf32", True), ("ieee", "ieee", False),
    ("none", "tf32", True), ("none", "ieee", False), ("none", "none", False), ("tf32", "none", True)])
def test_new_api_with_none_inheritance(matmul, glob, want):
    from graphinvent_b200.config import tf32_enabled
    torch.backends.fp32_precision = glob
    torch.backends.cuda.matmul.fp32_precision = matmul
    assert tf32_enabled() is want


def test_mixed_legacy_and_new_use_never_raises():
    """after a mix of the two APIs torch's legacy getters raise; the switch reads only the new ones"""
    from graphinvent_b200.config import tf32_enabled
    torch.backends.cuda.matmul.fp32_precision = "none"
    torch.backends.fp32_precision = "tf32"
    torch.backends.cuda.matmul.allow_tf32 = False
    assert tf32_enabled() is False
    torch.set_float32_matmul_precision("high")
    torch.backends.fp32_precision = "ieee"
    assert tf32_enabled() is True
    torch.backends.cuda.matmul.fp32_precision = "none"
    assert tf32_enabled() is False


def _net():
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    return mpnn.create(O.make_constants("GGNN"))


def test_make_dims_and_dims_key_carry_the_mode():
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import Dims
    net = _net()
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    d0, k0 = Fn.make_dims(net, 64), Fn.dims_key(net, 64)
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    d1, k1 = Fn.make_dims(net, 64), Fn.dims_key(net, 64)
    assert (d0.tf32, d1.tf32) == (0, 1)
    assert k0 != k1 and k0[:-1] == k1[:-1] and (k0[-1], k1[-1]) == (0, 1)
    assert Fn.make_dims(net, 64, tf32=False).tf32 == 0 and Fn.dims_key(net, 64, tf32=0) == k0
    assert Fn.key_of(d1) == k1 == tuple(getattr(d1, name) for name, _ in Dims._fields_)
    assert bytes(d0) != bytes(d1)                # the mode is part of the C struct
    d1.tf32 = 0
    assert bytes(d0) == bytes(d1)


def test_abi_struct_layouts_match_the_header():
    """gib_dims has 28 fields; it and the test-hook problems end in `int tf32`"""
    from graphinvent_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "gib200.h")).read()
    assert ctypes.sizeof(_lib.Dims) == 28 * 4 and len(_lib.Dims._fields_) == 28
    for struct, cls in (("gib_dims", _lib.Dims), ("gib_gemm_problem", _lib.GemmProblem),
                        ("gib_dw_problem", _lib.DwProblem)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr, re.S).group(1)
        assert body.strip().endswith("int tf32;"), struct
        assert cls._fields_[-1] == ("tf32", ctypes.c_int)
        assert cls.tf32.offset + 4 <= ctypes.sizeof(cls)
    assert _lib.ABI_VERSION == _lib.lib.gib_version()


def _model_calls(d):
    """gib_model_pack, gib_model_forward and gib_model_backward on dims `d` with null device pointers (an exact-mode
    host header): each one that refuses the dims returns before it touches the device"""
    from graphinvent_b200._lib import lib
    h = (ctypes.c_int * 16)(1000, 1024, 1000, 0, 0, 0, 0, 1024)      # E, P, one type group of 1000 entries
    bd = ctypes.byref(d)
    return {"gib_model_pack": lambda: lib.gib_model_pack(bd, None, None, None),
            "gib_model_forward": lambda: lib.gib_model_forward(bd, h, *[None] * 7),
            "gib_model_backward": lambda: lib.gib_model_backward(bd, h, *[None] * 10)}


def test_model_calls_refuse_an_unknown_precision():
    """the precision travels with the dims: an unknown code is refused by each call that reads it"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import lib
    d = Fn.make_dims(_net(), 256)
    for code in (5, -1):
        d.tf32 = code
        for name, call in _model_calls(d).items():
            assert call() == -2, (name, code)
            err = lib.gib_last_error().decode()
            assert err.startswith(name) and "precision %d" % code in err, (name, err)


def test_size_queries_do_not_depend_on_the_mode():
    import numpy as np
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import DwProblem, GemmProblem, lib
    for model in ("GGNN", "EMN"):
        from graphinvent_b200.gnn import mpnn
        from oracle import mpnn_oracle as O
        net = mpnn.create(O.make_constants(model))
        d = Fn.make_dims(net, 256)
        hdr = np.zeros(16, np.int32)
        hdr[0], hdr[1], hdr[2], hdr[6], hdr[7] = 1000, 1024, 1000, 0, 1024
        h = hdr.ctypes.data_as(ctypes.c_void_p)
        sizes = []
        for on in (0, 1):
            d.tf32 = on
            sizes.append((lib.gib_model_packed_bytes(ctypes.byref(d)), lib.gib_model_workspace_bytes(ctypes.byref(d), h),
                          lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), h)))
        assert sizes[0] == sizes[1] and all(s > 0 for s in sizes[0]), (model, sizes)
    qs = (DwProblem * 2)()
    ps = (GemmProblem * 2)()
    for q, p, m in zip(qs, ps, (4097, 1500)):
        q.M, q.Nn, q.Kk = m, 112, 144
        p.M, p.N, p.K = m, 64, 32
    sizes = (ctypes.c_int * 1)(2)
    a = (lib.gib_test_dw_scratch_bytes(qs, sizes, 1, 0), lib.gib_test_chain_flag_bytes(ps, 2))
    for q, p in zip(qs, ps):
        q.tf32 = p.tf32 = 1
    assert (lib.gib_test_dw_scratch_bytes(qs, sizes, 1, 0), lib.gib_test_chain_flag_bytes(ps, 2)) == a
