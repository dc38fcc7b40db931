"""CPU: the autocast precision rule -- `config.autocast_dtype` / `config.matmul_code` over torch's autocast and TF32
state, the codes 2 / 3 carried by `make_dims` / `dims_key` in `gib_dims.tf32` -- and the C-ABI pieces of the 16-bit
modes that need no GPU.  A real `torch.autocast("cuda")` context turns itself off without a CUDA device, so the
state is set with torch's setters and restored afterwards."""
import contextlib
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT


@contextlib.contextmanager
def autocast_state(enabled, dtype=None, tf32=None):
    e, d = torch.is_autocast_enabled("cuda"), torch.get_autocast_dtype("cuda")
    m = torch.backends.cuda.matmul.fp32_precision
    try:
        torch.set_autocast_enabled("cuda", enabled)
        if dtype is not None:
            torch.set_autocast_dtype("cuda", dtype)
        if tf32 is not None:
            torch.backends.cuda.matmul.fp32_precision = "tf32" if tf32 else "ieee"
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = m
        torch.set_autocast_dtype("cuda", d)
        torch.set_autocast_enabled("cuda", e)


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64])
@pytest.mark.parametrize("enabled", [False, True])
def test_rule_matrix(enabled, dtype, tf32):
    from graphinvent_b200.config import autocast_dtype, matmul_code
    with autocast_state(enabled, dtype, tf32):
        want_dt = dtype if enabled and dtype in (torch.bfloat16, torch.float16) else None
        assert autocast_dtype() is want_dt
        want = {torch.bfloat16: 2, torch.float16: 3}.get(want_dt, int(tf32))
        assert matmul_code() == want
        # the captured training step does not take fp16: it falls through to the TF32 setting
        assert matmul_code(fp16=False) == (2 if want_dt is torch.bfloat16 else int(tf32))
    assert autocast_dtype() is None and matmul_code() == 0


def _net(model="GGNN"):
    from graphinvent_b200.gnn import mpnn
    from oracle import mpnn_oracle as O
    return mpnn.create(O.make_constants(model))


def test_make_dims_and_keys_carry_the_16bit_codes():
    from graphinvent_b200 import functional as Fn
    net = _net()
    k0 = Fn.dims_key(net, 64)
    got = {}
    for dt, code in ((torch.bfloat16, 2), (torch.float16, 3)):
        with autocast_state(True, dt, tf32=True):
            d, k = Fn.make_dims(net, 64), Fn.dims_key(net, 64)
        assert d.tf32 == code and k[-1] == code and k[:-1] == k0[:-1] and Fn.key_of(d) == k
        assert Fn.autocast_dtype_of(d) is dt
        assert bytes(d) != bytes(Fn.make_dims(net, 64, tf32=0))    # the mode is part of the C struct
        got[code] = k
    assert len({k0, got[2], got[3], Fn.dims_key(net, 64, tf32=1)}) == 4
    assert Fn.make_dims(net, 64, tf32=2).tf32 == 2 and Fn.make_dims(net, 64, tf32=3).tf32 == 3
    assert Fn.make_dims(net, 64, tf32=True).tf32 == 1 and Fn.make_dims(net, 64, tf32=7).tf32 == 1
    assert Fn.autocast_dtype_of(Fn.make_dims(net, 64, tf32=1)) is None


def test_model_calls_refuse_16bit_codes_without_tensor_cores():
    """the 16-bit codes travel with the dims to each call that reads them, which refuses them on the fp32 SIMT path"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import lib
    from tests.test_tf32_host import _model_calls
    d = Fn.make_dims(_net(), 256)
    prev = lib.gib_get_tensor_cores()
    lib.gib_set_tensor_cores(0)
    try:
        for code in (2, 3):
            d.tf32 = code
            for name, call in _model_calls(d).items():
                assert call() == -2, (name, code)
                err = lib.gib_last_error().decode()
                assert err.startswith(name) and "tensor-core path" in err, (name, err)
    finally:
        lib.gib_set_tensor_cores(prev)


def test_size_queries_do_not_depend_on_any_mode():
    import numpy as np
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200._lib import DwProblem, GemmProblem, lib
    for model in ("GGNN", "MNN", "AttGGNN", "EMN"):
        d = Fn.make_dims(_net(model), 256)
        hdr = np.zeros(16, np.int32)
        hdr[0], hdr[1], hdr[2], hdr[6], hdr[7] = 1000, 1024, 1000, 0, 1024
        h = hdr.ctypes.data_as(ctypes.c_void_p)
        sizes = []
        for on in (0, 1, 2, 3):
            d.tf32 = on
            sizes.append((lib.gib_model_packed_bytes(ctypes.byref(d)), lib.gib_model_workspace_bytes(ctypes.byref(d), h),
                          lib.gib_model_bwd_scratch_bytes(ctypes.byref(d), h)))
        assert len(set(sizes)) == 1 and all(s > 0 for s in sizes[0]), (model, sizes)
    qs = (DwProblem * 2)()
    ps = (GemmProblem * 2)()
    for q, p, m in zip(qs, ps, (4097, 1500)):
        q.M, q.Nn, q.Kk = m, 112, 144
        p.M, p.N, p.K = m, 64, 32
    n = (ctypes.c_int * 1)(2)
    a = (lib.gib_test_dw_scratch_bytes(qs, n, 1, 0), lib.gib_test_chain_flag_bytes(ps, 2))
    for code in (1, 2, 3):
        for q, p in zip(qs, ps):
            q.tf32 = p.tf32 = code
        assert (lib.gib_test_dw_scratch_bytes(qs, n, 1, 0), lib.gib_test_chain_flag_bytes(ps, 2)) == a


def test_abi_layout_unchanged_and_the_plane_helper_is_exported():
    from graphinvent_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "gib200.h")).read()
    assert ctypes.sizeof(_lib.Dims) == 28 * 4 and _lib.ABI_VERSION == 206 == _lib.lib.gib_version()
    for struct in ("gib_dims", "gib_gemm_problem", "gib_dw_problem"):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr, re.S).group(1)
        assert body.strip().endswith("int tf32;"), struct
    assert "gib_round_plane16" in _lib.exported_symbols()
    assert re.search(r"int gib_round_plane16\(const float\* W, void\* out, long long n, int kind, gib_stream stream\);",
                     hdr)
    assert _lib.lib.gib_round_plane16(None, None, 4, 1, None) < 0     # kind 1 is not a 16-bit code: refused
    assert b"kind" in _lib.lib.gib_last_error()


def test_train_step_maps_fp16_autocast_to_the_fp32_input_modes():
    """the captured training step's rule, as it applies it at construction: bf16 kept, fp16 not taken"""
    from graphinvent_b200 import functional as Fn
    from graphinvent_b200.config import matmul_code
    net = _net()
    for dt, tf32, want in ((torch.bfloat16, False, 2), (torch.float16, False, 0), (torch.float16, True, 1)):
        with autocast_state(True, dt, tf32):
            d = Fn.make_dims(net, 32, 0, tf32=matmul_code(fp16=False))
        assert d.tf32 == want and (Fn.autocast_dtype_of(d) is None) == (want < 2)
    src = open(os.path.join(ROOT, "graphinvent_b200", "graphed.py")).read()
    train = src[src.index("class TrainStep"):src.index("class EvalStep")]
    assert "matmul_code(fp16=False)" in train
