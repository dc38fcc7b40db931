"""
ctypes binding of libgib200.so (C-ABI declared in include/gib200.h).

There is NO fallback: if the library cannot be built or loaded the import fails, and every
entry point raises on a non-zero return code.
"""
import ctypes
import os

from . import build as _build

c_p = ctypes.c_void_p
c_i = ctypes.c_int
c_ll = ctypes.c_longlong
c_f = ctypes.c_float
c_d = ctypes.c_double
c_sz = ctypes.c_size_t


class Dims(ctypes.Structure):
    """mirror of `gib_dims` (include/gib200.h).  `tf32`: the matmul precision the model entry points run in for these
    dims (0 = 3xTF32, 1 = single-pass TF32, 2 = bf16, 3 = fp16 operands)."""
    _fields_ = [(n, c_i) for n in (
        "model", "B", "N", "F", "Ef", "H", "M", "T", "msg_hidden", "msg_depth", "att_hidden", "att_depth",
        "eemb_hidden", "eemb_depth", "gather_width", "gatt_hidden", "gatt_depth", "gemb_hidden", "gemb_depth",
        "mlp1_hidden", "mlp1_depth", "mlp2_hidden", "mlp2_depth", "f_add", "f_conn")] + [
        ("big", c_f), ("in_dtype", c_i), ("tf32", c_i)]


class GemmProblem(ctypes.Structure):
    """mirror of `gib_gemm_problem` (include/gib200.h, test hooks)"""
    _fields_ = [("A", c_p), ("lda", c_i), ("W", c_p), ("ldw", c_i), ("W_hi", c_p), ("W_lo", c_p), ("C", c_p),
                ("ldc", c_i), ("M", c_i), ("N", c_i), ("K", c_i), ("bias", c_p), ("act", c_i), ("mode", c_i),
                ("aux", c_p), ("ldaux", c_i), ("n_store", c_i), ("n_valid", c_i), ("m_dev", c_p), ("base_dev", c_p),
                ("tf32", c_i)]


class DwProblem(ctypes.Structure):
    """mirror of `gib_dw_problem` (include/gib200.h, test hooks)"""
    _fields_ = [("G", c_p), ("ldg", c_i), ("Nn", c_i), ("X", c_p), ("ldx", c_i), ("Kk", c_i), ("M", c_i),
                ("dW", c_p), ("dbias", c_p), ("R", c_i), ("C", c_i), ("Rb", c_i), ("Rbp", c_i), ("rs", c_ll),
                ("cs", c_ll), ("m_dev", c_p), ("base_dev", c_p), ("tf32", c_i)]


class BatchCtl(ctypes.Structure):
    """mirror of `gib_batch_ctl` (include/gib200.h): the live molecule count and loss scale of a captured batch"""
    _fields_ = [("live", c_i), ("scale", c_f)]


class EvalPass(ctypes.Structure):
    """mirror of `gib_eval_pass` (include/gib200.h): the device-resident state of one validation pass"""
    _fields_ = [("batch_loss", c_p), ("lik", c_p), ("lik_len", c_ll), ("n_slots", c_i), ("idx", c_i),
                ("n_structures", c_f), ("flags", c_i), ("clipped", c_i), ("reserved", c_i)]


class MolLayout(ctypes.Structure):
    """mirror of `gib_mol_layout` (include/gib200.h): how `_features_to_atom` reads a node feature row"""
    _fields_ = [(n, c_i) for n in ("n_atom_types", "n_formal_charge", "n_imp_H", "use_imp_H", "use_chirality",
                                   "len_atom_types", "len_formal_charge", "len_imp_H", "len_chirality")]


class PPDims(ctypes.Structure):
    """mirror of `gib_pp_dims` (include/gib200.h): dims and action layout of the training-set construction"""
    _fields_ = [(n, c_i) for n in ("N", "F", "Ef", "n_atom_types", "n_formal_charge", "n_imp_H", "n_chirality",
                                   "batch_size")]


PP_STATUS_INTS = 8                                                  # GIB_PP_* (include/gib200.h)
PP_BAD_NODES, PP_BAD_EDGES, PP_EMPTY, PP_DISCONNECTED = 1, 2, 4, 8

MOL_HDR_WORDS, MOL_WORDS, MOL_ATOM_WORDS = 8, 6, 3                 # GIB_MOL_* (include/gib200.h)
MOL_DECODES, MOL_KEY_ERROR, MOL_DUPLICATE_BOND = 1, 2, 4
MOL_ERR_VALUE, MOL_ERR_OVERFLOW, MOL_ERR_INDEX = 1, 2, 3

MODEL_ID = {"GGNN": 0, "MNN": 1, "AttGGNN": 2, "EMN": 3}
HDR_INTS = 16
HDR_E, HDR_P, HDR_TYPE_COUNT, HDR_TYPE_BASE, HDR_FLAGS, HDR_CAPACITY = 0, 1, 2, 6, 11, 12
FLAG_MULTITYPE, FLAG_NONBINARY, FLAG_OVERFLOW = 1, 2, 4
ABI_VERSION = 206     # must equal gib_version() of the loaded library (include/gib200.h)

_PROTOS = {
    "gib_last_error": (ctypes.c_char_p, []),
    "gib_version": (c_i, []),
    "gib_set_tensor_cores": (None, [c_i]),
    "gib_get_tensor_cores": (c_i, []),
    "gib_tc_debug": (None, [c_i]),
    "gib_device_sm_count": (c_i, []),
    "gib_scatter_variant": (None, [c_i]),
    "gib_tc_trace": (None, [c_p, c_i]),
    "gib_graph_count_ws_bytes": (c_sz, [c_p]),
    "gib_graph_count": (c_i, [c_p, c_p, c_p, c_p]),
    "gib_graph_header_capacity": (c_i, [c_p, c_i, c_p, c_p]),
    "gib_graph_bytes": (c_sz, [c_p, c_p]),
    "gib_graph_fill": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p]),
    "gib_graph_array": (c_p, [c_p, c_p, c_p, c_i]),
    "gib_model_num_params": (c_i, [c_p]),
    "gib_model_param_numel": (c_ll, [c_p, c_i]),
    "gib_model_packed_bytes": (c_sz, [c_p]),
    "gib_model_pack": (c_i, [c_p, c_p, c_p, c_p]),
    "gib_model_workspace_bytes": (c_sz, [c_p, c_p]),
    "gib_model_forward": (c_i, [c_p] * 9),
    "gib_model_msg_rows": (c_p, [c_p, c_p, c_p, c_i]),
    "gib_model_bwd_scratch_bytes": (c_sz, [c_p, c_p]),
    "gib_model_backward": (c_i, [c_p] * 12),
    "gib_model_backward_part": (c_i, [c_p] * 11 + [c_i, c_p]),
    "gib_kl_loss_fwd_bwd": (c_i, [c_p, c_p, c_i, c_i, c_f, c_p, c_p, c_p]),
    "gib_linear_fwd": (c_i, [c_p, c_i, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "gib_linear_fwd_tc": (c_i, [c_p, c_i, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "gib_linear_fwd_tc_planes": (c_i, [c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_p]),
    "gib_split_planes": (c_i, [c_p, c_p, c_p, c_ll, c_p]),
    "gib_round_plane16": (c_i, [c_p, c_p, c_ll, c_i, c_p]),
    "gib_dw_scratch_bytes": (c_sz, [c_i, c_i, c_i]),
    "gib_linear_bwd_dw": (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "gib_scatter_sum": (c_i, [c_p, c_p, c_i, c_p, c_p, c_p, c_ll, c_p]),
    "gib_seg_softmax": (c_i, [c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_ll, c_p]),
    "gib_gru_gates": (c_i, [c_p, c_p, c_p, c_p, c_i, c_p, c_ll, c_p]),
    "gib_graph_gather": (c_i, [c_p, c_p, c_p, c_p, c_i, c_p, c_i, c_i, c_f, c_p]),
    "gib_validation_nll": (c_i, [c_p, c_p, c_i, c_i, c_p, c_p]),
    "gib_sum_scaled": (c_i, [c_p, c_i, c_f, c_p, c_p]),
    "gib_fill_zero": (c_i, [c_p, c_sz, c_p]),
    "gib_kl_loss_fwd_bwd_ctl": (c_i, [c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "gib_kl_loss_fwd_bwd_ctl_scaled": (c_i, [c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p]),
    "gib_sum_scaled_ctl": (c_i, [c_p, c_i, c_p, c_p, c_p]),
    "gib_validation_nll_ctl": (c_i, [c_p, c_p, c_i, c_i, c_p, c_p, c_p]),
    "gib_eval_collect": (c_i, [c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "gib_gather_rows": (c_i, [c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p, c_p, c_i, c_p, c_p, c_p]),
    "gib_adam_step": (c_i, [c_p, c_p, c_p, c_p, c_ll, c_ll, c_d, c_d, c_d, c_d, c_d, c_d, c_p]),
    "gib_nonfinite_check": (c_i, [c_p, c_ll, c_p, c_p]),
    "gib_adam_step_scaled": (c_i, [c_p, c_p, c_p, c_p, c_ll, c_p, c_p, c_p, c_d, c_d, c_d, c_d, c_d, c_d, c_p]),
    "gib_amp_update_scale": (c_i, [c_p, c_p, c_p, c_d, c_d, c_i, c_p, c_i, c_p]),
    "gib_sample_actions": (c_i, [c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "gib_generation_scratch_bytes": (c_sz, [c_i]),
    "gib_generation_round": (c_i, [c_i] * 7 + [c_p] * 11 + [c_i, c_p, c_p, c_p]),
    "gib_generation_round_layout": (c_i, [c_i] * 9 + [c_p] * 11 + [c_i, c_p, c_p, c_p]),
    "gib_generation_sample_round": (c_i, [c_i] * 8 + [c_p, c_i] + [c_p] * 13 + [c_i, c_p, c_p, c_p]),
    "gib_rl_sample_round": (c_i, [c_i] * 8 + [c_p, c_p, c_i] + [c_p] * 17 + [c_i, c_p, c_p, c_p]),
    "gib_rl_snapshot": (c_i, [c_i] * 5 + [c_p] * 9),
    "gib_rl_restore": (c_i, [c_i] * 4 + [c_p] * 6),
    "gib_rl_gather": (c_i, [c_i] * 3 + [c_p] * 6),
    "gib_rl_scatter_grad": (c_i, [c_i] * 3 + [c_p] * 6),
    "gib_rl_dlogits": (c_i, [c_i, c_i] + [c_p] * 7),
    "gib_rl_next_round": (c_i, [c_p, c_p]),
    "gib_molecule_table_bytes": (c_sz, [c_i] * 4),
    "gib_molecule_table": (c_i, [c_i] * 4 + [c_p] * 6),
    "gib_graph_statistics_bytes": (c_sz, [c_i] * 3),
    "gib_graph_statistics_ws_bytes": (c_sz, [c_i] * 4),
    "gib_graph_statistics": (c_i, [c_i] * 4 + [c_p] * 6),
    "gib_preprocess_apd_length": (c_i, [c_p]),
    "gib_preprocess_ws_bytes": (c_sz, [c_p, c_i, c_i]),
    "gib_preprocess_chunk": (c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i] + [c_p] * 7),
    "gib_preprocess_group_statistics_bytes": (c_sz, [c_p, c_i]),
    "gib_preprocess_group_statistics_ws_bytes": (c_sz, [c_p, c_i]),
    "gib_preprocess_group_statistics": (c_i, [c_p, c_p, c_p, c_i, c_i] + [c_p] * 5),
    "gib_route_plan_ws_bytes": (c_sz, [c_p, c_i]),
    "gib_route_max_states": (c_ll, [c_p, c_i]),
    "gib_route_plan": (c_i, [c_p, c_p, c_p, c_i, c_i] + [c_p] * 4),
    "gib_route_fill": (c_i, [c_p, c_p, c_p, c_i] + [c_p] * 8),
    "gib_route_probs": (c_i, [c_i, c_i, c_p, c_p, c_p, c_p]),
    "gib_route_reduce": (c_i, [c_i] + [c_p] * 5),
    "gib_route_grad_coef": (c_i, [c_i] + [c_p] * 7),
    "gib_route_dlogits": (c_i, [c_i, c_i] + [c_p] * 6),
    "gib_profile_enable": (None, [c_i]),
    "gib_launch_count": (c_ll, []),
    "gib_profile_collect": (c_i, [c_p, c_p, c_p]),
    "gib_profile_records": (c_i, [c_p, c_p, c_p, c_i]),
    "gib_test_chain_flag_bytes": (c_sz, [c_p, c_i]),
    "gib_test_gemm_nt": (c_i, [c_p, c_i, c_p, c_p, c_p]),
    "gib_test_dw_scratch_bytes": (c_sz, [c_p, c_p, c_i, c_ll]),
    "gib_test_dw_groups": (c_i, [c_p, c_p, c_i, c_ll, c_p, c_p]),
    "gib_test_scatter_bwd": (c_i, [c_p, c_p, c_p, c_i, c_p, c_p, c_i, c_ll, c_p]),
    "gib_test_seg_reduce_dact": (c_i, [c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_ll, c_p]),
    "gib_test_seg_softmax_bwd": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_ll, c_p]),
    "gib_test_gru_bwd": (c_i, [c_p] * 7 + [c_i, c_p, c_ll, c_p, c_p]),
    "gib_test_colsum_add": (c_i, [c_p, c_p, c_i, c_ll, c_i, c_i, c_i, c_p, c_p]),
    "gib_test_graph_gather_bwd": (c_i, [c_p] * 6 + [c_i, c_i, c_i, c_p]),
    "gib_test_emn_aggregate_fwd": (c_i, [c_p] * 5 + [c_i] + [c_p] * 3 + [c_ll, c_p, c_p]),
    "gib_test_emn_aggregate_bwd": (c_i, [c_p] * 10 + [c_i] + [c_p] * 5 + [c_ll, c_p, c_p]),
    "gib_test_scatter_sum": (c_i, [c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_ll, c_p]),
    "gib_test_gru_fwd": (c_i, [c_p, c_p, c_p, c_p, c_i, c_p, c_ll, c_p, c_p]),
    "gib_test_gather_rows": (c_i, [c_p, c_p, c_i, c_p, c_p, c_i, c_ll, c_p, c_p]),
    "gib_test_sum_nodes_fwd": (c_i, [c_p, c_p, c_i, c_i, c_i, c_p]),
    "gib_test_bcast_nodes_add": (c_i, [c_p, c_p, c_i, c_i, c_ll, c_p]),
    "gib_test_concat2_in": (c_i, [c_p, c_i, c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_ll, c_p]),
    "gib_test_concat_flat": (c_i, [c_p, c_i, c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_p]),
    "gib_test_unflatten_dact": (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_ll, c_p]),
    "gib_test_dact_slice": (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "gib_test_sum3_cols": (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_p]),
    "gib_test_tanh_fwd": (c_i, [c_p, c_p, c_ll, c_i, c_p, c_p]),
    "gib_test_tanh_selu_bwd": (c_i, [c_p, c_p, c_p, c_p, c_ll, c_i, c_p, c_p]),
    "gib_test_mul_dselu": (c_i, [c_p, c_p, c_p, c_ll, c_i, c_p, c_p]),
    "gib_test_emn_input": (c_i, [c_p, c_i, c_p, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_ll, c_p]),
    "gib_test_plan_linear": (c_i, [c_p, c_i, c_p]),
}
PLAN_LINEAR_FIELDS = ("pw", "pb", "src_off", "rs", "cs", "nblk", "Rb", "Rbp", "C", "Cp", "Ct", "Ctp",
                      "ow", "owt", "ob", "ow_hi", "ow_lo", "owt_hi", "owt_lo")   # GIB_PLAN_LINEAR_FIELDS, in order


def exported_symbols():
    """every symbol include/gib200.h declares (checked by the CPU test-suite)"""
    return sorted(_PROTOS)


def _load():
    path = _build.LIB
    try:
        path = _build.build()
    except Exception as e:  # no nvcc on this box (the GPU box runs the library built in the container)
        if not os.path.exists(path):
            raise ImportError(f"libgib200.so is missing and could not be built: {e}") from e
        if _build.is_stale():
            import warnings
            warnings.warn(f"libgib200.so is older than its sources and could not be rebuilt ({e}); loading it anyway "
                          "-- the ABI version check below decides")
    lib = ctypes.CDLL(path)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    got = lib.gib_version()
    if got != ABI_VERSION:
        raise ImportError(f"{path} implements ABI version {got}, this package binds version {ABI_VERSION}: "
                          "rebuild with `python -m graphinvent_b200.build --force`")
    return lib


lib = _load()
LIB_PATH = _build.LIB
# A/B measurements only: GIB_TC_DEBUG=<mode> applies gib_tc_debug(mode) to the whole process (include/gib200.h) so that
# any test or tool can be re-run with another GEMM call pattern
if os.environ.get("GIB_TC_DEBUG"):
    lib.gib_tc_debug(int(os.environ["GIB_TC_DEBUG"], 0))


def check(rc, what=""):
    if rc == 0:
        return
    msg = lib.gib_last_error().decode(errors="replace")
    if rc > 0:
        raise RuntimeError(f"{what}: CUDA error {rc} ({msg})")
    raise RuntimeError(f"{what}: invalid argument ({rc}): {msg}")
