"""
Hyper-parameter tuple for the drop-in modules when no reference `parameters.constants` is
around (benchmarks, tests, standalone use).  Field names and default values are the
reference's (`parameters/defaults.py:93-128, 145-433`; derived dims `constants.py:158-211`);
any namedtuple/object with these attributes works -- the reference's own `constants` does.
"""
from collections import namedtuple

DEFAULTS = dict(
    model="GGNN", device="cuda", big_positive=1e6, big_negative=-1e6,
    n_node_features=8, n_edge_features=3, max_n_nodes=13,          # gdb13: 5 atom types + 3 charges
    len_f_add_per_node=45, len_f_conn_per_node=3,
    hidden_node_features=100, message_size=100, message_passes=3,
    enn_hidden_dim=250, enn_depth=4, enn_dropout_p=0.0,
    msg_hidden_dim=250, msg_depth=4, msg_dropout_p=0.0,
    att_hidden_dim=250, att_depth=4, att_dropout_p=0.0,
    gather_width=100,
    gather_att_hidden_dim=250, gather_att_depth=4, gather_att_dropout_p=0.0,
    gather_emb_hidden_dim=250, gather_emb_depth=4, gather_emb_dropout_p=0.0,
    mlp1_hidden_dim=500, mlp1_depth=4, mlp1_dropout_p=0.0,
    mlp2_hidden_dim=500, mlp2_depth=4, mlp2_dropout_p=0.0,
    edge_emb_size=100, edge_emb_hidden_dim=250, edge_emb_depth=4, edge_emb_dropout_p=0.0,
)


def tf32_enabled():
    """True when torch would run a CUDA float32 matmul on single-pass TF32 tensor cores, which is then the precision of
    this package's tensor-core GEMMs too (else 3xTF32, fp32-accurate).  torch's rule: the matmul backend's
    `torch.backends.cuda.matmul.fp32_precision`, or the global `torch.backends.fp32_precision` when the backend's is
    "none"; "tf32" means TF32.  `torch.set_float32_matmul_precision("high")` and `("medium")` show up as "tf32" there.
    Only these two values are read: the legacy getters (`allow_tf32`, `get_float32_matmul_precision`) raise after a
    mix of the legacy and the new setters."""
    import torch
    p = getattr(torch.backends.cuda.matmul, "fp32_precision", "none")
    if p == "none":
        p = getattr(torch.backends, "fp32_precision", "none")
    return p == "tf32"


def autocast_dtype():
    """`torch.bfloat16` / `torch.float16` when torch's CUDA autocast is on with one of these dtypes -- the reference's
    `Linear`s and `GRUCell`s then run on 16-bit tensor cores, and so do this package's tensor-core GEMMs -- else None
    (autocast off, or another autocast dtype)."""
    import torch
    if not torch.is_autocast_enabled("cuda"):
        return None
    dt = torch.get_autocast_dtype("cuda")
    return dt if dt in (torch.bfloat16, torch.float16) else None


# precision codes of the tensor-core GEMMs (`gib_dims.tf32`, `Dims.tf32`)
PREC_3XTF32, PREC_TF32, PREC_BF16, PREC_FP16 = 0, 1, 2, 3


def matmul_code(fp16=True):
    """The precision code the tensor-core GEMMs follow, by torch's own precedence: a 16-bit autocast dtype
    (`autocast_dtype`: 2 = bf16, 3 = fp16), else the TF32 setting (`tf32_enabled`: 1), else 3xTF32 (0).  Under autocast
    the TF32 setting does not matter, as for torch's autocast matmuls.  `fp16=False`: fp16 autocast is not honoured and
    the rule continues with the TF32 setting (the captured training step, whose fused loss has no gradient scaling)."""
    import torch
    dt = autocast_dtype()
    if dt is torch.bfloat16:
        return PREC_BF16
    if dt is torch.float16 and fp16:
        return PREC_FP16
    return PREC_TF32 if tf32_enabled() else PREC_3XTF32


def dtype_of_code(code):
    """the autocast dtype a precision code stands for (None for the fp32-input codes 0 / 1)"""
    import torch
    return {PREC_BF16: torch.bfloat16, PREC_FP16: torch.float16}.get(int(code))


def make_constants(model="GGNN", **overrides):
    d = dict(DEFAULTS, model=model)
    d.update(overrides)
    d.setdefault("edge_features", d["n_edge_features"])          # names EdgeMPNN.__init__ reads
    d.setdefault("edge_embedding_size", d["edge_emb_size"])      # (edge_mpnn.py:16-17)
    return namedtuple("constants", sorted(d))(**d)


def apd_length(C):
    return C.max_n_nodes * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1


def layout_dims(n_atom_types, n_formal_charge, n_edge_features=3, use_explicit_H=False, ignore_H=True,
                use_chirality=False, n_imp_H_values=4, n_chirality_values=3):
    """Derived node-feature and action dims of one of the reference's four action layouts, restated from
    `parameters/constants.py:23-95, 169-184` (`n_imp_H_values` = len(imp_H), `n_chirality_values` = len(chirality)):
    implicit-H counts form a node-feature segment only when H is neither explicit nor ignored, chirality when
    `use_chirality` is set.  Pass the result to `make_constants` to build a model of the right shape."""
    if use_explicit_H and ignore_H:
        raise ValueError("use_explicit_H and ignore_H cannot both be set (the reference refuses the same flags)")
    implicit_H = not use_explicit_H and not ignore_H
    n_imp_H = int(implicit_H) * n_imp_H_values
    n_chirality = int(use_chirality) * n_chirality_values
    dim_f_add = [n_atom_types, n_formal_charge] + [n_imp_H] * implicit_H + [n_chirality] * use_chirality
    len_f_add = n_edge_features
    for n in dim_f_add:
        len_f_add *= n
    return dict(n_node_features=n_atom_types + n_formal_charge + n_imp_H + n_chirality,
                n_edge_features=n_edge_features, len_f_add_per_node=len_f_add,
                len_f_conn_per_node=n_edge_features,
                n_atom_types=n_atom_types, n_formal_charge=n_formal_charge, n_imp_H=n_imp_H, n_chirality=n_chirality)
