"""
Hyper-parameter tuple for the drop-in modules when no reference `parameters.constants` is
around (benchmarks, tests, standalone use).  Field names and default values are the
reference's (`parameters/defaults.py:93-128, 145-433`; derived dims `constants.py:158-211`);
any namedtuple/object with these attributes works -- the reference's own `constants` does.
"""
from collections import namedtuple

import numpy as np

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


# The action mask's valence limits (`action_mask="valence"`): the largest valence, in bonds counted by order (aromatic
# 1.5) plus implicit hydrogens, that the mask lets an atom of that element and formal charge reach.  They are upper
# bounds by design -- the mask removes only bonds that no valence state of the (element, charge) allows -- and this
# package's own values, not checked against RDKit's valence model.
DEFAULT_MAX_VALENCE = {
    ("C", -1): 3, ("C", 0): 4, ("C", 1): 3,
    ("N", -1): 2, ("N", 0): 3, ("N", 1): 4,
    ("O", -1): 1, ("O", 0): 2, ("O", 1): 3,
    ("S", -1): 5, ("S", 0): 6, ("S", 1): 7,
    ("Cl", -1): 0, ("Cl", 0): 1, ("Cl", 1): 2,
    ("H", 0): 1, ("B", 0): 3, ("F", 0): 1, ("Si", 0): 4, ("P", 0): 5, ("Br", 0): 1, ("I", 0): 1,
}
# bond orders in half-bond units, by the name of the reference's `int_to_bondtype` entries
BOND_HALF_ORDERS = {"SINGLE": 2, "DOUBLE": 4, "TRIPLE": 6, "AROMATIC": 3}


def _bond_name(bt):
    """"SINGLE" for rdkit's BondType.SINGLE, its str() or the plain name"""
    name = getattr(bt, "name", None) or str(bt)
    return name.rsplit(".", 1)[-1].upper()


def action_rule_table(n_atom_types, n_formal_charge, n_edge_features, n_imp_H=0, max_valence=None, constants=None):
    """The action mask's rule table: (V int32 [A, CH], bond orders int32 [Ef] in half-bond units, implicit-H counts
    int32 [H]).  Bond orders come from `constants.int_to_bondtype` (SINGLE / DOUBLE / TRIPLE / AROMATIC = 2 / 4 / 6 /
    3), or in that order without it; implicit-H counts from `constants.imp_H`, or the index without it.

    max_valence: None (DEFAULT_MAX_VALENCE), a dict keyed by element symbol (every charge of that element) or by
    (symbol, charge), which overrides the defaults and is resolved through `constants.atom_types` /
    `constants.formal_charge`, or an int array [A, CH] by index, which needs no constants.  A (type, charge) pair of
    the layout that neither covers raises ValueError naming it."""
    A, CH, Ef, H = int(n_atom_types), int(n_formal_charge), int(n_edge_features), int(n_imp_H)
    itb = getattr(constants, "int_to_bondtype", None)
    if itb is not None:
        if len(itb) != Ef:
            raise ValueError(f"constants.int_to_bondtype names {len(itb)} bond types, the layout has {Ef}")
        names = [_bond_name(itb[i]) for i in range(Ef)]
    elif Ef <= 4:
        names = ["SINGLE", "DOUBLE", "TRIPLE", "AROMATIC"][:Ef]
    else:
        raise ValueError(f"{Ef} bond types need constants.int_to_bondtype to name their orders")
    bad = [n for n in names if n not in BOND_HALF_ORDERS]
    if bad:
        raise ValueError(f"bond type {bad[0]} has no order here (known: {', '.join(BOND_HALF_ORDERS)})")
    order = np.array([BOND_HALF_ORDERS[n] for n in names], np.int32)
    imp = getattr(constants, "imp_H", None)
    imp_h = np.array(list(imp) if imp is not None else range(H), np.int64) if H else np.zeros(0, np.int64)
    if imp_h.size != H:
        raise ValueError(f"constants.imp_H lists {imp_h.size} counts, the layout has {H} implicit-H indices")
    if max_valence is not None and not isinstance(max_valence, dict):
        V = np.asarray(max_valence)
        if V.shape != (A, CH) or not np.issubdtype(V.dtype, np.integer):
            raise ValueError(f"max_valence must be an int array [n_atom_types, n_formal_charge] = [{A}, {CH}] or a "
                             f"dict, got {V.dtype} {V.shape}")
    else:
        atoms, charges = getattr(constants, "atom_types", None), getattr(constants, "formal_charge", None)
        if atoms is None or charges is None:
            raise ValueError("a valence table by element needs constants with atom_types and formal_charge; give "
                             "max_valence as an int array [n_atom_types, n_formal_charge] instead")
        if len(atoms) != A or len(charges) != CH:
            raise ValueError(f"constants list {len(atoms)} atom types and {len(charges)} charges, the layout has "
                             f"{A} and {CH}")
        user = dict(max_valence or {})
        V = np.zeros((A, CH), np.int64)
        for t, sym in enumerate(atoms):
            for c, q in enumerate(charges):
                key = (sym, int(q))
                v = user.get(key, user.get(sym, DEFAULT_MAX_VALENCE.get(key)))
                if v is None:
                    raise ValueError(f"no valence limit for atom type {sym!r} with formal charge {int(q):+d}: add "
                                     f"max_valence={{({sym!r}, {int(q)}): ...}}")
                V[t, c] = int(v)
    if (V < 0).any() or (V > 1 << 20).any() or (imp_h < 0).any() or (imp_h > 1 << 20).any():
        raise ValueError("valence limits and implicit-H counts must lie in [0, 2**20]")
    return V.astype(np.int32), order, imp_h.astype(np.int32)


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
