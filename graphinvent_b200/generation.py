"""
Batched graph generation with the round post-processing on the device (SURVEY.md §8f rank 1).

Mirror of the reference's `GraphGenerator` (GraphGenerator.py:25-161) for the part that is tensor work:
`build_graphs()` runs model forward -> softmax/sample -> ONE `gib_generation_round(_layout)` call per round (decode, validity
rules, copy-out, apply, reset; the reference issues ~800 ATen ops for the same) until `batch_size` molecules are
finished; `sample()` returns the finished tensors and likelihood summaries.  Converting tensors to RDKit molecules
(`graph_to_graph`, GraphGenerator.py:659-804) stays the reference's job -- feed it `generated_nodes/edges/n_nodes`.

All four of the reference's action layouts are supported (parameters/constants.py:23-95): node features atom type +
formal charge, plus an implicit-H segment (`n_imp_H` > 0) and / or a chirality segment (`n_chirality` > 0), with the
add actions laid out as [bond_to, atom, charge, (imp_h,) (chirality,) bond_type].  `config.layout_dims` derives the
dims of a layout from the reference's flags.  The reference's quirks are kept in every layout (graphinvent_b200/csrc/
generate.cu lists them): with both segments present the first atom of every molecule gets chirality index 0.  An add
into a graph that already holds max_n_nodes atoms terminates the molecule as invalid in every layout; outside the
gdb13 layout the reference raises IndexError there instead.

The sampler draws with inverse-CDF on `torch.rand` uniforms (same distribution as `Multinomial(1, probs)`, different
RNG stream); `build_graphs(replay=...)` replays recorded draws instead, which is how the parity tests pin the state
machine bit-exactly against a trace of the unmodified reference.

Scaffold decoration (`scaffolds=(nodes, edges)`, `attachment=`, `set_scaffolds`): every slot but the dummy one starts
from a given partial graph instead of the empty one and restarts from the next scaffold in round-robin order when its
molecule terminates; `generated_scaffolds` says which scaffold each molecule grew from.  The action space only ever
appends, so the model, the sampler, the validity rules and the likelihood bookkeeping are unchanged: the likelihoods
cover the decoration actions.  With attachment points, adds and connects onto the other scaffold atoms, and connects
while the newest atom is still a scaffold atom, get logit -inf before the softmax (`ScaffoldTable`).

`GraphGeneratorRL` is the twin used by the reinforcement-learning loop (reference GraphGeneratorRL.py:25-172):
two models are evaluated on every round -- the sampling "agent" and a second model whose probability of the SAME
action is recorded -- and, unlike plain generation, autograd runs through the whole rollout
(`Workflow.learning_step`, Workflow.py:569-612, back-propagates a loss on the summed likelihoods).
"""
import ctypes

import numpy as np
import torch

from . import functional as Fn
from ._lib import Scaffolds, check, lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def action_layout(model, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None, n_chirality=None):
    """(constants, n_atom_types, n_formal_charge, n_imp_H, n_chirality) of a generator's layout arguments: each one
    not given comes from the constants (the model's by default); raises ValueError for a layout the constants'
    n_node_features and len_f_add_per_node do not fit"""
    C = constants if constants is not None else model.constants
    A = n_atom_types if n_atom_types is not None else getattr(C, "n_atom_types")
    CH = n_formal_charge if n_formal_charge is not None else getattr(C, "n_formal_charge")
    H = n_imp_H if n_imp_H is not None else getattr(C, "n_imp_H", 0)
    X = n_chirality if n_chirality is not None else getattr(C, "n_chirality", 0)
    counts = (A, CH, H, X)
    len_f_add = A * CH * max(H, 1) * max(X, 1) * C.n_edge_features
    if (min(A, CH) < 1 or min(H, X) < 0 or max(counts) > 255
            or sum(counts) != C.n_node_features or len_f_add != C.len_f_add_per_node):
        raise ValueError(
            f"inconsistent action layout: n_atom_types={A}, n_formal_charge={CH}, n_imp_H={H}, "
            f"n_chirality={X} (each <= 255; 0 = segment absent) need n_node_features = {sum(counts)} "
            f"and len_f_add_per_node = {len_f_add}, the constants have {C.n_node_features} and {C.len_f_add_per_node} "
            "(graphinvent_b200.config.layout_dims derives them from the reference's flags)")
    return C, A, CH, H, X


class ScaffoldTable:
    """The scaffolds a generator decorates, as the device table of `gib_scaffolds` (include/gib200.h).

    nodes int8 [S, N', F] / edges int8 [S, N', N', Ef]: scaffold s holds k_s >= 1 atoms in rows 0..k_s-1 (N' rows, the
    rows past the generator's N must be empty), in the format `preprocess.stacks` makes from `PreprocessingGraph`s.
    They are checked by the training-set construction's own kernels (`preprocess.groups`), which refuse, naming the
    first bad scaffold, a node row that is not one-hot per segment, a gap between atom rows, an edge entry that is not
    a symmetric single-type bond, no atoms, and a graph whose decoding route disconnects -- a disconnected graph, or
    one whose atom order the generator could not have produced, since every add bonds the new atom to an existing one.
    The whole pass runs, not only its count stage: the count kernel's status words are read back once per chunk, after
    the route stage, and that route stage is the check of the atom order.  For a scaffold set it is one chunk of a few
    route states per scaffold, so it costs one small launch sequence and one read when the scaffolds are set.

    attachment: None (nothing is masked; the scaffold may gain bonds anywhere), a bool [S, N'] array (True = an
    attachment point), or one list of atom indices per scaffold.  The other atoms of scaffold s are protected: bit i
    of `protect[s]` (4 x 32 bits, N <= 127)."""

    def __init__(self, nodes, edges, attachment, N, F, Ef, layout, device):
        from . import preprocess
        if attachment is not None and N > 127:
            raise ValueError(f"attachment points need max_n_nodes N <= 127 (4 x 32 protect bits per scaffold), "
                             f"got N = {N}")
        nodes = np.ascontiguousarray(torch.as_tensor(nodes).cpu().numpy())
        edges = np.ascontiguousarray(torch.as_tensor(edges).cpu().numpy())
        if (nodes.ndim != 3 or edges.ndim != 4 or nodes.shape[0] < 1 or nodes.shape[2] != F or edges.shape[3] != Ef
                or edges.shape[:3] != (nodes.shape[0], nodes.shape[1], nodes.shape[1])):
            raise ValueError(f"scaffolds must be int8 stacks nodes [S, N, {F}] / edges [S, N, N, {Ef}] with S >= 1, "
                             f"got {nodes.shape} / {edges.shape}")
        if nodes.dtype != np.int8 or edges.dtype != np.int8:
            if not (np.array_equal(nodes, nodes.astype(np.int8)) and np.array_equal(edges, edges.astype(np.int8))):
                raise ValueError("scaffold features are not int8-exact")
            nodes, edges = nodes.astype(np.int8), edges.astype(np.int8)
        S, rows = nodes.shape[:2]
        try:
            for _ in preprocess.groups(nodes, edges, 64, *layout, device=device):
                pass
        except ValueError as e:
            raise ValueError(f"invalid scaffold (molecule i below is scaffold i): {e}") from None
        k = (nodes != 0).any(-1).sum(-1).astype(np.int32)
        if int(k.max()) > N:
            s = int(np.argmax(k > N))
            raise ValueError(f"scaffold {s} holds {int(k[s])} atoms, the generator's max_n_nodes is {N}")
        if rows > N:
            nodes, edges = nodes[:, :N], edges[:, :N, :N]
        elif rows < N:
            nodes = np.pad(nodes, ((0, 0), (0, N - rows), (0, 0)))
            edges = np.pad(edges, ((0, 0), (0, N - rows), (0, N - rows), (0, 0)))
        self.S, self.N = S, N
        self.n_atoms = k
        self.n_bonds = (edges.reshape(S, -1).astype(np.int64).sum(1) // 2)
        self.m_max = int(self.n_bonds.max())
        self.protect_mask = None
        if attachment is not None:
            attach = np.zeros((S, N), bool)
            if isinstance(attachment, (list, tuple)):
                if len(attachment) != S:
                    raise ValueError(f"attachment lists {len(attachment)} scaffolds, there are {S}")
                for s, idx in enumerate(attachment):
                    idx = np.asarray(list(idx), np.int64)
                    if idx.size and (idx.min() < 0 or idx.max() >= k[s]):
                        raise ValueError(f"attachment point of scaffold {s} outside its atoms 0..{int(k[s]) - 1}")
                    attach[s, idx] = True
            else:
                a = np.asarray(torch.as_tensor(attachment).cpu().numpy(), bool)
                if a.ndim != 2 or a.shape[0] != S or a.shape[1] < min(rows, N):
                    raise ValueError(f"attachment must be a bool [S, N] array, got shape {a.shape}")
                attach[:, :min(a.shape[1], N)] = a[:, :N]
            self.protect_mask = (np.arange(N)[None] < k[:, None]) & ~attach
        dev = torch.device(device)
        self.nodes = torch.from_numpy(nodes).to(dev)
        self.edges = torch.from_numpy(edges).to(dev)
        self.n_atoms_dev = torch.from_numpy(k).to(dev)
        self.protect = None
        if self.protect_mask is not None:
            bits = np.zeros((S, 128), bool)
            bits[:, :N] = self.protect_mask
            words = (bits.reshape(S, 4, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
            self.protect = torch.from_numpy(words.astype(np.uint32).view(np.int32)).to(dev)

    def copy_(self, other):
        """`other`'s scaffolds into this table's buffers, in place (same S, attachment points given in both or in
        neither)"""
        self.nodes.copy_(other.nodes)
        self.edges.copy_(other.edges)
        self.n_atoms_dev.copy_(other.n_atoms_dev)
        if self.protect is not None:
            self.protect.copy_(other.protect)
        self.n_atoms, self.n_bonds, self.protect_mask = other.n_atoms, other.n_bonds, other.protect_mask

    def struct(self, slot_ids=None, started=None, gen_scaffolds=None):
        """the `gib_scaffolds` of this table and the per-batch state buffers (None: null, for the route scorer's
        entry points, which read only the table)"""
        return Scaffolds(nodes=_ptr(self.nodes), edges=_ptr(self.edges), n_atoms=_ptr(self.n_atoms_dev),
                         protect=_ptr(self.protect), slot_ids=_ptr(slot_ids), started=_ptr(started),
                         gen_scaffolds=_ptr(gen_scaffolds), S=self.S)


ACTION_MASK_MODES = {"structure": 1, "valence": 2}          # GIB_ACTION_MASK_* (include/gib200.h)
CONS_OFF = -1                                                   # a maximum's "off" value in the constraint table


def _bound(v, what, min_only=False, max_only=False):
    """(min, max) of a bound given as (min, max) (None = off) or, for a maximum-only field, as an int"""
    if v is None:
        return 0, CONS_OFF
    if isinstance(v, (int, np.integer)) and not isinstance(v, bool) and max_only:
        v = (None, int(v))
    try:
        lo, hi = v
    except (TypeError, ValueError):
        raise ValueError(f"{what} must be a (min, max) pair (None = no bound), got {v!r}") from None
    for x in (lo, hi):
        if x is not None and (isinstance(x, bool) or not isinstance(x, (int, np.integer)) or x < 0):
            raise ValueError(f"{what}: bounds are non-negative ints or None, got {v!r}")
    if max_only and lo not in (None, 0):
        raise ValueError(f"{what} has a maximum only, got a minimum of {lo}")
    lo, hi = int(lo or 0), CONS_OFF if hi is None else int(hi)
    if hi != CONS_OFF and lo > hi:
        raise ValueError(f"{what}: the minimum {lo} is over the maximum {hi}")
    return lo, hi


class Constraints:
    """What a generated molecule may contain, applied as a mask on the actions (`constraints=`; the rule is
    graphinvent_b200/csrc/constraints.cuh).  Each argument is optional; None is no bound:

        Constraints(atoms=(9, 13), atom_types={"N": (1, None), "S": (0, 0)}, charges={1: 0}, bonds={"TRIPLE": 0},
                    rings=(0, 2), min_ring_size=5)

    atoms / rings: (min, max) atom count / cycle rank (bonds - atoms + 1, the number of rings a route closes);
    atom_types: {type: (min, max)}; charges: {formal charge: max} and bonds: {bond type: max} (maxima only);
    min_ring_size: no ring shorter than this (>= 3), i.e. no connect that closes one.
    Keys are resolved through the reference's constants (`atom_types`, `formal_charge`, `int_to_bondtype`, or the bond
    names SINGLE / DOUBLE / TRIPLE / AROMATIC in that order without it); integer keys are indices when no constants
    are given (charge keys are formal charges when `constants.formal_charge` is there).  Maxima forbid the adds and
    connects that would pass them; minima forbid terminate while the molecule is below them, unless no other action
    is allowed (a dead end: the molecule then ends under its minimum).  Bad values raise ValueError here or, for those
    that depend on the layout (max_atoms over max_n_nodes, minima adding up past max_atoms), in `table`."""

    def __init__(self, atoms=None, atom_types=None, charges=None, bonds=None, rings=None, min_ring_size=None,
                 constants=None):
        self.atoms, self.rings = _bound(atoms, "atoms"), _bound(rings, "rings")
        self.atom_types = {k: _bound(v, f"atom_types[{k!r}]") for k, v in dict(atom_types or {}).items()}
        self.charges = {k: _bound(v, f"charges[{k!r}]", max_only=True)[1] for k, v in dict(charges or {}).items()}
        self.bonds = {k: _bound(v, f"bonds[{k!r}]", max_only=True)[1] for k, v in dict(bonds or {}).items()}
        m = 0 if min_ring_size is None else min_ring_size
        if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or m < 0 or m in (1, 2):
            raise ValueError(f"min_ring_size must be None / 0 (off) or an int >= 3, got {min_ring_size!r}")
        self.min_ring_size = int(m)
        self.constants = constants
        self._mask = None                                   # the ActionMask this set is bound to (check())

    def _key(self):
        return (self.atoms, self.rings, sorted(self.atom_types.items(), key=repr),
                sorted(self.charges.items(), key=repr), sorted(self.bonds.items(), key=repr), self.min_ring_size)

    def __eq__(self, other):
        return isinstance(other, Constraints) and self._key() == other._key()

    def __repr__(self):
        return (f"Constraints(atoms={self.atoms}, atom_types={self.atom_types}, charges={self.charges}, "
                f"bonds={self.bonds}, rings={self.rings}, min_ring_size={self.min_ring_size})")

    @property
    def off(self):
        """True when no field bounds anything (the mask is then the unconstrained one, bit for bit)"""
        return (self.atoms == (0, CONS_OFF) and self.rings == (0, CONS_OFF) and not self.min_ring_size
                and all(v == (0, CONS_OFF) for v in self.atom_types.values())
                and all(v == CONS_OFF for v in self.charges.values())
                and all(v == CONS_OFF for v in self.bonds.values()))

    def values(self, layout, N, n_edge_features, constants=None):
        """the table's words (int32 numpy, include/gib200.h GIB_CONS_*) for the layout (A, CH, H, C), max_n_nodes N and
        Ef bond types"""
        A, CH = int(layout[0]), int(layout[1])
        Ef = int(n_edge_features)
        C = self.constants if self.constants is not None else constants      # the set's own constants first
        t = np.zeros(8 + 2 * A + CH + Ef, np.int32)
        t[0], t[1] = self.atoms
        t[2], t[3] = self.rings
        t[4] = self.min_ring_size
        t[8 + A:8 + 2 * A] = CONS_OFF
        t[8 + 2 * A:] = CONS_OFF
        for k, (lo, hi) in self.atom_types.items():
            i = _index(k, "atom type", A, getattr(C, "atom_types", None))
            t[8 + i], t[8 + A + i] = lo, hi
        charges = getattr(C, "formal_charge", None)
        for k, hi in self.charges.items():
            t[8 + 2 * A + _index(k, "formal charge", CH, charges, by_value=charges is not None)] = hi
        names = _bond_names(C, Ef)
        for k, hi in self.bonds.items():
            key = k.upper() if isinstance(k, str) else k
            t[8 + 2 * A + CH + _index(key, "bond type", Ef, names)] = hi
        if t[1] != CONS_OFF and t[1] > N:
            raise ValueError(f"atoms: the maximum {int(t[1])} is over max_n_nodes = {N}")
        if t[0] > N:
            raise ValueError(f"atoms: the minimum {int(t[0])} is over max_n_nodes = {N}")
        cap = N if t[1] == CONS_OFF else int(t[1])
        if int(t[8:8 + A].sum()) > cap:
            raise ValueError(f"atom_types: the minima add up to {int(t[8:8 + A].sum())} atoms, more than "
                             f"{'max_n_nodes' if t[1] == CONS_OFF else 'the maximum atom count'} {cap}")
        return t

    def table(self, layout, N, device, n_edge_features=None, constants=None):
        """the device table (int32, written by `gib_constraints_set`, which checks it again) for the layout (A, CH, H,
        C), max_n_nodes N and n_edge_features bond types (default: `constants.n_edge_features`)"""
        C = self.constants if self.constants is not None else constants      # the set's own constants first
        Ef = n_edge_features if n_edge_features is not None else getattr(C, "n_edge_features", None)
        if Ef is None:
            raise ValueError("Constraints.table needs n_edge_features (or constants with n_edge_features)")
        vals = self.values(layout, N, Ef, C)
        out = torch.empty(vals.size, dtype=torch.int32, device=torch.device(device))
        check(lib.gib_constraints_set(_ptr(out), vals.ctypes.data_as(ctypes.c_void_p), int(N), int(layout[0]),
                                      int(layout[1]), int(Ef), torch.cuda.current_stream(out.device).cuda_stream),
              "gib_constraints_set")
        return out

    def check(self, nodes, edges, n_nodes=None, scaffold_ids=None):
        """int32 flags [M] on the device of finished molecules nodes [M, N, F] / edges [M, N, N, Ef] (float or int8,
        device tensors) with atom counts n_nodes [M] (None: the non-empty node rows), judged with the action mask of
        the generator or scorer this set belongs to (`gen.constraints.check(...)`): bit 1 over a maximum, 2 a ring
        shorter than min_ring_size, 4 under a minimum while another action was allowed (probability 0), 8 under a
        minimum at a dead end (allowed).  scaffold_ids [M]: the molecules' scaffolds, for the attachment points of a
        scaffold generator."""
        if self._mask is None:
            raise ValueError("this Constraints is not bound to a generator or scorer: use gen.constraints.check(...) "
                             "or make one with make_action_mask(..., constraints=)")
        return self._mask.check(nodes, edges, n_nodes, scaffold_ids)


def _index(k, what, n, names, by_value=False):
    """index of key k among n entries: a name (or a value, by_value) looked up in `names`, or an int index"""
    if names is not None and (by_value or isinstance(k, str)):
        lst = [str(x) if isinstance(k, str) else x for x in names]
        if k not in lst:
            raise ValueError(f"unknown {what} {k!r} (the constants list {list(names)})")
        i = lst.index(k)
    elif isinstance(k, (int, np.integer)) and not isinstance(k, bool):
        i = int(k)
    else:
        raise ValueError(f"{what} {k!r}: names need constants; give an integer index instead")
    if not 0 <= i < n:
        raise ValueError(f"{what} index {i} outside the layout's 0..{n - 1}")
    return i


def _bond_names(C, Ef):
    from .config import _bond_name
    itb = getattr(C, "int_to_bondtype", None)
    if itb is not None and len(itb) == Ef:
        return [_bond_name(itb[i]) for i in range(Ef)]
    return ["SINGLE", "DOUBLE", "TRIPLE", "AROMATIC"][:Ef] if Ef <= 4 else None


class ActionMask:
    """The action mask of a generator or route scorer (`action_mask=`, `gib_action_mask_logits`): logit -inf for
    every action the round would reject as invalid in the slot's state ("structure": a bond to an atom that does not
    exist, a self loop, a bond that exists, an add into a full graph, ...), and with "valence" also every bond that
    takes an atom past its limit in the table of `config.action_rule_table(max_valence=...)`.  Terminate is never
    masked.  The rule is graphinvent_b200/csrc/action_mask.cuh, the one the round's decode kernel flags invalid
    actions with.

    With `constraints` (a `Constraints`) the constraint rule runs in the same launch
    (`gib_action_mask_logits_constrained`), from a device table that `set_constraints` rewrites in place: its minima
    are the only rule that masks terminate."""

    def __init__(self, mode, max_valence, constants, layout, N, F, Ef, apd, device, constraints=None):
        if mode not in ACTION_MASK_MODES:
            raise ValueError(f"action_mask must be None, 'structure' or 'valence', got {mode!r}")
        if max_valence is not None and mode != "valence":
            raise ValueError("max_valence is read by action_mask='valence' only")
        if N > 127:
            raise ValueError(f"the action mask needs max_n_nodes N <= 127, got N = {N}")
        from .config import action_rule_table
        self.mode, self.code = mode, ACTION_MASK_MODES[mode]
        self.layout, self.N, self.F, self.Ef, self.apd = tuple(layout), N, F, Ef, apd
        self.constants, self.device = constants, torch.device(device)
        self.valence, self.bond_orders, self.imp_h, self.table = None, None, None, None
        if mode == "valence":
            A, CH, H, _ = layout
            self.valence, self.bond_orders, self.imp_h = action_rule_table(A, CH, Ef, H, max_valence, constants)
            flat = np.concatenate([self.valence.ravel(), self.bond_orders, self.imp_h]).astype(np.int32)
            self.table = torch.from_numpy(flat).to(torch.device(device))
        self.constraints, self.cons_table = None, None
        if constraints is not None:
            self.set_constraints(constraints)

    def set_constraints(self, constraints):
        """`constraints` into the device table, in place (allocated by the first call)"""
        if not isinstance(constraints, Constraints):
            raise TypeError(f"constraints must be a generation.Constraints, got {type(constraints).__name__}")
        vals = constraints.values(self.layout, self.N, self.Ef, self.constants)
        if self.cons_table is None:
            self.cons_table = torch.zeros(vals.size, dtype=torch.int32, device=self.device)
        check(lib.gib_constraints_set(_ptr(self.cons_table), vals.ctypes.data_as(ctypes.c_void_p), self.N,
                                      self.layout[0], self.layout[1], self.Ef,
                                      torch.cuda.current_stream(self.device).cuda_stream), "gib_constraints_set")
        bound = Constraints.__new__(Constraints)
        bound.__dict__.update(constraints.__dict__)
        bound._mask = self
        if bound.constants is None:
            bound.constants = self.constants
        self.constraints = bound

    def apply(self, B, logits, n_nodes, stream, nodes=None, edges=None, int8=False, sc=None, slot_ids=None, row=None,
              state=None, counters=None, first_slot=1):
        """-inf in place into logits [B, apd]; nodes / edges float (int8=False) or int8 [B, ...]; sc (a gib_scaffolds
        with attachment points) and slot_ids: that rule too, in the same launch"""
        fl = (_ptr(nodes), _ptr(edges), None, None) if not int8 else (None, None, _ptr(nodes), _ptr(edges))
        args = (B, self.N, self.F, self.Ef, *self.layout, self.apd, self.code, _ptr(self.table), *fl, _ptr(n_nodes),
                ctypes.byref(sc) if sc is not None else None, _ptr(slot_ids), _ptr(row), _ptr(state), _ptr(counters),
                _ptr(logits), first_slot, stream)
        if self.cons_table is not None:
            check(lib.gib_action_mask_logits_constrained(*args, _ptr(self.cons_table)),
                  "gib_action_mask_logits_constrained")
        else:
            check(lib.gib_action_mask_logits(*args), "gib_action_mask_logits")

    def check(self, nodes, edges, n_nodes=None, scaffold_ids=None, sc=None, out=None, stream=None):
        """`gib_constraints_check` of finished molecules: int32 flags [M] on the device (`Constraints.check`)"""
        if self.cons_table is None:
            raise ValueError("no constraints are set")
        M = nodes.shape[0]
        if (not (nodes.is_cuda and edges.is_cuda) or nodes.dtype != edges.dtype
                or nodes.dtype not in (torch.float32, torch.int8)
                or tuple(nodes.shape[1:]) != (self.N, self.F) or tuple(edges.shape) != (M, self.N, self.N, self.Ef)):
            raise ValueError(f"nodes / edges must be float32 or int8 device tensors [M, {self.N}, {self.F}] / "
                             f"[M, {self.N}, {self.N}, {self.Ef}], got {nodes.dtype} {tuple(nodes.shape)} / "
                             f"{edges.dtype} {tuple(edges.shape)}")
        nodes, edges = nodes.contiguous(), edges.contiguous()
        cnt = n_nodes.to(device=nodes.device, dtype=torch.int32).contiguous() if n_nodes is not None else None
        ids = None
        if scaffold_ids is not None:
            ids = torch.as_tensor(scaffold_ids).to(device=nodes.device, dtype=torch.int32).contiguous()
        flags = out if out is not None else torch.zeros(M, dtype=torch.int32, device=nodes.device)
        i8 = nodes.dtype == torch.int8
        fl = (None, None, _ptr(nodes), _ptr(edges)) if i8 else (_ptr(nodes), _ptr(edges), None, None)
        st = stream if stream is not None else torch.cuda.current_stream(nodes.device).cuda_stream
        check(lib.gib_constraints_check(M, self.N, self.F, self.Ef, *self.layout, self.code, _ptr(self.table), *fl,
                                        _ptr(cnt), ctypes.byref(sc) if sc is not None else None,
                                        _ptr(ids) if sc is not None else None, _ptr(self.cons_table), _ptr(flags), st),
              "gib_constraints_check")
        return flags


def _mask_logits(action_mask, logits, stream, nodes, edges, n_nodes, sc=None, slot_ids=None, int8=False, row=None,
                 state=None, counters=None, first_slot=1):
    """-inf in place into logits [B, apd]: `action_mask.apply`, or without one the attachment points of sc / slot_ids
    alone by `gib_generation_mask_logits` (first_slot 1) or `gib_route_mask_logits` (0; no row or gate)"""
    if action_mask is not None:
        return action_mask.apply(logits.shape[0], logits, n_nodes, stream, nodes, edges, int8, sc, slot_ids, row,
                                 state, counters, first_slot)
    B, apd = logits.shape
    name, gate = ("gib_generation_mask_logits", (row, state, counters)) if first_slot else ("gib_route_mask_logits", ())
    check(getattr(lib, name)(B, edges.shape[1], edges.shape[3], apd, ctypes.byref(sc), _ptr(slot_ids), _ptr(n_nodes),
                             *map(_ptr, gate), _ptr(logits), stream), name)


def make_action_mask(mode, max_valence, constants, layout, N, F, Ef, apd, device, constraints=None):
    """the ActionMask of a constructor's `action_mask=` / `max_valence=` / `constraints=` (None when all are None).
    Constraints without an action mask bring the structural rule with them: once a minimum masks terminate, the
    probability has to go to actions the round accepts, not to ones it would end as invalid."""
    if constraints is not None and not isinstance(constraints, Constraints):
        raise TypeError(f"constraints must be a generation.Constraints, got {type(constraints).__name__}")
    if mode is None:
        if max_valence is not None:
            raise ValueError("max_valence needs action_mask='valence'")
        if constraints is None:
            return None
        mode = "structure"
    return ActionMask(mode, max_valence, constants, layout, N, F, Ef, apd, device, constraints)


class _LogitMasks:
    """The logit masks of a generator or the route scorer: `action_mask` (rebuilt from `_mask_args`), `scaffolds`"""

    @property
    def constraints(self):
        """the constraint set of the following batches or scores (`Constraints`, bound to the mask for `check`)"""
        return self.action_mask.constraints if self.action_mask is not None else None

    def set_constraints(self, constraints=None):
        """the constraint set of the following batches or scores (None: none); rebuilds the mask if it has no table"""
        if constraints is not None and self.action_mask is not None and self.action_mask.cons_table is not None:
            self.action_mask.set_constraints(constraints)
        else:
            self.action_mask = make_action_mask(*self._mask_args, constraints)
            self._masks_rebuilt()
        self.constraints_version += 1

    def _masks_rebuilt(self):
        """the action mask object was replaced (captured objects capture again)"""

    @property
    def masked(self):
        """True when the scaffolds' attachment points restrict the actions"""
        return self.scaffolds is not None and self.scaffolds.protect is not None


def scaffold_table(scaffolds, attachment, N, F, Ef, layout, device):
    """the ScaffoldTable of `set_scaffolds`' arguments (None for None), for the generators and the route scorer"""
    if scaffolds is None:
        if attachment is not None:
            raise ValueError("attachment points need scaffolds")
        return None
    nodes, edges = scaffolds
    return ScaffoldTable(nodes, edges, attachment, N, F, Ef, layout, device)


class GraphGenerator(_LogitMasks):
    """`scaffolds=(nodes, edges)` / `attachment=`: decorate those scaffolds instead of growing molecules from the empty
    graph (`ScaffoldTable`; `set_scaffolds` changes them).  None (the default) keeps the reference's behaviour.

    `action_mask="structure"` / `"valence"` (`ActionMask`): sample only actions the round accepts, from the model's
    softmax renormalised over them; `max_valence=` overrides the valence table (`config.action_rule_table`).  With
    attachment points too, one launch applies both rules.

    `temperature=`, `top_k=`, `top_p=` (`functional.SamplingPolicy`; `set_sampling` changes them, `sampling` reads
    them): draw each action from the model's softmax at that temperature, cut to the top_k most likely actions and to
    the smallest set of them holding top_p of their probability (after the masks).  Only the draw changes: the
    recorded likelihoods stay the model's probabilities of the drawn actions.  The default (1, 0, 1) is the model's
    softmax itself.  In `GraphGeneratorRL` the policy applies to the agent's draw.

    `constraints=` (`Constraints`; `set_constraints` changes them, `constraints` reads them): sample only molecules
    within atom-count, element, charge, bond-type and ring budgets -- the maxima mask the actions that would pass them,
    the minima mask terminate while a molecule is below them, unless nothing else is allowed.  Without `action_mask=`
    the structural rule comes with them.  The likelihoods stay the model's masked-softmax probabilities, and the
    sampling policy acts after all masks.  `gen.constraints.check(nodes, edges, n_nodes)` flags finished molecules."""

    def __init__(self, model, batch_size, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None,
                 n_chirality=None, device="cuda", scaffolds=None, attachment=None, action_mask=None,
                 max_valence=None, temperature=1.0, top_k=0, top_p=1.0, constraints=None):
        self._sampling = Fn.sampling_policy(temperature, top_k, top_p)
        C, self.A, self.CH, self.n_imp_H, self.n_chirality = action_layout(
            model, constants, n_atom_types, n_formal_charge, n_imp_H, n_chirality)
        self.constants = C
        self.model, self.batch_size, self.device = model, int(batch_size), torch.device(device)
        self.N, self.F, self.Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
        self.apd = self.N * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
        self.rounds = 0
        self.scaffolds = None
        self.generated_scaffolds = None
        self._mask_args = (action_mask, max_valence, C, self.layout, self.N, self.F, self.Ef, self.apd, self.device)
        self.constraints_version = 0
        self.action_mask = make_action_mask(*self._mask_args, constraints)
        self._allocate()
        if scaffolds is not None:
            self.set_scaffolds(scaffolds, attachment)

    @property
    def layout(self):
        return (self.A, self.CH, self.n_imp_H, self.n_chirality)

    @property
    def sampling(self):
        """the sampling policy of the draws (`functional.SamplingPolicy`)"""
        return self._sampling

    def set_sampling(self, temperature=1.0, top_k=0, top_p=1.0):
        """the sampling policy of the following draws; raises ValueError naming an argument out of range"""
        self._sampling = Fn.sampling_policy(temperature, top_k, top_p)

    def _policy_kw(self):
        """the policy arguments of the draw: none when it is off, so the draw is today's call"""
        return {} if self._sampling == Fn.SAMPLING_OFF else self._sampling._asdict()

    def _table(self, scaffolds, attachment):
        """the ScaffoldTable of set_scaffolds' arguments (None for None)"""
        return scaffold_table(scaffolds, attachment, self.N, self.F, self.Ef, self.layout, self.device)

    def set_scaffolds(self, scaffolds, attachment=None):
        """decorate `scaffolds` = (nodes, edges) from the next batch on (None: grow from the empty graph again)"""
        self.scaffolds = self._table(scaffolds, attachment)
        self._allocate()

    def _scaffold_struct(self):
        return self.scaffolds.struct(self._slot_ids, self._started, self._gen_scaffolds)

    def _scaffold_init(self, stream):
        """the scaffold start state of slots 1..B-1 (gib_generation_scaffold_init)"""
        self._sc = self._scaffold_struct()
        check(lib.gib_generation_scaffold_init(self.batch_size, self.N, self.F, self.Ef, ctypes.byref(self._sc),
                                               _ptr(self.nodes), _ptr(self.edges), _ptr(self.n_nodes),
                                               _ptr(self.likelihoods), stream), "gib_generation_scaffold_init")

    def _mask(self, logits, stream):
        """-inf into logits [B, apd] (in place) where this round's state makes the masks forbid an action"""
        sc, ids = (self._sc, self._slot_ids) if self.masked else (None, None)
        _mask_logits(self.action_mask, logits, stream, self.nodes, self.edges, self.n_nodes, sc, ids)

    @property
    def masks_logits(self):
        """True when the round's logits are masked: attachment points or the action mask"""
        return self.masked or self.action_mask is not None

    def _allocate(self):
        B, N, F, Ef, dev = self.batch_size, self.N, self.F, self.Ef, self.device
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        # initialize_graph_batch (GraphGenerator.py:387-423): empty graphs + the dummy graph in slot 0
        self.nodes, self.edges = z(B, N, F), z(B, N, N, Ef)
        self.n_nodes = z(B, dt=torch.int32)
        self.nodes[0] = 1.0
        self.edges[0, 0, 0, 0] = 1.0
        self.n_nodes[0] = 1
        # allocate_graph_tensors (:163-209): finished-graph buffers with one extra batch of slack
        cap = 2 * B
        self.capacity = cap
        self.generated_nodes, self.generated_edges = z(cap, N, F), z(cap, N, N, Ef)
        self.generated_n_nodes = z(cap, dt=torch.int8)
        self.likelihoods, self.generated_likelihoods = z(B, 2 * N), z(cap, 2 * N)
        self.properly_terminated = z(cap, dt=torch.int8)     # must start zeroed: the rounds only set flags to 1
        self._counters = z(2, dt=torch.int32)
        self._scratch = torch.empty(lib.gib_generation_scratch_bytes(B), dtype=torch.uint8, device=dev)
        if getattr(self, "scaffolds", None) is not None:
            self._slot_ids, self._started = z(B, dt=torch.int32), z(1, dt=torch.int32)
            self._gen_scaffolds = torch.full((cap,), -1, dtype=torch.int32, device=dev)
            self._scaffold_init(torch.cuda.current_stream(dev).cuda_stream)

    def _round(self, rnd, action, lik, stream):
        """one round of the device state machine; the gdb13 layout goes through `gib_generation_round`"""
        state = (_ptr(action), _ptr(lik), _ptr(self.nodes), _ptr(self.edges), _ptr(self.n_nodes), _ptr(self.likelihoods),
                 _ptr(self.generated_nodes), _ptr(self.generated_edges), _ptr(self.generated_n_nodes),
                 _ptr(self.generated_likelihoods), _ptr(self.properly_terminated), self.capacity, _ptr(self._counters),
                 _ptr(self._scratch), stream)
        if self.scaffolds is not None:
            check(lib.gib_generation_round_scaffold(self.batch_size, self.N, self.F, self.Ef, self.A, self.CH,
                                                    self.n_imp_H, self.n_chirality, ctypes.byref(self._sc), rnd,
                                                    *state), "gib_generation_round_scaffold")
        elif self.n_imp_H == 0 and self.n_chirality == 0:
            check(lib.gib_generation_round(self.batch_size, self.N, self.F, self.Ef, self.A, self.CH, rnd, *state),
                  "gib_generation_round")
        else:
            check(lib.gib_generation_round_layout(self.batch_size, self.N, self.F, self.Ef, self.A, self.CH,
                                                  self.n_imp_H, self.n_chirality, rnd, *state),
                  "gib_generation_round_layout")

    def _model_inputs(self, model):
        """(nodes, edges) to evaluate `model` on.  The dummy graph in slot 0 is never reset (GraphGenerator.py:461-465
        re-arms nodes / n_nodes only) and accumulates every action it samples: two "add" actions with different bond
        types leave a bond with two non-zero types there.  The reference's AggregationMPNN / EMN prologues then fail
        with a shape mismatch (aggregation_mpnn.py:115-141, edge_mpnn.py:123-156) and the whole generation run dies;
        AttentionGGNN here rejects such input too.  Nothing ever reads the dummy slot's output, so for that model the
        dummy graph is evaluated with the first non-zero type of each bond only (a copy: the state machine keeps the
        reference's state of slot 0 bit for bit)."""
        if getattr(model, "MODEL", None) != "AttGGNN":
            return self.nodes, self.edges
        e0 = self.edges[0]
        nz = e0 != 0
        edges = self.edges.clone()
        edges[0] = e0 * (nz & (nz.to(torch.int32).cumsum(-1) == 1)).to(e0.dtype)
        return self.nodes, edges

    @torch.no_grad()
    def build_graphs(self, replay=None, generator=None):
        """replay: optional iterable of (action int32 [B], likelihood float32 [B]) per round (the model is then not
        evaluated); returns the number of finished molecules (may exceed batch_size, as in the reference)."""
        B = self.batch_size
        if self.rounds or int(self._counters[0].item()):
            self._allocate()          # a generator object can be used again: start from a fresh batch (:387-423)
        n_generated, rnd = 0, 0
        replay = iter(replay) if replay is not None else None
        st = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        while n_generated < B:
            if rnd >= 2 * self.N:
                raise RuntimeError("generation needs more than 2*max_n_nodes rounds: the per-slot likelihood buffer "
                                   "(GraphGenerator.py:173, 'the 2 is arbitrary') would overflow, as in the reference")
            if replay is not None:
                try:
                    action, lik = next(replay)
                except StopIteration:
                    raise RuntimeError("replay trace ended before batch_size molecules were finished") from None
                action = action.to(self.device, torch.int32).contiguous()
                lik = lik.to(self.device, torch.float32).contiguous()
            else:
                out = self.model(*self._model_inputs(self.model))    # GraphGenerator.py:121
                if self.masks_logits:
                    out = out.contiguous()
                    self._mask(out, st)
                action, lik = Fn.sample_actions(out, generator=generator, **self._policy_kw())
            self._round(rnd, action, lik, st)
            n_generated = int(self._counters[0].item())           # the loop condition lives on the host (:118)
            rnd += 1
        self.rounds = rnd
        self._keep_scaffold_ids()
        return n_generated

    def _keep_scaffold_ids(self):
        self.generated_scaffolds = (self._gen_scaffolds[:self.batch_size].clone() if self.scaffolds is not None
                                    else None)

    def sample(self, generator=None):
        """returns (generated_nodes, generated_edges, generated_n_nodes) of the first batch_size finished molecules,
        the non-zero per-action likelihoods, log(sum of likelihoods) per molecule and the properly-terminated flags
        (GraphGenerator.sample :48-96 without the RDKit conversion)."""
        self.build_graphs(generator=generator)
        B = self.batch_size
        final = torch.log(self.generated_likelihoods.sum(dim=1)[:B])              # :81-83
        flat = self.generated_likelihoods[self.generated_likelihoods != 0]        # :86-88
        graphs = (self.generated_nodes[:B], self.generated_edges[:B], self.generated_n_nodes[:B])
        return graphs, flat, final, self.properly_terminated[:B]

    def sample_molecules(self, *args, constants=None, **kw):
        """what the reference's `sample()` returns (GraphGenerator.py:48-96, GraphGeneratorRL.py:53-107): `sample(*args,
        **kw)` of this generator with its tensors turned into the reference's `GenerationGraph` list by one
        `molecules.MoleculeBatch`, which stays at `self.molecules` for `self.molecules.properties(...)` (the Analyzer's
        statistics of the same batch).  `constants`: the reference constants the molecules are read with (atom_types,
        formal_charge, int_to_bondtype, ...), by default those the generator was built with.  The likelihood tensors
        are those of `sample()`, autograd history included."""
        from .molecules import MoleculeBatch
        (nodes, edges, n_nodes), likelihoods_a, likelihoods_b, terminated = self.sample(*args, **kw)
        self.molecules = MoleculeBatch(nodes, edges, n_nodes, constants if constants is not None else self.constants)
        return self.molecules.generation_graphs(), likelihoods_a, likelihoods_b, terminated


class GraphGeneratorRL(GraphGenerator):
    """RL rollout (reference `GraphGeneratorRL`): `sample(agent_model, prior_model)` returns the finished tensors,
    `log(sum_t p_agent(a_t))` and `log(sum_t p_prior(a_t))` per molecule (GraphGeneratorRL.py:92-97) and the
    properly-terminated flags; both log-likelihood vectors are differentiable w.r.t. the parameters of their model.

    How the two differentiable likelihood streams ride on the one-stream round kernel: the kernel is given the slot
    id (b + 1, exact in fp32) as the "likelihood" of every slot, so that after the rollout
    `generated_likelihoods[g, t]` names the slot whose round-t action belongs to finished molecule g (0 = none).
    The per-round sampled probabilities `softmax(logits_t)[b, a_t[b]]` are kept as autograd tensors and gathered
    through that map -- the same values the reference scatters with in-place index assignments
    (GraphGeneratorRL.py:325-326, 357-358, 409-424), without ~30 indexed autograd ops per round.
    One K0 (bond lists + CSR) per round is shared by both models (SURVEY.md 8f rank 4)."""

    def __init__(self, model, batch_size, **kw):
        super().__init__(model, batch_size, **kw)
        self.generated_scaffolds = None
        self.generated_agent_likelihoods = None
        self.generated_prior_likelihoods = None

    def build_graphs(self, agent_model=None, prior_model=None, replay=None, generator=None):
        """replay: optional iterable of int32 [B] flat APD indices per round (instead of sampling from the agent).
        Gradients are recorded if autograd is enabled and the models' parameters require them."""
        agent = agent_model if agent_model is not None else self.model
        prior = prior_model if prior_model is not None else self.model
        B, N = self.batch_size, self.N
        if B + 1 >= 1 << 24:
            raise ValueError("batch_size must stay below 2**24 (slot ids travel as fp32)")
        self._allocate()                                    # a fresh rollout (the reference builds a new generator)
        tags = torch.arange(1, B + 1, dtype=torch.float32, device=self.device)
        fused = [hasattr(m, "dims") for m in (agent, prior)]      # this package's modules take a shared K0
        share = all(fused) and type(agent) is type(prior) and Fn.dims_key(agent, B) == Fn.dims_key(prior, B)
        lik_a, lik_p = [], []
        n_generated, rnd = 0, 0
        replay = iter(replay) if replay is not None else None
        st = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        while n_generated < B:
            if rnd >= 2 * N:
                raise RuntimeError("generation needs more than 2*max_n_nodes rounds: the per-slot likelihood buffer "
                                   "(GraphGeneratorRL.py:175, 'the 2 is arbitrary') would overflow, as in the reference")
            # the round kernel edits the batch in place while autograd keeps the inputs of every round: snapshot them
            nodes_in, edges_in = self.nodes.clone(), self._model_inputs(agent)[1].clone()
            if getattr(prior, "MODEL", None) == "AttGGNN" and getattr(agent, "MODEL", None) != "AttGGNN":
                edges_in = self._model_inputs(prior)[1].clone()
            graph = Fn.build_graph(agent, edges_in) if share else None
            out_a = agent(nodes_in, edges_in, graph=graph) if share else agent(nodes_in, edges_in)   # GraphGeneratorRL.py:131-132
            out_p = prior(nodes_in, edges_in, graph=graph) if share else prior(nodes_in, edges_in)
            if self.masks_logits:                # the masks as a detached 0 / -inf bias: both softmaxes renormalise
                bias = torch.zeros(B, self.apd, dtype=torch.float32, device=self.device)
                self._mask(bias, st)
                out_a, out_p = out_a + bias, out_p + bias
            if replay is not None:
                try:
                    action = next(replay)
                except StopIteration:
                    raise RuntimeError("replay trace ended before batch_size molecules were finished") from None
                action = action.to(self.device, torch.int32).contiguous()
            else:
                action, _ = Fn.sample_actions(out_a.detach(), generator=generator, **self._policy_kw())
            idx = action.long().unsqueeze(1)
            lik_a.append(torch.softmax(out_a, dim=1).gather(1, idx).squeeze(1))       # `apds[apd_one_hot == 1]` :547-548
            lik_p.append(torch.softmax(out_p, dim=1).gather(1, idx).squeeze(1))
            self._round(rnd, action, tags, st)
            n_generated = int(self._counters[0].item())
            rnd += 1
        self.rounds = rnd
        # (finished molecule, round) -> slot map written by the kernel; gather both likelihood streams through it
        owner = self.generated_likelihoods[:, :rnd]                                     # [2B, rounds] slot id + 1
        mask = (owner > 0).to(torch.float32)
        slot = (owner.long() - 1).clamp_(min=0).t().contiguous()                        # [rounds, 2B]
        pad = self.generated_likelihoods.shape[1] - rnd
        for name, rounds_l in (("generated_agent_likelihoods", lik_a), ("generated_prior_likelihoods", lik_p)):
            per_round = torch.stack(rounds_l)                                           # [rounds, B], differentiable
            g = per_round.gather(1, slot).t() * mask                                    # [2B, rounds]
            setattr(self, name, torch.nn.functional.pad(g, (0, pad)))                   # [2B, 2N] like the reference
        self._keep_scaffold_ids()
        return n_generated

    def sample(self, agent_model, prior_model, generator=None, replay=None):
        self.build_graphs(agent_model, prior_model, replay=replay, generator=generator)
        B = self.batch_size
        agent_ll = torch.log(torch.sum(self.generated_agent_likelihoods, dim=1)[:B])   # GraphGeneratorRL.py:92-94
        prior_ll = torch.log(torch.sum(self.generated_prior_likelihoods, dim=1)[:B])   # :95-97
        graphs = (self.generated_nodes[:B], self.generated_edges[:B], self.generated_n_nodes[:B])
        return graphs, agent_ll, prior_ll, self.properly_terminated[:B]
