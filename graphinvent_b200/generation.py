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

`GraphGeneratorRL` is the twin used by the reinforcement-learning loop (reference GraphGeneratorRL.py:25-172):
two models are evaluated on every round -- the sampling "agent" and a second model whose probability of the SAME
action is recorded -- and, unlike plain generation, autograd runs through the whole rollout
(`Workflow.learning_step`, Workflow.py:569-612, back-propagates a loss on the summed likelihoods).
"""
import ctypes

import torch

from . import functional as Fn
from ._lib import check, lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


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


class GraphGenerator:
    def __init__(self, model, batch_size, constants=None, n_atom_types=None, n_formal_charge=None, n_imp_H=None,
                 n_chirality=None, device="cuda"):
        C, self.A, self.CH, self.n_imp_H, self.n_chirality = action_layout(
            model, constants, n_atom_types, n_formal_charge, n_imp_H, n_chirality)
        self.constants = C
        self.model, self.batch_size, self.device = model, int(batch_size), torch.device(device)
        self.N, self.F, self.Ef = C.max_n_nodes, C.n_node_features, C.n_edge_features
        self.apd = self.N * (C.len_f_add_per_node + C.len_f_conn_per_node) + 1
        self.rounds = 0
        self._allocate()

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

    def _round(self, rnd, action, lik, stream):
        """one round of the device state machine; the gdb13 layout goes through `gib_generation_round`"""
        state = (_ptr(action), _ptr(lik), _ptr(self.nodes), _ptr(self.edges), _ptr(self.n_nodes), _ptr(self.likelihoods),
                 _ptr(self.generated_nodes), _ptr(self.generated_edges), _ptr(self.generated_n_nodes),
                 _ptr(self.generated_likelihoods), _ptr(self.properly_terminated), self.capacity, _ptr(self._counters),
                 _ptr(self._scratch), stream)
        if self.n_imp_H == 0 and self.n_chirality == 0:
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
                action, lik = Fn.sample_actions(out, generator=generator)
            self._round(rnd, action, lik, st)
            n_generated = int(self._counters[0].item())           # the loop condition lives on the host (:118)
            rnd += 1
        self.rounds = rnd
        return n_generated

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
            if replay is not None:
                try:
                    action = next(replay)
                except StopIteration:
                    raise RuntimeError("replay trace ended before batch_size molecules were finished") from None
                action = action.to(self.device, torch.int32).contiguous()
            else:
                action, _ = Fn.sample_actions(out_a.detach(), generator=generator)
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
        return n_generated

    def sample(self, agent_model, prior_model, generator=None, replay=None):
        self.build_graphs(agent_model, prior_model, replay=replay, generator=generator)
        B = self.batch_size
        agent_ll = torch.log(torch.sum(self.generated_agent_likelihoods, dim=1)[:B])   # GraphGeneratorRL.py:92-94
        prior_ll = torch.log(torch.sum(self.generated_prior_likelihoods, dim=1)[:B])   # :95-97
        graphs = (self.generated_nodes[:B], self.generated_edges[:B], self.generated_n_nodes[:B])
        return graphs, agent_ll, prior_ll, self.properly_terminated[:B]
