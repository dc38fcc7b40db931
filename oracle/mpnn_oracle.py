"""
CPU oracle for the GraphINVENT MPNN hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline legs may
import this file.  Nothing under `graphinvent_b200/` imports it; the product path
raises if its CUDA library is missing instead of falling back to this code.

What it is: a restatement, in plain PyTorch CPU ops, of the algorithm the
reference runs for `model(nodes, edges)` (forward) -- the arithmetic of this path
lives in the third-party dependency PyTorch (reference pins pytorch=1.8.0,
`environments/graphinvent.yml:95`; this image has 2.11.0), so the oracle uses the
same ATen ops (`nonzero`, `matmul`, `addmm`, `elu`/SELU, `softmax`, GRU gates) at
the same call sites.  It is written functionally over a `state_dict` whose keys
and shapes equal the reference's (`SURVEY.md` Appendix A), so the reference's
checkpoints and the drop-in modules' parameters feed it unchanged.  Backward is
PyTorch autograd through these ops, exactly as in the reference
(`Workflow.py:794`).

Parity pin: the reference ships no tests and no golden vectors, so the oracle is
pinned against the reference itself, as `__graft_entry__.build()` installs its modules
into `oracle/_ref/`: `tests/golden/make_golden.py` runs the unmodified reference modules
and writes the fixtures under `tests/golden/`; `tests/test_oracle.py` checks this file
against those fixtures and against the reference's pretrained checkpoint.

The restatement deliberately keeps the reference's cost profile where it is part
of the algorithm (dense V x E summation matrix, all edge-type MLPs evaluated on
all edges, padded neighbour tensors), because `bench.py --impl reference` times
this code as the reference's CPU path.

Each function cites the reference file:line it follows (paths relative to
`/root/reference/graphinvent/`).
"""
from collections import OrderedDict, namedtuple

import torch
import torch.nn.functional as F

BIG = 1e6  # constants.big_positive / -big_negative (parameters/defaults.py)


# --------------------------------------------------------------------------- #
# hyper-parameter tuple (the subset of `constants` the hot path reads, SURVEY §5)
# --------------------------------------------------------------------------- #
def make_constants(model="GGNN", **kw):
    """Build the namedtuple the reference constructors read (SURVEY §5 config row,
    `parameters/defaults.py:145-433` for the default values).  Contains every field
    any of MNN / GGNN / AttentionGGNN / EMN touches, so one tuple serves the
    reference classes, the oracle and the drop-in modules alike."""
    d = dict(
        model=model, device="cpu", big_positive=BIG, big_negative=-BIG,
        n_node_features=8, n_edge_features=3, max_n_nodes=13,
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
        edge_emb_size=100, edge_emb_hidden_dim=250, edge_emb_depth=4,
        edge_emb_dropout_p=0.0,
    )
    d.update(kw)
    # EdgeMPNN.__init__ reads two names defaults.py never defines (SURVEY §2 note b)
    d.setdefault("edge_features", d["n_edge_features"])
    d.setdefault("edge_embedding_size", d["edge_emb_size"])
    return namedtuple("constants", sorted(d))(**d)


# --------------------------------------------------------------------------- #
# building blocks
# --------------------------------------------------------------------------- #
# Conditioning probe (tests only).  The path is NOT differentiable everywhere: SELU'(x) jumps from
# 1.05 to 1.76 at x = 0 and, for molecules without any bonded atom, `energies - 1e6` is rounded to
# multiples of 1/16 in fp32.  Two fp32 evaluations that differ by rounding noise (~1e-6) can land on
# different sides of such a point; the reference's own fp32-vs-fp64 gradients differ by up to 7e-3
# for that reason (DESIGN.md "numerical conditioning").  When MARGINS is a list, every SELU input and
# every masked energy records its distance to the nearest discontinuity, so tests can pick inputs
# that are provably away from them and demand the strict tolerance there.
MARGINS = None


# SELU-kink probe (tests only).  KINK = (tau, side): the derivative of every SELU whose input lies within tau of 0 is
# forced to its right ('R': scale) or left ('L': scale*alpha) limit in the backward pass; the forward values are
# untouched (SELU is continuous).  The difference between the two fp64 gradients is the total effect the units
# inside the band can have on a gradient -- what two correct fp32 evaluations may legitimately disagree by when their
# rounding noise puts some of those inputs on different sides of 0.
KINK = None
_SELU_SCALE, _SELU_ALPHA = 1.0507009873554804934193349852946, 1.6732632423543772848170429916717


# Operand-rounding probe (tests only).  OPERANDS = "tf32" | "bf16" | "fp16": every product the package runs on its GEMM
# kernels -- each Linear of `mlp`, both Linears of `gru_cell` and the MNN message product -- takes its operands rounded
# the way the package rounds them, in the backward too (dX = r(G) r(W), dW = r(G)^T r(X), db = sum G unrounded), while
# the arithmetic stays in the oracle's dtype.  The summation-matrix product and the attention softmax stay unrounded: the
# package computes them in fp32 kernels.  |o_mode - o64| is then what a correct implementation of that precision loses
# against exact arithmetic.  None: the plain ops, unchanged.
OPERANDS = None
_DTYPE16 = {"bf16": torch.bfloat16, "fp16": torch.float16}


def round_operand(x, mode):
    """x rounded as the package rounds a GEMM operand, returned in x's dtype.  The package's operands are fp32 values,
    so x goes through fp32 first.  tf32: round to nearest, ties away from zero (cvt.rna); bf16 / fp16: torch's
    `.to(dtype)` (round to nearest even; fp16 overflows to +-inf)."""
    x32 = x.float()
    if mode == "tf32":
        b = x32.contiguous().view(torch.int32)
        return ((b + 0x1000) & -0x2000).view(torch.float32).to(x.dtype)
    return x32.to(_DTYPE16[mode]).to(x.dtype)


class _RoundedMatmul(torch.autograd.Function):
    """r(a) @ r(b); the backward rounds the incoming gradient and reuses the rounded operands"""

    @staticmethod
    def forward(ctx, a, b, mode):
        ra, rb = round_operand(a, mode), round_operand(b, mode)
        ctx.save_for_backward(ra, rb)
        ctx.mode = mode
        return ra @ rb

    @staticmethod
    def backward(ctx, g):
        ra, rb = ctx.saved_tensors
        rg = round_operand(g, ctx.mode)
        return rg @ rb.transpose(-1, -2), ra.transpose(-1, -2) @ rg, None


def linear(x, w, b):
    """F.linear, or under OPERANDS its product on rounded operands (the bias added unrounded)"""
    if OPERANDS is None:
        return F.linear(x, w, b)
    y = _RoundedMatmul.apply(x.reshape(-1, x.shape[-1]), w.t(), OPERANDS)
    return y.reshape(*x.shape[:-1], w.shape[0]) + b


def matmul(a, b):
    """torch.matmul, or under OPERANDS its product on rounded operands (same batch shape on both sides)"""
    if OPERANDS is None:
        return torch.matmul(a, b)
    return _RoundedMatmul.apply(a, b, OPERANDS)


class _SeluKink(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, tau, side):
        ctx.save_for_backward(x)
        ctx.tau, ctx.side = tau, side
        return F.selu(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        d = torch.where(x > 0, torch.full_like(x, _SELU_SCALE), _SELU_SCALE * _SELU_ALPHA * torch.exp(x))
        forced = _SELU_SCALE if ctx.side == "R" else _SELU_SCALE * _SELU_ALPHA
        d = torch.where(x.abs() < ctx.tau, torch.full_like(x, forced), d)
        return g * d, None, None


def mlp(sd, prefix, x):
    """gnn/modules.py:111-170 -- Linear -> SELU (-> AlphaDropout(p=0) == identity)
    for every layer INCLUDING the last; Linear layers sit at seq.0, seq.3, ..."""
    i = 0
    while f"{prefix}.seq.{i}.weight" in sd:
        pre = linear(x, sd[f"{prefix}.seq.{i}.weight"], sd[f"{prefix}.seq.{i}.bias"])
        if MARGINS is not None and pre.numel():
            MARGINS.append(float(pre.detach().abs().min()))
        x = F.selu(pre) if KINK is None else _SeluKink.apply(pre, KINK[0], KINK[1])
        i += 3
    return x


def gru_cell(sd, x, h):
    """torch.nn.GRUCell as used at gnn/mpnn.py:67,296,391,488 (gate order r,z,n;
    SURVEY Appendix D).  Written out so the gate arithmetic is explicit."""
    gi = linear(x, sd["gru.weight_ih"], sd["gru.bias_ih"])
    gh = linear(h, sd["gru.weight_hh"], sd["gru.bias_hh"])
    i_r, i_z, i_n = gi.chunk(3, 1)
    h_r, h_z, h_n = gh.chunk(3, 1)
    r = torch.sigmoid(i_r + h_r)
    z = torch.sigmoid(i_z + h_z)
    n = torch.tanh(i_n + r * h_n)
    return (1.0 - z) * n + z * h


def graph_gather(sd, hidden, inputs, node_mask):
    """gnn/modules.py:39-52 -- per-channel masked softmax over the node axis."""
    cat = torch.cat((hidden, inputs), dim=2)
    energy_mask = (node_mask == 0).to(cat.dtype) * BIG
    raw = mlp(sd, "gather.att_nn", cat)
    if MARGINS is not None and bool((node_mask == 0).any()):
        q = raw.detach()[node_mask == 0].double() * 16.0        # fp32 spacing near 1e6 is 1/16
        MARGINS.append(float(((q - q.floor() - 0.5).abs().min()) / 16.0))
    energies = raw - energy_mask.unsqueeze(-1)
    attention = torch.softmax(energies, dim=1)
    embedding = mlp(sd, "gather.emb_nn", hidden)
    return torch.sum(attention * embedding, dim=1)


def global_readout(sd, node_level, graph_emb):
    """gnn/modules.py:237-281 -- two-tier APD head, output is SELU-activated."""
    f_add_1 = mlp(sd, "APDReadout.fAddNet1", node_level)
    f_conn_1 = mlp(sd, "APDReadout.fConnNet1", node_level)
    b = f_add_1.shape[0]
    f_add_1 = f_add_1.reshape(b, -1)
    f_conn_1 = f_conn_1.reshape(b, -1)
    f_add_2 = mlp(sd, "APDReadout.fAddNet2", torch.cat((f_add_1, graph_emb), dim=1))
    f_conn_2 = mlp(sd, "APDReadout.fConnNet2", torch.cat((f_conn_1, graph_emb), dim=1))
    f_term_2 = mlp(sd, "APDReadout.fTermNet2", graph_emb)
    return torch.cat((f_add_2, f_conn_2, f_term_2), dim=1)


def _pad_hidden(nodes, width):
    """summation_mpnn.py:121-125 -- zero-pad node features to the hidden width."""
    hidden = torch.zeros(nodes.shape[0], nodes.shape[1], width, dtype=nodes.dtype)
    hidden[:, :, :nodes.shape[2]] = nodes
    return hidden


# --------------------------------------------------------------------------- #
# SummationMPNN family: GGNN, MNN  (gnn/summation_mpnn.py:80-149)
# --------------------------------------------------------------------------- #
def _summation_forward(sd, C, nodes, edges, message_terms, readout):
    adjacency = edges.sum(dim=3)                                       # :102
    e_b, e_i, e_j = adjacency.nonzero(as_tuple=True)                   # :105-107 dst=i src=j
    n_b, n_i = adjacency.sum(-1).nonzero(as_tuple=True)                # :109
    same = (n_b.view(-1, 1) == e_b) * (n_i.view(-1, 1) == e_i)         # :111-112
    summation_matrix = same.to(nodes.dtype)                            # :116 `.float()`; dense [V,E]
    edge_feats = edges[e_b, e_i, e_j, :]                               # :118
    hidden = _pad_hidden(nodes, C.hidden_node_features)
    node_rows = hidden[n_b, n_i, :]                                    # :126
    for _ in range(C.message_passes):                                  # :128-144
        nghb_rows = hidden[e_b, e_j, :]
        terms = message_terms(nghb_rows, edge_feats)
        if terms.dim() == 1:
            terms = terms.unsqueeze(0)
        messages = torch.matmul(summation_matrix, terms)               # :141 scatter-add
        node_rows = gru_cell(sd, messages, node_rows)
        hidden = hidden.index_put((n_b, n_i), node_rows)               # :144
    node_mask = adjacency.sum(-1) != 0                                 # :146
    return readout(hidden, nodes, node_mask)


def ggnn_forward(sd, C, nodes, edges):
    """gnn/mpnn.py:229-303."""
    def message_terms(nghb_rows, edge_feats):                          # mpnn.py:284-294
        ev = edge_feats.view(-1, C.n_edge_features, 1)
        scaled = ev * nghb_rows.view(-1, 1, C.hidden_node_features)
        return sum(ev[:, t, :] * mlp(sd, f"msg_nns.{t}", scaled[:, t, :])
                   for t in range(C.n_edge_features))

    def readout(hidden, inputs, mask):                                 # mpnn.py:299-303
        return global_readout(sd, hidden, graph_gather(sd, hidden, inputs, mask))

    return _summation_forward(sd, C, nodes, edges, message_terms, readout)


def mnn_forward(sd, C, nodes, edges):
    """gnn/mpnn.py:16-74."""
    W = sd["message_weights"]                                          # [msg, H, Ef]

    def message_terms(nghb_rows, edge_feats):                          # mpnn.py:60-65
        per_edge = (edge_feats.view(-1, 1, 1, C.n_edge_features) * W.unsqueeze(0)).sum(3)
        # the package's message product (one Linear per bond type on the strided slice W[:, :, t]); with unit bond
        # values the rounded per_edge is the rounded slice
        return matmul(per_edge, nghb_rows.unsqueeze(-1)).squeeze()

    def readout(hidden, inputs, mask):                                 # mpnn.py:70-74
        return global_readout(sd, hidden, hidden.sum(dim=1))

    return _summation_forward(sd, C, nodes, edges, message_terms, readout)


# --------------------------------------------------------------------------- #
# AggregationMPNN family: AttentionGGNN  (gnn/aggregation_mpnn.py:83-168)
# --------------------------------------------------------------------------- #
def attggnn_forward(sd, C, nodes, edges):
    """gnn/aggregation_mpnn.py:105-168 + gnn/mpnn.py:370-398.  The per-node Python
    loops of the reference (:126-132) are restated with repeat_interleave, which
    yields the same index vectors."""
    adjacency = edges.sum(dim=3)
    e_b, e_i, e_j = adjacency.nonzero(as_tuple=True)
    n_b, n_i = adjacency.sum(-1).nonzero(as_tuple=True)
    node_adj = adjacency[n_b, n_i, :]
    V = n_b.shape[0]
    degrees = node_adj.sum(-1).long()
    D = int(degrees.max())                                             # :115
    H = C.hidden_node_features
    slot = torch.cat([torch.arange(int(d)) for d in degrees]).long()   # :126-128
    owner = torch.repeat_interleave(torch.arange(V), degrees)          # :130-132
    mask = torch.zeros(V, D, dtype=nodes.dtype)
    mask[owner, slot] = 1                                              # :138
    nb_edges = torch.zeros(V, D, C.n_edge_features, dtype=nodes.dtype)
    nb_edges[owner, slot, :] = edges[e_b, e_i, e_j, :]                 # :140-141
    hidden = _pad_hidden(nodes, H)
    for _ in range(C.message_passes):                                  # :150-164
        node_rows = hidden[n_b, n_i, :]
        nghbs = torch.zeros(V, D, H, dtype=nodes.dtype).index_put((owner, slot), hidden[e_b, e_j, :])
        energy_mask = (mask == 0).to(nodes.dtype) * BIG                # mpnn.py:374
        emb = sum(nb_edges[:, :, t].unsqueeze(-1) * mlp(sd, f"msg_nns.{t}", nghbs)
                  for t in range(C.n_edge_features))
        ene = sum(nb_edges[:, :, t].unsqueeze(-1) * mlp(sd, f"att_nns.{t}", nghbs)
                  for t in range(C.n_edge_features)) - energy_mask.unsqueeze(-1)
        messages = torch.sum(torch.softmax(ene, dim=1) * emb, dim=1)   # mpnn.py:387-389
        hidden = hidden.index_put((n_b, n_i), gru_cell(sd, messages, node_rows))
    node_mask = adjacency.sum(-1) != 0
    return global_readout(sd, hidden, graph_gather(sd, hidden, nodes, node_mask))


# --------------------------------------------------------------------------- #
# EdgeMPNN family: EMN  (gnn/edge_mpnn.py:82-192)
# --------------------------------------------------------------------------- #
def emn_forward(sd, C, nodes, edges):
    """gnn/edge_mpnn.py:104-192 + gnn/mpnn.py:466-494.

    Directed edge r = (b, i, j).  Its incoming set is {memory of s=(b, j, k) : k != i},
    stored at slot = rank of k among j's neighbours (slots are NOT compacted after the
    reverse edge is dropped, `edge_mpnn.py:162-173`)."""
    adjacency = edges.sum(dim=3)
    e_b, e_i, e_j = adjacency.nonzero(as_tuple=True)                   # :110
    E = e_i.shape[0]
    B, N = adjacency.shape[0], adjacency.shape[1]
    emb = C.edge_emb_size
    edge_id = torch.zeros(B, N, N, dtype=torch.long)
    edge_id[e_b, e_i, e_j] = torch.arange(1, E + 1)                    # :113-118
    rows = edge_id[e_b, e_j, :]                                        # row of the head node j
    recv, slot_k = rows.nonzero(as_tuple=True)                         # ascending (r, k)
    send = rows[recv, slot_k] - 1                                      # :120-123
    head_deg = adjacency[e_b, e_j, :].sum(-1).long()                   # :125
    slot = torch.cat([torch.arange(int(d)) for d in head_deg] or
                     [torch.zeros(0, dtype=torch.long)]).long()        # :129
    keep = e_i[recv] != e_j[send]                                      # :158-160 (k != i)
    recv, send, slot = recv[keep], send[keep], slot[keep]
    D = int(adjacency.sum(-1).max())                                   # :134
    in_mask = torch.zeros(E, D, dtype=nodes.dtype)
    in_mask[recv, slot] = 1                                            # :173
    x = torch.tanh(mlp(sd, "embedding_nn", torch.cat(
        (nodes[e_b, e_i, :], nodes[e_b, e_j, :], edges[e_b, e_i, e_j, :]), dim=1)))  # mpnn.py:466-469
    memories = torch.zeros(E, emb, dtype=nodes.dtype)
    energy_mask = ((1 - in_mask).to(nodes.dtype) * (-BIG)).unsqueeze(-1)  # mpnn.py:475-477
    for _ in range(C.message_passes):                                  # :175-182
        in_mem = torch.zeros(E, D, emb, dtype=nodes.dtype).index_put((recv, slot), memories[send, :])
        cat = torch.cat((x.unsqueeze(1), in_mem), dim=1)               # mpnn.py:478
        embeddings = mlp(sd, "emb_msg_nn", cat)
        energies = torch.cat((mlp(sd, "att_msg_nn", x).unsqueeze(1),
                              mlp(sd, "att_msg_nn", in_mem) + energy_mask), dim=1)
        message = (torch.softmax(energies, dim=1) * embeddings).sum(dim=1)
        memories = gru_cell(sd, message, torch.zeros(E, emb, dtype=nodes.dtype))   # mpnn.py:488, hx=None
    node_mask = adjacency.sum(-1) != 0
    # :184-189 -- node vector = sum of the memories of its outgoing edges
    graph_sets = torch.zeros(B * N, emb, dtype=nodes.dtype).index_add(0, e_b * N + e_i, memories).view(B, N, emb)
    return global_readout(sd, graph_sets, graph_gather(sd, graph_sets, graph_sets, node_mask))


FORWARD = {"GGNN": ggnn_forward, "MNN": mnn_forward,
           "AttGGNN": attggnn_forward, "EMN": emn_forward}


def forward(sd, C, nodes, edges):
    return FORWARD[C.model](sd, C, nodes, edges)


# --------------------------------------------------------------------------- #
# call-site post-ops
# --------------------------------------------------------------------------- #
def kl_loss(output, target):
    """Workflow.py:833-860 -- KLDivLoss(batchmean)(log_softmax(output), target/sum)."""
    logp = torch.log_softmax(output, dim=1)
    target = target / torch.sum(target, dim=1, keepdim=True)
    return F.kl_div(logp, target, reduction="batchmean")


def train_step_grads(sd, C, nodes, edges, target, dtype=None):
    """One forward + loss + backward (Workflow.py:785-794).  Returns loss, logits and
    an OrderedDict of gradients keyed like the state_dict.

    dtype=torch.float64 evaluates the same expression in double precision: the anchor of the
    gradient-parity tests (`|cuda - fp64| <= c * |reference_fp32 - fp64|`) -- the reference's own
    fp32 rounding then sets the yardstick instead of a hand-picked tolerance."""
    if dtype is not None:
        sd = OrderedDict((k, v.to(dtype)) for k, v in sd.items())
        nodes, edges, target = nodes.to(dtype), edges.to(dtype), target.to(dtype)
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in sd.items())
    out = forward(leaves, C, nodes, edges)
    loss = kl_loss(out, target)
    grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    g = OrderedDict((k, (gi if gi is not None else torch.zeros_like(v)))
                    for (k, v), gi in zip(leaves.items(), grads))
    return loss.detach(), out.detach(), g


# --------------------------------------------------------------------------- #
# parameter construction with the reference's shapes / init (SURVEY Appendix A)
# --------------------------------------------------------------------------- #
def _mlp_shapes(prefix, fin, hidden, depth, fout):
    sizes = [fin] + [hidden] * depth + [fout]
    out = []
    for li, (a, b) in enumerate(zip(sizes, sizes[1:])):
        out.append((f"{prefix}.seq.{3 * li}.weight", (b, a)))
        out.append((f"{prefix}.seq.{3 * li}.bias", (b,)))
    return out


def param_shapes(C):
    """state_dict schema per model, in the reference's registration order
    (gnn/mpnn.py:16-52, 229-282, 306-368, 401-464)."""
    N, fa, fc = C.max_n_nodes, C.len_f_add_per_node, C.len_f_conn_per_node
    F_, Ef = C.n_node_features, C.n_edge_features
    s = []
    if C.model == "MNN":
        H, msg, gemb = C.hidden_node_features, C.message_size, C.hidden_node_features
        s.append(("message_weights", (msg, H, Ef)))
        s += [("gru.weight_ih", (3 * H, msg)), ("gru.weight_hh", (3 * H, H)),
              ("gru.bias_ih", (3 * H,)), ("gru.bias_hh", (3 * H,))]
    elif C.model in ("GGNN", "AttGGNN"):
        H, msg, gemb = C.hidden_node_features, C.message_size, C.gather_width
        if C.model == "GGNN":
            for t in range(Ef):
                s += _mlp_shapes(f"msg_nns.{t}", H, C.enn_hidden_dim, C.enn_depth, msg)
        else:
            for t in range(Ef):
                s += _mlp_shapes(f"msg_nns.{t}", H, C.msg_hidden_dim, C.msg_depth, msg)
            for t in range(Ef):
                s += _mlp_shapes(f"att_nns.{t}", H, C.att_hidden_dim, C.att_depth, msg)
        s += [("gru.weight_ih", (3 * H, msg)), ("gru.weight_hh", (3 * H, H)),
              ("gru.bias_ih", (3 * H,)), ("gru.bias_hh", (3 * H,))]
        s += _mlp_shapes("gather.att_nn", H + F_, C.gather_att_hidden_dim, C.gather_att_depth, gemb)
        s += _mlp_shapes("gather.emb_nn", H, C.gather_emb_hidden_dim, C.gather_emb_depth, gemb)
    elif C.model == "EMN":
        H, gemb = C.edge_emb_size, C.gather_width
        s += _mlp_shapes("embedding_nn", 2 * F_ + Ef, C.edge_emb_hidden_dim, C.edge_emb_depth, H)
        s += _mlp_shapes("emb_msg_nn", H, C.msg_hidden_dim, C.msg_depth, H)
        s += _mlp_shapes("att_msg_nn", H, C.att_hidden_dim, C.att_depth, H)
        s += [("gru.weight_ih", (3 * H, H)), ("gru.weight_hh", (3 * H, H)),
              ("gru.bias_ih", (3 * H,)), ("gru.bias_hh", (3 * H,))]
        s += _mlp_shapes("gather.att_nn", 2 * H, C.gather_att_hidden_dim, C.gather_att_depth, gemb)
        s += _mlp_shapes("gather.emb_nn", H, C.gather_emb_hidden_dim, C.gather_emb_depth, gemb)
    else:
        raise ValueError(C.model)
    s += _mlp_shapes("APDReadout.fAddNet1", H, C.mlp1_hidden_dim, C.mlp1_depth, fa)
    s += _mlp_shapes("APDReadout.fConnNet1", H, C.mlp1_hidden_dim, C.mlp1_depth, fc)
    s += _mlp_shapes("APDReadout.fAddNet2", N * fa + gemb, C.mlp2_hidden_dim, C.mlp2_depth, N * fa)
    s += _mlp_shapes("APDReadout.fConnNet2", N * fc + gemb, C.mlp2_hidden_dim, C.mlp2_depth, N * fc)
    s += _mlp_shapes("APDReadout.fTermNet2", gemb, C.mlp2_hidden_dim, C.mlp2_depth, 1)
    return s


def init_state_dict(C, seed=0):
    """Random parameters of the reference's shapes: xavier-uniform MLP weights
    (modules.py:162-163), U(+-1/sqrt(fan)) for biases / GRU / MNN message weights
    (PyTorch defaults, mpnn.py:56-58).  Same distributions as the reference, own
    RNG stream -- use a reference-built state_dict when identical values matter."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, shape in param_shapes(C):
        if name.startswith("gru."):
            bound = 1.0 / (C.edge_emb_size if C.model == "EMN" else C.hidden_node_features) ** 0.5
        elif name == "message_weights":
            bound = 1.0 / shape[1] ** 0.5
        elif name.endswith(".weight"):
            bound = (6.0 / (shape[0] + shape[1])) ** 0.5
        else:  # Linear bias: U(+-1/sqrt(fan_in)); fan_in from the matching weight
            bound = 1.0 / sd[name[:-4] + "weight"].shape[1] ** 0.5
        sd[name] = (torch.rand(shape, generator=g) * 2 - 1) * bound
    return sd
