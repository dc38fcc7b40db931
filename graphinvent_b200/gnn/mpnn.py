"""
Drop-in `torch.nn.Module`s for the reference's `gnn.mpnn.{MNN, GGNN, AttentionGGNN, EMN}`
(reference `gnn/mpnn.py:16-74, 229-303, 306-398, 401-494`): same constructor
(`Model(constants)`), same parameter names / shapes / registration order (so the reference's
`.pth` checkpoints load unchanged, SURVEY.md Appendix A), same call
`logits = model(nodes, edges)` on the `BlockDatasetLoader` dense layout.

`forward` runs entirely in libgib200.so (hand-written sm_90a kernels); backward is the
library's explicit backward wired in through one `torch.autograd.Function`.
"""
import math
from collections import namedtuple

import torch

from .. import functional as _F
from .modules import GlobalReadout, GraphGather, MLP


def _c(constants, name, default=None):
    return getattr(constants, name, default)


class _FusedMPNN(torch.nn.Module):
    """Shared machinery: hyper-parameter table for the C-ABI, packed-weight cache, forward."""
    MODEL = None

    def __init__(self, constants: namedtuple) -> None:
        super().__init__()
        self.constants = constants
        self._packed = None
        self._packed_key = None
        self._grad_hook = None      # set by graphinvent_b200.parallel: called on the flat gradient bucket
        self._graph_in = None       # transient: a shared GraphBatch handed to the next forward
        # None: exact mode (one 64-byte header read per forward).  An int = capacity mode: buffers are sized for that
        # many bond entries per batch and the forward performs no host synchronisation (functional.GraphBatch)
        self.entry_capacity = None
        self.last_stats = {}

    # dims shared by every model; subclasses add their own fields
    def _base_dims(self):
        C = self.constants
        return dict(model=self.MODEL, N=C.max_n_nodes, F=C.n_node_features, Ef=C.n_edge_features,
                    f_add=C.len_f_add_per_node, f_conn=C.len_f_conn_per_node,
                    mlp1_hidden=C.mlp1_hidden_dim, mlp1_depth=C.mlp1_depth,
                    mlp2_hidden=C.mlp2_hidden_dim, mlp2_depth=C.mlp2_depth,
                    big=float(_c(C, "big_positive", 1e6)))

    def _dropout_ps(self):
        return [m.dropout_p for m in self.modules() if isinstance(m, MLP)]

    def _check_dropout(self):
        """refuses training mode with dropout: every fused path (forward, the captured generators) runs without it"""
        if self.training and any(p > 0.0 for p in self._dropout_ps()):
            # AlphaDropout draws from torch's RNG stream inside the reference's ATen graph; the
            # fused path cannot reproduce that stream (all reference defaults use p = 0).
            raise NotImplementedError("dropout_p > 0 in training mode is not supported by the fused sm_90a path")

    def forward(self, nodes: torch.Tensor, edges: torch.Tensor, graph=None) -> torch.Tensor:
        """`graph`: optional `functional.build_graph(model, edges)` shared between several models of one family
        evaluated on the same batch (not part of the reference's signature)"""
        self._check_dropout()
        return _F.mpnn_forward(self, nodes, edges, graph)

    def _gather_kwargs(self, node_features, hidden):
        C = self.constants
        return dict(node_features=node_features, hidden_node_features=hidden, out_features=C.gather_width,
                    att_depth=C.gather_att_depth, att_hidden_dim=C.gather_att_hidden_dim,
                    att_dropout_p=C.gather_att_dropout_p, emb_depth=C.gather_emb_depth,
                    emb_hidden_dim=C.gather_emb_hidden_dim, emb_dropout_p=C.gather_emb_dropout_p,
                    big_positive=C.big_positive)

    def _readout_kwargs(self, node_emb, graph_emb):
        C = self.constants
        return dict(node_emb_size=node_emb, graph_emb_size=graph_emb, mlp1_hidden_dim=C.mlp1_hidden_dim,
                    mlp1_depth=C.mlp1_depth, mlp1_dropout_p=C.mlp1_dropout_p, mlp2_hidden_dim=C.mlp2_hidden_dim,
                    mlp2_depth=C.mlp2_depth, mlp2_dropout_p=C.mlp2_dropout_p, f_add_elems=C.len_f_add_per_node,
                    f_conn_elems=C.len_f_conn_per_node, f_term_elems=1, max_n_nodes=C.max_n_nodes,
                    device=_c(C, "device", "cuda"))


class MNN(_FusedMPNN):
    """The "message neural network" (reference mpnn.py:16-74)."""
    MODEL = "MNN"

    def __init__(self, constants: namedtuple) -> None:
        super().__init__(constants)
        C = constants
        self.message_weights = torch.nn.Parameter(
            torch.empty(C.message_size, C.hidden_node_features, C.n_edge_features))
        self.gru = torch.nn.GRUCell(input_size=C.message_size, hidden_size=C.hidden_node_features, bias=True)
        self.APDReadout = GlobalReadout(**self._readout_kwargs(C.hidden_node_features, C.hidden_node_features))
        self.reset_parameters()

    def reset_parameters(self) -> None:
        stdev = 1.0 / math.sqrt(self.message_weights.size(1))    # mpnn.py:56-58
        self.message_weights.data.uniform_(-stdev, stdev)

    def dims(self):
        C = self.constants
        return dict(self._base_dims(), H=C.hidden_node_features, M=C.message_size, T=C.message_passes)


class GGNN(_FusedMPNN):
    """The "gated-graph neural network" (reference mpnn.py:229-303)."""
    MODEL = "GGNN"

    def __init__(self, constants: namedtuple) -> None:
        super().__init__(constants)
        C = constants
        self.msg_nns = torch.nn.ModuleList(
            MLP(C.hidden_node_features, [C.enn_hidden_dim] * C.enn_depth, C.message_size, C.enn_dropout_p)
            for _ in range(C.n_edge_features))
        self.gru = torch.nn.GRUCell(input_size=C.message_size, hidden_size=C.hidden_node_features, bias=True)
        self.gather = GraphGather(**self._gather_kwargs(C.n_node_features, C.hidden_node_features))
        self.APDReadout = GlobalReadout(**self._readout_kwargs(C.hidden_node_features, C.gather_width))

    def dims(self):
        C = self.constants
        return dict(self._base_dims(), H=C.hidden_node_features, M=C.message_size, T=C.message_passes,
                    msg_hidden=C.enn_hidden_dim, msg_depth=C.enn_depth, gather_width=C.gather_width,
                    gatt_hidden=C.gather_att_hidden_dim, gatt_depth=C.gather_att_depth,
                    gemb_hidden=C.gather_emb_hidden_dim, gemb_depth=C.gather_emb_depth)


class AttentionGGNN(_FusedMPNN):
    """The "GGNN with attention" (reference mpnn.py:306-398)."""
    MODEL = "AttGGNN"

    def __init__(self, constants: namedtuple) -> None:
        super().__init__(constants)
        C = constants
        self.msg_nns = torch.nn.ModuleList()
        self.att_nns = torch.nn.ModuleList()
        for _ in range(C.n_edge_features):
            self.msg_nns.append(MLP(C.hidden_node_features, [C.msg_hidden_dim] * C.msg_depth, C.message_size,
                                    C.msg_dropout_p))
            self.att_nns.append(MLP(C.hidden_node_features, [C.att_hidden_dim] * C.att_depth, C.message_size,
                                    C.att_dropout_p))
        self.gru = torch.nn.GRUCell(input_size=C.message_size, hidden_size=C.hidden_node_features, bias=True)
        self.gather = GraphGather(**self._gather_kwargs(C.n_node_features, C.hidden_node_features))
        self.APDReadout = GlobalReadout(**self._readout_kwargs(C.hidden_node_features, C.gather_width))

    def dims(self):
        C = self.constants
        return dict(self._base_dims(), H=C.hidden_node_features, M=C.message_size, T=C.message_passes,
                    msg_hidden=C.msg_hidden_dim, msg_depth=C.msg_depth, att_hidden=C.att_hidden_dim,
                    att_depth=C.att_depth, gather_width=C.gather_width,
                    gatt_hidden=C.gather_att_hidden_dim, gatt_depth=C.gather_att_depth,
                    gemb_hidden=C.gather_emb_hidden_dim, gemb_depth=C.gather_emb_depth)


class EMN(_FusedMPNN):
    """The "edge memory network" (reference mpnn.py:401-494, edge_mpnn.py)."""
    MODEL = "EMN"

    def __init__(self, constants: namedtuple) -> None:
        super().__init__(constants)
        C = constants
        emb = C.edge_emb_size
        self.embedding_nn = MLP(C.n_node_features * 2 + C.n_edge_features,
                                [C.edge_emb_hidden_dim] * C.edge_emb_depth, emb, C.edge_emb_dropout_p)
        self.emb_msg_nn = MLP(emb, [C.msg_hidden_dim] * C.msg_depth, emb, C.msg_dropout_p)
        self.att_msg_nn = MLP(emb, [C.att_hidden_dim] * C.att_depth, emb, C.att_dropout_p)
        self.gru = torch.nn.GRUCell(input_size=emb, hidden_size=emb, bias=True)
        self.gather = GraphGather(**self._gather_kwargs(emb, emb))
        self.APDReadout = GlobalReadout(**self._readout_kwargs(emb, C.gather_width))

    def dims(self):
        C = self.constants
        return dict(self._base_dims(), H=C.edge_emb_size, M=C.edge_emb_size, T=C.message_passes,
                    msg_hidden=C.msg_hidden_dim, msg_depth=C.msg_depth, att_hidden=C.att_hidden_dim,
                    att_depth=C.att_depth, eemb_hidden=C.edge_emb_hidden_dim, eemb_depth=C.edge_emb_depth,
                    gather_width=C.gather_width, gatt_hidden=C.gather_att_hidden_dim,
                    gatt_depth=C.gather_att_depth, gemb_hidden=C.gather_emb_hidden_dim,
                    gemb_depth=C.gather_emb_depth)


MODELS = {"MNN": MNN, "GGNN": GGNN, "AttGGNN": AttentionGGNN, "EMN": EMN}


def create(constants):
    """`Workflow.create_model` dispatch (Workflow.py:274-287) without the S2V variants, which
    cannot be constructed in the reference either (SURVEY.md §2 note a)."""
    try:
        return MODELS[constants.model](constants)
    except KeyError:
        raise NotImplementedError(f"model {constants.model!r} is not on the accelerated path") from None
