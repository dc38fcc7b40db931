"""fp64 restatement of the decoding-route likelihood (graphinvent_b200.graphed.RouteScorer), the oracle of its tests:
the route states of tests/preprocess_reference.route, reversed into build order (the empty graph first, the full
graph with the terminate action last), each scored by softmax(oracle/mpnn_oracle.forward(state))[action] in float64."""
from collections import OrderedDict

import numpy as np
import torch

from tests import preprocess_reference as P


def build_order_states(nodes, edges, segs):
    """(X [S, N, F], E [S, N, N, Ef], actions [S], offsets [M + 1]) of every molecule's route, in build order"""
    Xs, Es, acts, offsets = [], [], [], [0]
    for m in range(nodes.shape[0]):
        states = P.route(nodes[m], edges[m], segs)[::-1]
        Xs += [s[0] for s in states]
        Es += [s[1] for s in states]
        acts += [s[2] for s in states]
        offsets.append(offsets[-1] + len(states))
    return np.stack(Xs), np.stack(Es), np.array(acts, np.int64), np.array(offsets, np.int64)


def probabilities(sd, C, X, E, actions, batch=512, dtype=torch.float64):
    """softmax(forward(state))[action] of every state in `dtype`, and the logits"""
    from oracle import mpnn_oracle as O
    sd = OrderedDict((k, v.to(dtype)) for k, v in sd.items())
    out = []
    for s in range(0, X.shape[0], batch):
        out.append(O.forward(sd, C, torch.from_numpy(X[s:s + batch]).to(dtype),
                             torch.from_numpy(E[s:s + batch]).to(dtype)).detach())
    logits = torch.cat(out)
    p = torch.softmax(logits, dim=1).gather(1, torch.from_numpy(actions).view(-1, 1)).view(-1)
    return p, logits


def log_p_bound(sd, C, X, E, actions, logits64):
    """per state, a bound on |log p - log p_fp64| for a forward that keeps the logits contract -- per molecule within
    3x the reference's own fp32 error plus 1e-4 (DESIGN.md section 4): log p = o_a - logsumexp(o) moves by at most
    twice the largest logit error.  The fp32 error is the oracle's own fp32 evaluation against fp64."""
    _, logits32 = probabilities(sd, C, X, E, actions, dtype=torch.float32)
    e32 = (logits32.double() - logits64).abs().max(1).values
    return 2 * (3 * e32 + 1e-4)


def reduce(p, offsets):
    """per molecule: -sum log p and log(sum p), in p's dtype and build order"""
    nll = torch.stack([-torch.log(p[a:b]).sum() for a, b in zip(offsets[:-1], offsets[1:])])
    final = torch.stack([torch.log(p[a:b].sum()) for a, b in zip(offsets[:-1], offsets[1:])])
    return nll, final


def score(sd, C, nodes, edges, segs):
    """(likelihoods, offsets, nll, final, log_p_bound) of the molecules in fp64"""
    X, E, acts, offsets = build_order_states(nodes, edges, segs)
    p, logits = probabilities(sd, C, X, E, acts)
    nll, final = reduce(p, offsets)
    return p, offsets, nll, final, log_p_bound(sd, C, X, E, acts, logits)


def assert_within(lik, nll, final, oracle, what=""):
    """likelihoods, nll and final of a scorer against `score`'s fp64 values and bound: per state |d log p| <= b, per
    molecule |d nll| <= the sum of its states' b, |d final| <= their max (log sum p moves no more than its largest
    term's log)"""
    p64, offsets, nll64, final64, b = oracle
    lik, nll, final = (t.detach().cpu().double() for t in (lik, nll, final))
    d = (torch.log(lik) - torch.log(p64)).abs()
    assert lik.shape == p64.shape and (d <= b).all(), f"{what}: worst |d log p| / bound {(d / b).max().item():.3g}"
    for m, (a, e) in enumerate(zip(offsets[:-1], offsets[1:])):
        tol_n = b[a:e].sum().item() + 1e-6 * abs(nll64[m].item())
        tol_f = b[a:e].max().item() + 1e-6
        assert abs(nll[m].item() - nll64[m].item()) <= tol_n, f"{what}: molecule {m} nll"
        assert abs(final[m].item() - final64[m].item()) <= tol_f, f"{what}: molecule {m} final"
