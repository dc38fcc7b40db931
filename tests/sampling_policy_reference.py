"""numpy fp64 restatement of the sampling policy (include/gib200.h: gib_sampling_policy), the oracle of the policy
sampler's tests.

On a row of logits o (masked entries -inf), m = max(o):
  ranking  the finite entries by o descending, ties to the lower index;
  weights  exp((o - m) / T) for T > 0; T = 0: weight 1 on the first entry of the ranking, 0 elsewhere;
  top-k    k > 0: the first k entries of the ranking (all finite ones if fewer);
  top-p    p < 1: of those, the shortest prefix of the ranking whose weight reaches p times their total (>= 1 entry);
  draw     inverse CDF over the kept weights in index order at u * total.
A row without a finite entry, or with NaN / +inf, is degenerate: the sampler writes terminate and NaN.
"""
import numpy as np


def degenerate(o):
    o = np.asarray(o, np.float64)
    return bool(np.isnan(o).any() or np.isposinf(o).any() or not np.isfinite(o).any())


def ranking(o):
    """finite indices of o, by o descending, ties to the lower index"""
    o = np.asarray(o, np.float64)
    idx = np.flatnonzero(np.isfinite(o))
    return idx[np.lexsort((idx, -o[idx]))]


def policy(o, T, k, p):
    """(q, kept, margin_p) of a non-degenerate row: q the policy's distribution [apd] (0 outside the kept set), kept the
    kept indices in ranking order, margin_p the distance of the top-p threshold p * total from the nearest prefix sum
    of the ranking, relative to the total (inf when the top-p cut is off)"""
    o = np.asarray(o, np.float64)
    assert not degenerate(o)
    rank = ranking(o)
    m = o[rank[0]]
    w = np.zeros(o.shape, np.float64)
    if T > 0:
        w[rank] = np.exp((o[rank] - m) / T)
        kept = rank[:k] if k > 0 else rank
    else:
        w[rank[0]] = 1.0
        kept = rank[:1]
    margin = np.inf
    if T > 0 and p < 1:
        cs = np.cumsum(w[kept])
        total = cs[-1]
        thr = p * total
        n = int(np.argmax(cs >= thr)) + 1
        near = [abs(cs[n - 1] - thr)] + ([abs(cs[n - 2] - thr)] if n >= 2 else [])
        margin = min(near) / total
        kept = kept[:n]
    q = np.zeros(o.shape, np.float64)
    q[kept] = w[kept]
    q /= q.sum()
    return q, kept, margin


def draw(q, u):
    """(action, margin): the inverse-CDF draw of q in index order at u, and the distance of u from the nearest CDF
    boundary, relative to 1"""
    cdf = np.cumsum(q)
    total = cdf[-1]
    t = min(u * total, np.nextafter(total, 0))
    a = int(np.searchsorted(cdf, t, side="right"))
    nz = np.flatnonzero(q > 0)
    a = int(nz[np.searchsorted(nz, a)]) if a <= nz[-1] else int(nz[-1])
    bounds = cdf[nz]
    return a, float(np.min(np.abs(bounds - t)) / total)


def model_prob(o, a):
    """the masked softmax of o at a, in fp64"""
    o = np.asarray(o, np.float64)
    f = np.isfinite(o)
    m = o[f].max()
    return float(np.exp(o[a] - m) / np.exp(o[f] - m).sum())
