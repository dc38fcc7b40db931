"""
Numpy restatement of the reference's training-set construction -- the decoding route of
`PreprocessingGraph` (MolecularGraph.py:463-555, 635-732) and the per-group deduplication of
`DataProcesser.get_subgraphs` / `get_molecule_subset` / `save_group` (DataProcesser.py:82-117, 167-271, 340-361,
434-457) -- written from the reference's rules, not from the kernels.  The oracle of graphinvent_b200.preprocess.

Groups are deduplicated with a dict on the state's bytes instead of the reference's quadratic scan; the reference's
append rule is kept: a state is appended as a new row when it matches no row, or when its first match is the LAST row
(its APD is then added to that row and the new row carries it too).
"""
import numpy as np


def segments(n_atom_types, n_formal_charge, n_imp_H=0, n_chirality=0):
    """widths of the one-hot node-feature segments (util.get_feature_vector_indices); 0 = segment absent"""
    return [n_atom_types, n_formal_charge] + [s for s in (n_imp_H, n_chirality) if s]


def apd_length(N, Ef, segs):
    return N * (int(np.prod(segs)) * Ef + Ef) + 1


def n_atoms(nodes):
    """node count of one padded graph: rows up to the last non-zero one"""
    nz = np.flatnonzero(nodes.any(1))
    return int(nz[-1]) + 1 if nz.size else 0


def _bonds(E, last):
    """nonzero(E[:, last, t]) concatenated over t: (node, type) pairs, type-major"""
    return [(int(v), t) for t in range(E.shape[2]) for v in np.flatnonzero(E[:, last, t])]


def _apd_index(X, E, n, segs):
    N, Ef = E.shape[0], E.shape[2]
    last = n - 1
    idc = np.flatnonzero(X[last])
    cum = np.cumsum(segs)
    seg = [int(idc[0])] + [int(v - cum[j]) for j, v in enumerate(idc[1:])]
    flat = 0
    for s, d in zip(seg, segs):
        flat = flat * d + s
    f_add = int(np.prod(segs)) * Ef
    bonds = _bonds(E, last)
    if not bonds:
        return flat * Ef
    v, b = bonds[-1]
    if len(bonds) == 1:
        return v * f_add + flat * Ef + b
    return N * f_add + v * Ef + b


def _truncate(X, E, n):
    last = n - 1
    if n == 1:
        X[last] = 0
        return n - 1
    bonds = _bonds(E, last)
    if not bonds:
        raise ValueError("disconnected graph: the reference's truncate_graph raises IndexError")
    v = bonds[-1][0]
    if len(bonds) == 1:
        X[last] = 0
        n -= 1
    E[v, last] = 0
    E[last, v] = 0
    return n


def route(nodes, edges, segs):
    """[(nodes, edges, flat APD index)] of one molecule's decoding route: n_edges + 2 states"""
    X, E = nodes.copy(), edges.copy()
    n = n_atoms(X)
    N, Ef = E.shape[0], E.shape[2]
    apd_len = apd_length(N, Ef, segs)
    out = [(X.copy(), E.copy(), apd_len - 1)]
    for _ in range(int(E.sum()) // 2 + 1):
        a = _apd_index(X, E, n, segs)
        n = _truncate(X, E, n)
        out.append((X.copy(), E.copy(), a))
    return out


def groups(nodes, edges, batch_size, segs):
    """The groups `DataProcesser.preprocess` writes, in order: dicts with rows (int8 nodes / edges, int64 APD counts),
    the molecule range [start, stop) the group visited, `init_idx` (its first row in the chunked file), `full`, and the
    reference's `resume_idx` / `dataset_size` counters after the group."""
    M, N, _ = nodes.shape
    Ef = edges.shape[3]
    apd_len = apd_length(N, Ef, segs)
    B = batch_size
    resume, size, g = 0, 0, 0
    while resume < M:
        rows, apds, where = [], [], {}
        stop, full = min(resume + B, M), False
        for m in range(resume, stop):
            for X, E, a in route(nodes[m], edges[m], segs):
                key = X.tobytes() + E.tobytes()
                r = where.get(key)
                if r is not None:
                    apds[r][a] += 1
                if r is None or r == len(rows) - 1:
                    if r is None:
                        where[key] = len(rows)
                    rows.append((X, E))
                    apd = np.zeros(apd_len, np.int64)
                    apd[a] = 1
                    apds.append(apd)
                if len(rows) == B:
                    full, stop = True, m + 1
                    break
            if full:
                break
        start, resume = resume, stop
        size += B if full else stop - start
        yield dict(index=g, init_idx=g * B, start=start, stop=stop, full=full,
                   nodes=np.array([r[0] for r in rows], np.int8).reshape(-1, N, nodes.shape[2]),
                   edges=np.array([r[1] for r in rows], np.int8).reshape(-1, N, N, Ef),
                   apds=np.array(apds, np.int64).reshape(-1, apd_len),
                   resume_idx=resume, dataset_size=size)
        g += 1


def total_subgraphs(edges):
    """DataProcesser.get_n_subgraphs: sum over molecules of n_edges + 2 (the chunked file's row count)"""
    return int((edges.reshape(edges.shape[0], -1).astype(np.int64).sum(1) // 2 + 2).sum())


def assemble(groups_, n_rows, N, F, Ef, apd_len):
    """the rows of the chunked file after every save_group (int8, as h5py stores them): zeros where no group wrote"""
    nodes = np.zeros((n_rows, N, F), np.int8)
    edges = np.zeros((n_rows, N, N, Ef), np.int8)
    apds = np.zeros((n_rows, apd_len), np.int8)
    for g in groups_:
        r0, r = g["init_idx"], g["nodes"].shape[0]
        nodes[r0:r0 + r], edges[r0:r0 + r] = g["nodes"], g["edges"]
        apds[r0:r0 + r] = np.clip(g["apds"], -128, 127)
    return nodes, edges, apds
