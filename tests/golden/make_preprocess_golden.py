"""Writes tests/golden/preprocess_gdb13.npz from the reference's shipped preprocessed gdb13 sets.

    python tests/golden/make_preprocess_golden.py [/path/to/reference]

For each of gdb13_1K/train (batch_size 1000) and gdb13_1K-debug/{train,valid} (batch_size 50) it stores the full
graphs in input order -- recovered from the file as the rows with a terminate count, since every molecule's first
route state is its full graph with the terminate APD and is processed first -- and the file itself: its 2048-byte
header and its three int8 datasets (read by graphinvent_b200.data.read_hdf5_raw).  The numpy restatement
(tests/preprocess_reference.py) must rebuild each file byte for byte from those graphs before anything is written.
The shipped files hold (groups * batch_size) rows: the unfilled slots of the last group are zeros.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from graphinvent_b200 import data  # noqa: E402
from tests import preprocess_reference as P  # noqa: E402

SETS = (("gdb13_1K/train", 1000), ("gdb13_1K-debug/train", 50), ("gdb13_1K-debug/valid", 50))
N, F, EF, APD = 13, 8, 3, 625
SEGS = P.segments(5, 3)


def rebuild(full_nodes, full_edges, B, header):
    gs = list(P.groups(full_nodes, full_edges, B, SEGS))
    nodes, edges, apds = P.assemble(gs, len(gs) * B, N, F, EF, APD)
    return header + apds.tobytes() + edges.tobytes() + nodes.tobytes(), gs


def main(ref):
    out = {}
    for name, B in SETS:
        path = os.path.join(ref, "data", "pre-training", name + ".h5")
        raw = open(path, "rb").read()
        nodes, edges, apds = data.read_hdf5_raw(path, N, F, EF, APD)
        full = apds[:, -1] > 0
        X, E = nodes[full], edges[full]
        blob, gs = rebuild(X, E, B, raw[:2048])
        assert blob == raw, f"{name}: the restatement does not rebuild the shipped file"
        key = name.replace("/", "_").replace("-", "_")
        out[f"{key}/nodes"], out[f"{key}/edges"] = X, E
        out[f"{key}/header"] = np.frombuffer(raw[:2048], np.uint8)
        out[f"{key}/batch_size"] = np.int64(B)
        out[f"{key}/sha256"] = np.array(hashlib.sha256(raw).hexdigest())
        out[f"{key}/counters"] = np.array([[g["start"], g["stop"], g["init_idx"], g["nodes"].shape[0],
                                            g["resume_idx"], g["dataset_size"]] for g in gs], np.int64)
        print(f"{name}: {X.shape[0]} molecules, {len(gs)} groups, {apds.shape[0]} rows, file rebuilt byte for byte")
    np.savez_compressed(os.path.join(HERE, "preprocess_gdb13.npz"), **out)


if __name__ == "__main__":
    from oracle.reference_install import REF
    main(sys.argv[1] if len(sys.argv) > 1 else REF)
