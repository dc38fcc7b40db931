"""Training-set properties of the preprocessing phase: the reference's per-group `get_ts_properties` loop
(Analyzer.get_molecular_properties + combine_ts_properties, DataProcesser.py:389-417) with constants.device = "cuda",
as a real preprocessing job runs it, against the device pass (gib_preprocess_group_statistics via
graphinvent_b200.preprocess.groups(..., statistics=True), the dicts and the merge).

    python tools/bench_ts_properties.py [--repeats 5] [--synthetic 5000] [--reference-repeats 1]

Sets: gdb13_1K/train (979 molecules, batch_size 1000; tests/golden/preprocess_gdb13.npz) and a synthetic set of
38-atom molecules (graphinvent_b200.synthetic, batch_size 1000).  Each time is the host clock around the whole
computation, ended by a device synchronise; the median of the repeats after one warm-up.
  reference     the get_ts_properties loop over the groups' graph slices (the graphs are built before the clock starts)
  device        groups(statistics=True) with the per-group dicts and merges: the construction AND the properties
  construction  groups() alone, so device - construction is what the properties add to the device pass
The reference's Analyzer comes from oracle/_ref (installed by __graft_entry__.build()), with the stub modules of
tests/molecules_reference.py.  One JSON line per set, with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_preprocess import card, gdb13, synthetic  # noqa: E402


def timed(fn, repeats):
    import torch
    fn()
    out = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return float(np.median(out)), [float(min(out)), float(max(out))]


def measure(name, nodes, edges, B, repeats, ref_repeats):
    from graphinvent_b200 import preprocess as PP
    from tests import molecules_reference as MR
    from tests import ts_properties_reference as TR
    C = TR.constants("gdb13", nodes.shape[1], edges.shape[3], B, device="cuda")
    ref = MR.load_reference(C)
    if ref is None:
        raise SystemExit("oracle/_ref holds no Analyzer.py: run __graft_entry__.build() where the reference is present")
    MR.set_constants(ref, C)
    graphs = TR.preprocessing_graphs(ref, C, nodes, edges)
    spans = [(g.start, g.stop) for g in PP.groups(nodes, edges, B, 5, 3)]
    analyzer = ref.Analyzer.Analyzer.__new__(ref.Analyzer.Analyzer)
    smiles = [g.get_smiles() for g in graphs]

    def device():
        props = None
        for g in PP.groups(nodes, edges, B, 5, 3, statistics=True):
            props = PP.merge_ts_properties(analyzer, props, PP.ts_properties(g.statistics, smiles[g.start:g.stop], C),
                                           B)
        return props

    t_ref, s_ref = timed(lambda: TR.reference_ts_properties(ref, graphs, spans, B), ref_repeats)
    t_dev, s_dev = timed(device, repeats)
    t_con, s_con = timed(lambda: list(PP.groups(nodes, edges, B, 5, 3)), repeats)
    TR.assert_identical(device(), TR.reference_ts_properties(ref, graphs, spans, B))
    M = int(nodes.shape[0])
    print(json.dumps(dict(set=name, molecules=M, groups=len(spans), batch_size=B,
                          reference_seconds=t_ref, reference_spread=s_ref,
                          device_seconds=t_dev, device_spread=s_dev,
                          construction_seconds=t_con, construction_spread=s_con,
                          properties_added_seconds=t_dev - t_con,
                          reference_molecules_per_s=M / t_ref, device_molecules_per_s=M / t_dev,
                          device=card())))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--reference-repeats", type=int, default=1)
    ap.add_argument("--synthetic", type=int, default=5000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("this measurement needs a CUDA device")
    for name, (nodes, edges) in (("gdb13_1K/train", gdb13()), (f"synthetic N=38 x{a.synthetic}",
                                                               synthetic(a.synthetic))):
        measure(name, nodes, edges, 1000, a.repeats, a.reference_repeats)


if __name__ == "__main__":
    main()
