"""Installs the unmodified reference's MolecularGraph.py, Analyzer.py and GraphGeneratorRL.py into the git-ignored
oracle/_ref/graphinvent/ (called by __graft_entry__.build(), after reference_install.install)."""
import os
import shutil

from oracle.reference_install import REF

FILES = ("MolecularGraph.py", "Analyzer.py", "GraphGeneratorRL.py")


def install(root):
    """When a checkout of the reference is present, its `graph_to_graph` (GraphGenerator.py, installed by
    reference_install; GraphGeneratorRL.py), `GenerationGraph` (MolecularGraph.py) and `get_molecular_properties`
    (Analyzer.py) are copied file by file next to GraphGenerator.py, so that tests/test_*molecules*.py and
    tools/bench_molecules.py can run them live (with stub modules for rdkit, matplotlib, tensorboard, util and
    parameters.constants, tests/molecules_reference.py).  Nothing in the product path imports them."""
    src = os.path.join(REF, "graphinvent")
    dst = os.path.join(root, "oracle", "_ref", "graphinvent")
    if not all(os.path.isfile(os.path.join(src, f)) for f in FILES):
        return
    os.makedirs(dst, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(src, f), os.path.join(dst, f))
    print(f"installed the reference's {', '.join(FILES)} into {dst}")
