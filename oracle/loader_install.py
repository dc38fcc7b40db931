"""Installs the unmodified reference's BlockDatasetLoader.py into the git-ignored oracle/_ref/graphinvent/ (called by
__graft_entry__.build(), after reference_install.install)."""
import os
import shutil

from oracle.reference_install import REF

FILE = "BlockDatasetLoader.py"


def install(root):
    """When a checkout of the reference is present, its block loader (`BlockDataLoader`, `HDFDataset`) is copied next
    to GraphGenerator.py, so that tests/test_device_loader_host.py can compare `loader.DeviceBlockLoader`'s order with
    it live, tests/golden/make_loader_order.py can record it, and tools/bench_epoch.py can time it (its `import h5py`
    is stubbed there).  Nothing in the product path imports it."""
    src = os.path.join(REF, "graphinvent", FILE)
    dst = os.path.join(root, "oracle", "_ref", "graphinvent")
    if not os.path.isfile(src):
        return
    os.makedirs(dst, exist_ok=True)
    shutil.copyfile(src, os.path.join(dst, FILE))
    print(f"installed the reference's {FILE} into {dst}")
