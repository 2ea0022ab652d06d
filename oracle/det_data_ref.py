"""Stages the original VoteNet detection datasets next to the oracle, so that the tests, tests/golden/make_det_data_golden.py and
profiles/bench_det_data.py can run their `__getitem__` unmodified against pointcontrast_b200.det_data:

    python oracle/det_data_ref.py       (also run by __graft_entry__.build(), after oracle/det_eval_ref.py, which clears and stages
                                         oracle/_ref/votenet/lib/ with the model-util modules these files import)

Copies, byte for byte, `lib/datasets/scannet/scannet_detection_dataset.py`, `lib/datasets/sunrgbd/sunrgbd_detection_dataset.py` and
`lib/utils/pc_util.py` from `<root>/downstream/votenet_det_new/` into `oracle/_ref/votenet/` (git-ignored).  <root> is
$PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the original is absent nothing is staged.  Nothing under
pointcontrast_b200/ imports this.

load() imports both modules the way the original runs them, through oracle/det_eval_ref.load() (its root and `lib/utils` on sys.path,
stubs for trimesh, matplotlib and cv2, which `pc_util` and `sunrgbd_utils` import but these paths never call).
"""
import importlib
import os
import shutil

from oracle import det_eval_ref

SRC = det_eval_ref.SRC
ROOT = det_eval_ref.ROOT
FILES = (os.path.join("lib", "datasets", "scannet", "scannet_detection_dataset.py"),
         os.path.join("lib", "datasets", "sunrgbd", "sunrgbd_detection_dataset.py"),
         os.path.join("lib", "utils", "pc_util.py"))


def stage(verbose=False):
    if not os.path.isfile(os.path.join(SRC, FILES[0])) or not det_eval_ref.available():
        return False
    for f in FILES:
        os.makedirs(os.path.dirname(os.path.join(ROOT, f)), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, f), os.path.join(ROOT, f))
    if verbose:
        print("staged", SRC, "(detection datasets) ->", ROOT)
    return True


def available():
    return det_eval_ref.available() and all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES)


def load():
    """(scannet_detection_dataset, sunrgbd_detection_dataset) modules of the original, or None where nothing is staged."""
    if not available():
        return None
    det_eval_ref.load()
    return (importlib.import_module("lib.datasets.scannet.scannet_detection_dataset"),
            importlib.import_module("lib.datasets.sunrgbd.sunrgbd_detection_dataset"))


def item(module_cls, data_path, scan_names, num_points, use_color, use_height, augment, idx, draws):
    """The original `__getitem__(idx)` on an instance whose attributes are set directly (its constructor derives the paths from its
    own location), with np.random.random / np.random.choice replaced by `draws` (a callable(kind, *args) -> value)."""
    import numpy as np
    ds = module_cls.__new__(module_cls)
    ds.data_path, ds.scan_names, ds.num_points = data_path, list(scan_names), num_points
    ds.use_color, ds.use_height, ds.augment = use_color, use_height, augment
    saved = np.random.random, np.random.choice
    np.random.random = lambda *a: draws("random", *a)
    np.random.choice = lambda *a, **kw: draws("choice", *a, **kw)
    try:
        return ds[idx]
    finally:
        np.random.random, np.random.choice = saved


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present (or the evaluation code is not staged): nothing staged")
