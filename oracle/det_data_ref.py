"""The original VoteNet detection datasets, staged by oracle/stage_ref.py under `oracle/_ref/votenet/lib/` beside the model-util
modules they import, so that the tests, tests/golden/make_det_data_golden.py and profiles/bench_det_data.py can run their `__getitem__`
unmodified against pointcontrast_b200.det_data.  Nothing under pointcontrast_b200/ imports this.

load() imports both modules the way the original runs them, through oracle/det_eval_ref.load() (its root and `lib/utils` on sys.path,
stubs for trimesh, matplotlib and cv2, which `pc_util` and `sunrgbd_utils` import but these paths never call).
"""
import importlib

from oracle import det_eval_ref


def load():
    """(scannet_detection_dataset, sunrgbd_detection_dataset) modules of the original, or None where nothing is staged."""
    if det_eval_ref.load() is None:
        return None
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
