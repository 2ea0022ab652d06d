"""The original semantic-segmentation full point-cloud evaluation (`lib/{utils.py, datasets/scannet.py, datasets/stanford.py}`),
staged by oracle/stage_ref.py under `oracle/_ref/semseg/lib/`, so that tests/golden/make_semseg_fulleval_golden.py can run it
unmodified.  Nothing under pointcontrast_b200/ imports this.

load() imports the three staged modules under the package name `lib`, with stand-ins for what they import but this path does not
compute with: `omegaconf`, `plyfile`, `lib.distributed_utils`, `lib.transforms`, `lib.dataset` (the base classes, `DatasetPhase`,
`cache`) and `lib.pc_utils` (`save_point_cloud` writes nothing; `read_plyfile` returns the vertex table as pandas' `.values` does,
every column cast to their common dtype).  The staged functions then run with these shims, each needed by a defect of the original
(DESIGN.md section 5):

* `np.int` is `int` while they run (removed from numpy 1.24);
* `save_predictions` is handed batch-LAST coords (x, y, z, batch), the ME 0.3 layout it indexes (`coords[:, -1]`); `lib.dataset`
  defines `OnlineVoxelizationDatasetBase`, which the dataset is not an instance of, and the dataset has `IS_ONLINE_VOXELIZATION = True`,
  `IS_TEMPORAL = False`, so the inverse transformation and the `label_map` decoding run;
* the datasets are built without `__init__` (which reads split files and voxelises): `data_paths`, `data_root` (a Path), `label_map`
  and the reduced `NUM_LABELS` are set on the instance;
* S3DIS: `load_ply(i)` returns the 7-column `[x, y, z, r, g, b, label]` cloud as its first element (the original stacks the 3-column
  coordinates onto 7 columns) and `label2masked` (never defined) is the label map as a table;
* the histograms, which `test_pointcloud` only prints, are recorded by wrapping each module's `fast_hist`.
"""
import contextlib
import enum
import importlib.util
import os
import sys
import types
from pathlib import Path

import numpy as np

from oracle import stage_ref


class _Anything:
    def __getattr__(self, attr):
        return self

    def __call__(self, *a, **k):
        return self


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__getattr__ = lambda a: _Anything() if not a.startswith("__") else (_ for _ in ()).throw(AttributeError(a))
    return m


def _read_plyfile(path):
    from pointcontrast_b200.semseg_data import read_ply
    v = read_ply(path)
    cols = [v[k] for k in v.dtype.names]
    dt = np.result_type(*[c.dtype for c in cols])
    return np.stack([c.astype(dt) for c in cols], 1)


class DatasetPhase(enum.Enum):
    Train = 0
    Val = 1
    Val2 = 2
    TrainVal = 3
    Test = 4


class _Base:
    pass


class OnlineVoxelizationDatasetBase:
    pass


_MODS = {}
# the stand-in and staged modules, in sys.modules while the original runs (it imports `lib.dataset` inside a function)
_STUBS = {}


def load():
    """The staged (utils, scannet, stanford) modules."""
    if _MODS:
        return _MODS["utils"], _MODS["scannet"], _MODS["stanford"]
    lib = types.ModuleType("lib")
    lib.__path__ = [stage_ref.path("semseg/lib")]
    datasets = types.ModuleType("lib.datasets")
    datasets.__path__ = [stage_ref.path("semseg/lib", "datasets")]
    stubs = {"lib": lib, "lib.datasets": datasets, "omegaconf": _module("omegaconf"), "plyfile": _module("plyfile"),
             "lib.distributed_utils": _module("lib.distributed_utils", get_world_size=lambda: 1, get_rank=lambda: 0),
             "lib.transforms": _module("lib.transforms"),
             "lib.pc_utils": _module("lib.pc_utils", read_plyfile=_read_plyfile, save_point_cloud=lambda *a, **k: None,
                                     colorize_pointcloud=None),
             "lib.dataset": _module("lib.dataset", VoxelizationDataset=_Base, DatasetPhase=DatasetPhase, cache=lambda f: f,
                                    str2datasetphase_type=lambda s: DatasetPhase[s], OnlineVoxelizationDatasetBase=OnlineVoxelizationDatasetBase)}
    _STUBS.update(stubs)
    staged = (("utils", "lib.utils", "utils.py"), ("scannet", "lib.datasets.scannet", "datasets/scannet.py"),
              ("stanford", "lib.datasets.stanford", "datasets/stanford.py"))
    with stage_ref.installed({**_STUBS, **{full: None for _, full, _ in staged}}):
        for name, full, f in staged:
            spec = importlib.util.spec_from_file_location(full, stage_ref.path("semseg/lib", f))
            m = importlib.util.module_from_spec(spec)
            sys.modules[full] = m
            spec.loader.exec_module(m)
            _MODS[name] = m
            _STUBS[full] = m
    return _MODS["utils"], _MODS["scannet"], _MODS["stanford"]


@contextlib.contextmanager
def _np_int():
    had = hasattr(np, "int")
    if not had:
        np.int = int
    try:
        yield
    finally:
        if not had:
            del np.int


def _recording(module, sink):
    inner = module.fast_hist

    def fast_hist(pred, label, n):
        h = inner(pred, label, n)
        sink.append(np.asarray(h, np.int64))
        return h
    module.fast_hist = fast_hist
    return inner


def _lut(label_map):
    lut = np.full(max(label_map) + 1, -1, np.int64)
    for k, v in label_map.items():
        lut[k] = v
    return lut


def dataset(kind, data_root, data_paths, label_map, num_labels):
    """An instance of the staged ScanNet (`kind == "scannet"`) or S3DIS dataset class with what the evaluation reads."""
    _, scannet, stanford = load()
    cls = scannet.ScannetVoxelizationDataset if kind == "scannet" else stanford.StanfordDataset
    ds = cls.__new__(cls)
    ds.data_paths, ds.data_root, ds.label_map, ds.NUM_LABELS = list(data_paths), Path(data_root), dict(label_map), int(num_labels)
    ds.IS_ONLINE_VOXELIZATION, ds.IS_TEMPORAL = True, False
    if kind != "scannet":
        ds.label2masked = _lut(label_map)
        ds.load_ply = lambda i: (_read_plyfile(os.path.join(data_root, ds.data_paths[i])).astype(np.float64),)
    return ds


def save_predictions(coords_batch_first, pred, transformation, ds, iteration, save_pred_dir):
    """The original `save_predictions` on batch-first coords (int [N, 4]), masked pred (int [N]) and transformation rows [B, 17]."""
    import torch
    utils, _, _ = load()
    c = np.asarray(coords_batch_first)
    coords = torch.from_numpy(np.ascontiguousarray(np.concatenate([c[:, 1:4], c[:, :1]], 1)))
    with _np_int(), stage_ref.installed(_STUBS):
        utils.save_predictions(coords, np.asarray(pred, np.int64), torch.as_tensor(np.asarray(transformation, np.float32)), ds, None,
                               iteration, save_pred_dir)


def test_pointcloud(ds, pred_dir):
    """The original `ds.test_pointcloud(pred_dir)`; returns the histograms it bins, in order (int64 [C, C] each)."""
    _, scannet, stanford = load()
    module = scannet if isinstance(ds, scannet.ScannetVoxelizationDataset) else stanford
    sink = []
    inner = _recording(module, sink)
    try:
        with _np_int(), stage_ref.installed(_STUBS):
            ds.test_pointcloud(pred_dir)
    finally:
        module.fast_hist = inner
    return sink
