"""VoteNet's detection data on the GPU (DESIGN.md 8f-13): the ScanNet and SUN RGB-D training sets of
`downstream/votenet_det_new/lib/datasets/{scannet/scannet_detection_dataset.py, sunrgbd/sunrgbd_detection_dataset.py}` with their
`__getitem__` run for a whole batch by libpcb200 (csrc/det_data.cu) instead of one numpy call per item in `DataLoader` workers.

    DC = ScannetDatasetConfig()                                   # the original's config object (nyu40ids, mean_size_arr, ...)
    ds = ScannetDetectionDataset("train", 40000, use_height=False, augment=True, data_path=".../scannet_train_detection_data",
                                 split_file=".../scannetv2_train.txt", dataset_config=DC)
    loader = DetectionLoader(ds, batch_size=32, shuffle=True, voxel_size=0.025)   # replaces DataLoader(...) in ddp_main.py
    for batch in loader: ...                                      # lib/train.py unmodified: every value is already a device tensor

Each batch is one pass of a handful of launches: floor heights, choice sets, the fused point pass (with the ScanNet instance votes) and
the box labels.  Scenes stay ragged (per-scene row offsets); the host reads the next batch's files on a thread (SUN RGB-D inflates its
npz files on a pool) while the GPU works, and each array goes up in one pinned copy.

Randomness (`semseg_data.Draws` / `ReplayDraws`): the scalar draws stay on the host, from `np.random.random()` / `np.random.random(3)`
(`Draws.rand`) in the original's order per scene -- ScanNet: x flip, y flip, rotation angle; SUN RGB-D: flip, rotation angle, two
`random(3)` when `use_color`, scale.  The array draws come from the device generator: the choice sets of all scenes in one
`Draws.choices` call (after every scene's scalars), and SUN RGB-D's per-point jitter and colour-dropout arrays (`Draws.rand_device`,
after the scene's two `random(3)`).  Moving the array draws to the device changes which host scalars a given `np.random` seed yields;
the distribution is the same.  Exact parity with a seeded original is by replay only: a `ReplayDraws` holding the original's draws in
this order reproduces its items.
"""
import io
import logging
import os
import zipfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib, detection
from ._lib import check, lib, ptr, stream, workspace
from .semseg_data import _draws

MAX_NUM_OBJ = 64
_POOL_THREADS = 16


def _pinned(arrays, dtype, shape_tail, device):
    """The row-wise concatenation of numpy arrays as ONE host-to-device copy through pinned staging."""
    n = sum(len(a) for a in arrays)
    host = torch.empty((n,) + shape_tail, dtype=dtype, pin_memory=True)
    if n:
        np.concatenate([np.asarray(a).reshape((len(a),) + shape_tail) for a in arrays], out=host.numpy())
    return host.to(device, non_blocking=True)


def _offsets(lengths):
    off = np.zeros(len(lengths) + 1, np.int64)
    off[1:] = np.cumsum(lengths)
    return off


def _read_npz(path, key):
    """One array of a `savez_compressed` file: the member is inflated by a single zlib call, which runs without the GIL (numpy's own
    reader inflates it in small chunks)."""
    with zipfile.ZipFile(path) as z:
        return np.load(io.BytesIO(z.read(key + ".npy")))


def floor_height(z, offsets):
    """np.percentile(scene z, 0.99) of every scene, float64 numpy [B] (synchronises).  z: fp32 or fp64 CUDA [M] or a column view of
    [M, C] rows; offsets: int64 numpy [B + 1] (scene b is rows [offsets[b], offsets[b+1]))."""
    _lib.require_cuda(z)
    off = np.ascontiguousarray(offsets, np.int64)
    stride = z.stride(0) if z.dim() == 1 else None
    if stride is None or z.dtype not in (torch.float32, torch.float64):
        raise ValueError("z must be a 1-d fp32 or fp64 view")
    out = torch.empty(len(off) - 1, dtype=torch.float64, device=z.device)
    with torch.cuda.device(z.device):
        check(lib.pcb_det_floor_height(z.data_ptr(), stride, int(z.dtype == torch.float64), off.ctypes.data,
                                       ptr(torch.from_numpy(off).to(z.device)), len(off) - 1, ptr(out), stream()))
    return out


class _DetectionDataset:
    """What both datasets share: the batched `__getitem__` (`_assemble`) and the host file reads."""
    SUN = False

    def __len__(self):
        return len(self.scan_names)

    def __getitem__(self, idx):
        """The original's item dict as device tensors: the batched kernels with B = 1."""
        batch = self._assemble(self._read_batch([idx]), [idx])
        return {k: v[0] for k, v in batch.items()}

    def _pool(self):
        if getattr(self, "_executor", None) is None:
            self._executor = ThreadPoolExecutor(_POOL_THREADS)
        return self._executor

    def _read_batch(self, idxs):
        return list(self._pool().map(self._read, [self.scan_names[i] for i in idxs]))

    def _setup(self, num_points, use_color, use_height, augment, data_path, dataset_config, device, draws):
        self.num_points, self.use_color, self.use_height, self.augment = int(num_points), use_color, use_height, augment
        self.data_path, self.dc, self.draws = data_path, dataset_config, draws
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._executor = None
        self._mean_size = np.ascontiguousarray(dataset_config.mean_size_arr, np.float64).reshape(-1, 3)

    def _assemble(self, items, idxs):
        B, k, dev, sun = len(items), self.num_points, self.device, self.SUN
        key = "pc" if sun else "vert"
        ns = [len(it[key]) for it in items]
        ks = [len(it["bbox"]) for it in items]
        for n, K, i in zip(ns, ks, idxs):
            if n < 1:
                raise ValueError(f"scene {self.scan_names[i]} has no points")
            if K > MAX_NUM_OBJ:
                raise ValueError(f"scene {self.scan_names[i]} has {K} boxes, more than MAX_NUM_OBJ = {MAX_NUM_OBJ}")
        boxes = [np.asarray(it["bbox"], np.float64).reshape(-1, 8 if sun else 7) for it in items]
        allb = np.concatenate(boxes) if boxes else np.zeros((0, 8 if sun else 7))
        if sun:
            cls = allb[:, 7]
            if ((cls != np.floor(cls)) | (cls < 0) | (cls >= len(self.dc.type2class))).any():
                raise ValueError("a box class is not a class of the dataset config")     # the original's KeyError
        elif not np.isin(allb[:, 6], self.nyu40ids).all():
            raise ValueError("a box's nyu40 id is not in dataset_config.nyu40ids")          # the original's IndexError
        d = _draws(self.draws)
        params = np.zeros((B, _lib.DET_NPARAM), np.float64)
        headings, jitter, dropout = [], [], []
        for b in range(B):
            p = params[b]
            if self.augment and not sun:
                p[0] = float(d.rand()) > 0.5
                p[1] = float(d.rand()) > 0.5
                angle = (float(d.rand()) * np.pi / 18) - np.pi / 36                  # -5 ... +5 degrees
                p[2], p[3] = np.cos(angle), np.sin(angle)
            elif self.augment:
                p[0] = float(d.rand()) > 0.5
                angle = (float(d.rand()) * np.pi / 3) - np.pi / 6                    # -30 ... +30 degrees
                p[2], p[3] = np.cos(angle), np.sin(angle)
                if self.use_color:
                    p[5:8] = 1 + 0.4 * np.asarray(d.rand(3)) - 0.2
                    p[8:11] = 0.1 * np.asarray(d.rand(3)) - 0.05
                    jitter.append(d.rand_device(ns[b]))
                    dropout.append(d.rand_device(ns[b]))
                p[4] = float(d.rand()) * 0.3 + 0.85
            if sun:      # the augmented heading (numpy evaluates its cos / sin, so the device sees the original's values)
                h = boxes[b][:, 6].copy()
                if self.augment:
                    if p[0]:
                        h = np.pi - h
                    h -= angle
                headings.append(np.stack([h, np.cos(-1 * h), np.sin(-1 * h)], 1))
        choices = d.choices(ns, k)
        off, boff = _offsets(ns), _offsets(ks)
        a = _lib.PcbDetBatch()
        a.B, a.M, a.num_points = B, int(off[-1]), k
        a.dataset = _lib.DET_SUNRGBD if sun else _lib.DET_SCANNET
        a.flags = ((_lib.DET_HEIGHT if self.use_height else 0) | (_lib.DET_COLOR if self.use_color else 0) |
                   (_lib.DET_AUGMENT if self.augment else 0))
        keep = [choices]                                 # device tensors whose pointers the launches read
        with torch.cuda.device(dev):
            def up(arrays, dtype, tail=()):
                t = _pinned(arrays, dtype, tail, dev)
                keep.append(t)
                return ptr(t)
            a.offsets_host, a.offsets = off.ctypes.data, up([off], torch.int64)
            a.box_offsets_host, a.box_offsets = boff.ctypes.data, up([boff], torch.int64)
            a.params = up([params], torch.float64, (_lib.DET_NPARAM,))
            a.choices = ptr(choices)
            a.mean_size, a.n_size = up([self._mean_size], torch.float64, (3,)), len(self._mean_size)
            a.num_heading_bin = int(self.dc.num_heading_bin)
            a.boxes = up(boxes, torch.float64, (8 if sun else 7,))
            C = 3 + (3 if self.use_color else 0) + (1 if self.use_height else 0)
            out = {"point_clouds": torch.empty(B, k, C, dtype=torch.float32, device=dev),
                   "center_label": torch.empty(B, MAX_NUM_OBJ, 3, dtype=torch.float32, device=dev),
                   "heading_class_label": torch.empty(B, MAX_NUM_OBJ, dtype=torch.int64, device=dev),
                   "heading_residual_label": torch.empty(B, MAX_NUM_OBJ, dtype=torch.float32, device=dev),
                   "size_class_label": torch.empty(B, MAX_NUM_OBJ, dtype=torch.int64, device=dev),
                   "size_residual_label": torch.empty(B, MAX_NUM_OBJ, 3, dtype=torch.float32, device=dev),
                   "sem_cls_label": torch.empty(B, MAX_NUM_OBJ, dtype=torch.int64, device=dev),
                   "box_label_mask": torch.empty(B, MAX_NUM_OBJ, dtype=torch.float32, device=dev),
                   "vote_label": torch.empty(B, k, 9, dtype=torch.float32, device=dev),
                   "vote_label_mask": torch.empty(B, k, dtype=torch.int64, device=dev),
                   "scan_idx": torch.as_tensor(np.asarray(idxs, np.int64)).to(dev)}
            if sun:
                a.pc = up([it["pc"] for it in items], torch.float64, (6,))
                a.votes = up([it["votes"] for it in items], torch.float64, (10,))
                a.headings = up(headings, torch.float64, (3,))
                if jitter:
                    j, dr = torch.cat(jitter), torch.cat(dropout)
                    keep += [j, dr]
                    a.jitter, a.dropout = ptr(j), ptr(dr)
                out["max_gt_bboxes"] = torch.empty(B, MAX_NUM_OBJ, 8, dtype=torch.float64, device=dev)
                z, zstride = a.pc + 2 * 8, 6
            else:
                a.vert = up([it["vert"] for it in items], torch.float32, (6,))
                a.sem = up([it["sem"].view(np.int32) for it in items], torch.int32)
                a.ins = up([it["ins"].view(np.int32) for it in items], torch.int32)
                a.nyu40ids, a.n_ids = up([self.nyu40ids], torch.int64), len(self.nyu40ids)
                out["pcl_color"] = torch.empty(B, k, 3, dtype=torch.float32, device=dev)
                z, zstride = a.vert + 2 * 4, 6
            if self.use_height:
                fl = torch.empty(B, dtype=torch.float64, device=dev)
                keep.append(fl)
                check(lib.pcb_det_floor_height(z, zstride, int(sun), a.offsets_host, a.offsets, B, ptr(fl), stream()))
                a.floor = ptr(fl)
            for name in ("point_clouds", "pcl_color", "vote_label", "vote_label_mask", "center_label", "heading_class_label",
                         "heading_residual_label", "size_class_label", "size_residual_label", "sem_cls_label", "box_label_mask",
                         "max_gt_bboxes"):
                if name in out:
                    setattr(a, name, ptr(out[name]))
            wsb = lib.pcb_det_points_ws_bytes(B, k)
            ws = workspace(wsb, dev)
            check(lib.pcb_det_points(a, ptr(ws), wsb, stream()))
            check(lib.pcb_det_boxes(a, stream()))
        return out


class ScannetDetectionDataset(_DetectionDataset):
    """`lib/datasets/scannet/scannet_detection_dataset.py` on the device.  `data_path`: the folder of `<scene>_{vert,sem_label,ins_label,
    bbox}.npy` files; `split_file`: `scannetv2_<split>.txt`; `dataset_config`: the original's `ScannetDatasetConfig()` (nyu40ids,
    mean_size_arr, num_heading_bin).  `use_color=True` raises ValueError: the original fails there (NameError on pcl_color)."""

    def __init__(self, split_set="train", num_points=20000, use_color=False, use_height=False, augment=False, data_ratio=1.0,
                 data_path=None, split_file=None, dataset_config=None, device="cuda", draws=None):
        if use_color:
            raise ValueError("ScannetDetectionDataset: use_color=True is not supported (the original raises NameError on pcl_color)")
        if split_set not in ("train", "val", "test"):
            raise ValueError(f"illegal split name {split_set!r}")
        if data_path is None or split_file is None or dataset_config is None:
            raise ValueError("data_path, split_file and dataset_config are required")
        all_scan_names = set(os.path.basename(x)[0:12] for x in os.listdir(data_path) if x.startswith("scene"))
        with open(split_file) as f:
            names = f.read().splitlines()
        num_scans = len(names)
        names = [s for s in names if s in all_scan_names]
        self.scan_names = names[:int(len(names) * data_ratio)]
        logging.info("kept {} scans out of {}".format(len(self.scan_names), num_scans))
        self._setup(num_points, use_color, use_height, augment, data_path, dataset_config, device, draws)
        self.nyu40ids = np.ascontiguousarray(dataset_config.nyu40ids, np.int64)

    def _read(self, name):
        p = os.path.join(self.data_path, name)
        return {"vert": np.ascontiguousarray(np.load(p + "_vert.npy"), np.float32),
                "ins": np.ascontiguousarray(np.load(p + "_ins_label.npy"), np.uint32),
                "sem": np.ascontiguousarray(np.load(p + "_sem_label.npy"), np.uint32),
                "bbox": np.load(p + "_bbox.npy")}


class SunrgbdDetectionVotesDataset(_DetectionDataset):
    """`lib/datasets/sunrgbd/sunrgbd_detection_dataset.py` on the device.  `data_path`: the folder of `<scan>_{pc.npz, bbox.npy,
    votes.npz}` files (the original's `sunrgbd_pc_bbox_votes_50k_v{1,2}_<split>`); `dataset_config`: the original's
    `SunrgbdDatasetConfig()` (num_heading_bin, mean_size_arr, type2class)."""
    SUN = True

    def __init__(self, split_set="train", num_points=20000, use_color=False, use_height=False, use_v1=False, augment=False,
                 scan_idx_list=None, data_ratio=1.0, data_path=None, dataset_config=None, device="cuda", draws=None):
        if num_points > 50000:
            raise ValueError(f"num_points {num_points} > 50000")
        if data_path is None or dataset_config is None:
            raise ValueError("data_path and dataset_config are required")
        self.use_v1 = use_v1
        self.scan_names = sorted(set(os.path.basename(x)[0:6] for x in os.listdir(data_path)))
        if scan_idx_list is not None:
            self.scan_names = [self.scan_names[i] for i in scan_idx_list]
        self.scan_names = self.scan_names[:int(len(self.scan_names) * data_ratio)]
        self._setup(num_points, use_color, use_height, augment, data_path, dataset_config, device, draws)

    def _read(self, name):
        p = os.path.join(self.data_path, name)
        return {"pc": np.ascontiguousarray(_read_npz(p + "_pc.npz", "pc"), np.float64),
                "votes": np.ascontiguousarray(_read_npz(p + "_votes.npz", "point_votes"), np.float64), "bbox": np.load(p + "_bbox.npy")}


class DetectionLoader:
    """`DataLoader(dataset, batch_size, shuffle)` for the two datasets above (`ddp_main.py`): `len()` batches, a fresh `torch.randperm`
    order per pass when `shuffle`, the last batch short.  Each batch is a dict of device tensors with the keys, dtypes and shapes of
    `default_collate` over the original's items.  With `voxel_size`, `detection.voxelize_batch` adds the voxel fields (the original's
    `VoxelizationDataset` + `collate_fn`); only [B, N, 3] clouds can be voxelised."""

    def __init__(self, dataset, batch_size, shuffle, voxel_size=None, draws=None):
        if voxel_size is not None and (dataset.use_color or dataset.use_height):
            raise ValueError("voxel_size needs [B, N, 3] point clouds (use_color=False, use_height=False)")
        self.dataset, self.batch_size, self.shuffle, self.voxel_size = dataset, int(batch_size), shuffle, voxel_size
        if draws is not None:
            dataset.draws = draws

    def __len__(self):
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        n = len(self.dataset)
        order = torch.randperm(n).tolist() if self.shuffle else list(range(n))
        batches = [order[i:i + self.batch_size] for i in range(0, n, self.batch_size)]
        if not batches:
            return
        with ThreadPoolExecutor(1) as reader:            # batch i + 1's files are read while the GPU works on batch i
            pending = reader.submit(self.dataset._read_batch, batches[0])
            for i, idxs in enumerate(batches):
                items = pending.result()
                if i + 1 < len(batches):
                    pending = reader.submit(self.dataset._read_batch, batches[i + 1])
                batch = self.dataset._assemble(items, idxs)
                if self.voxel_size is not None:
                    detection.voxelize_batch(batch, self.voxel_size)
                yield batch
