"""VoteNet detection data: the staged original `Dataset` + its voxelisation under `DataLoader(num_workers=8)` against
pointcontrast_b200.det_data.DetectionLoader, at the two finetuning scripts' workloads (ScanNet B 32, 40 000 points from ~50 000-vertex
scenes with ~30 instances; SUN RGB-D B 64, 20 000 points from 50 000-point scenes with ~10 boxes; both `data.voxel_size=0.025`,
no colour, no height), on synthetic scenes written to a temporary directory.

    python profiles/bench_det_data.py [--batches 6] [--rounds 3]

Per-batch wall time at steady state (the two legs alternate, `--rounds` times); the split of one library batch into its host file
reads, the host side of assembling it (to a device synchronise), the device time of its kernels alone and of its host-to-device copies
(torch.profiler); the host CPU time per batch of each leg (this process plus the workers that have exited: the original's persistent
workers are not counted), one VoteNet training step for scale, and the card's name and power
limit read in the same run.  The training step runs on the first STEP_SCENES scenes of a batch (a full 32-scene ScanNet batch
does not fit one card next to the two loaders).  The original's `sparse_quantize` is MinkowskiEngine's; it is absent, so its restatement in
oracle/detection_cpu.py runs per item in the workers.  Prints one JSON line.
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import det_data_ref, detection_cpu  # noqa: E402
from pointcontrast_b200 import det_data, detection, synth  # noqa: E402

WORKLOADS = {"scannet": (32, 40000), "sunrgbd": (64, 20000)}
STEP_SCENES = 8


class OriginalItems(torch.utils.data.Dataset):
    """The original `__getitem__` plus the voxelisation its `VoxelizationDataset` adds per item."""

    def __init__(self, cls, path, names, num_points):
        self.ds = cls.__new__(cls)
        self.ds.data_path, self.ds.scan_names, self.ds.num_points = path, names, num_points
        self.ds.use_color, self.ds.use_height, self.ds.augment = False, False, True

    def __len__(self):
        return len(self.ds.scan_names)

    def __getitem__(self, i):
        item = self.ds[i]
        c, ind, _ = detection_cpu.voxelize_scenes(item["point_clouds"][None], 0.025)
        item["voxel_coords"], item["voxel_inds"] = c[:, 1:], ind
        return item


def collate(items):
    vc = np.concatenate([np.concatenate([np.full((len(it["voxel_coords"]), 1), b, np.int32), it["voxel_coords"]], 1)
                         for b, it in enumerate(items)])
    vi = np.concatenate([it["voxel_inds"] for it in items])
    for it in items:
        del it["voxel_coords"], it["voxel_inds"]
    out = torch.utils.data.default_collate(items)
    out["voxel_coords"], out["voxel_inds"] = torch.from_numpy(vc), torch.from_numpy(vi)
    return out


def cpu_seconds():
    s, c = resource.getrusage(resource.RUSAGE_SELF), resource.getrusage(resource.RUSAGE_CHILDREN)
    return s.ru_utime + s.ru_stime + c.ru_utime + c.ru_stime


def run_leg(loader, batches, to_device):
    it = iter(loader)
    next(it)                                       # first batch: worker start-up / warm-up
    torch.cuda.synchronize()
    t0, c0 = time.perf_counter(), cpu_seconds()
    for _ in range(batches):
        b = next(it)
        if to_device:
            b = {k: v.cuda(non_blocking=True) for k, v in b.items()}
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) / batches, (cpu_seconds() - c0) / batches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    mods = det_data_ref.load()
    assert mods is not None and torch.cuda.is_available(), "needs the staged original and a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = {"gpu": q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0), "batches": args.batches,
           "rounds": args.rounds}
    for name, (B, k) in WORKLOADS.items():
        with tempfile.TemporaryDirectory() as d:
            n_scenes = B * (args.batches + 1)
            names = [f"scene{i:04d}_00" if name == "scannet" else f"{i + 1:06d}" for i in range(n_scenes)]
            uniq = 8                                    # distinct synthetic scenes, repeated under other names
            for i, s in enumerate(names):
                if name == "scannet":
                    synth.write_scannet_detection_scene(d, s, i % uniq, 50000, 20 + i % 10, n_inst=30)
                else:
                    synth.write_sunrgbd_detection_scene(d, s, i % uniq, 50000, 8 + i % 5)
            if name == "scannet":
                split = os.path.join(d, "split.txt")
                open(split, "w").write("\n".join(names) + "\n")
                ds = det_data.ScannetDetectionDataset("train", k, augment=True, data_path=d, split_file=split,
                                                      dataset_config=mods[0].DC)
                cls, dc = mods[0].ScannetDetectionDataset, mods[0].DC
            else:
                ds = det_data.SunrgbdDetectionVotesDataset("train", k, augment=True, data_path=d, dataset_config=mods[1].DC)
                cls, dc = mods[1].SunrgbdDetectionVotesDataset, mods[1].DC
            gpu_loader = det_data.DetectionLoader(ds, B, shuffle=True, voxel_size=0.025)
            ref_loader = torch.utils.data.DataLoader(OriginalItems(cls, d, names, k), batch_size=B, shuffle=True, num_workers=8,
                                                     collate_fn=collate, persistent_workers=True)
            walls = {"original": [], "library": []}
            cpus = {"original": [], "library": []}
            for _ in range(args.rounds):
                w, c = run_leg(ref_loader, args.batches, True)
                walls["original"].append(w); cpus["original"].append(c)
                w, c = run_leg(gpu_loader, args.batches, False)
                walls["library"].append(w); cpus["library"].append(c)
            # the split of one batch: host file reads (and SUN RGB-D's inflation), the host side of `_assemble` + voxelisation
            # (draws, checks, pinned staging, launches) timed to a device synchronise, and the device time of its kernels and of
            # its host-to-device copies from torch.profiler
            idxs = list(range(B))
            read_ms, assemble_ms, kernel_ms, h2d_ms = [], [], [], []
            items = ds._read_batch(idxs)
            detection.voxelize_batch(ds._assemble(items, idxs), 0.025)
            for _ in range(5):
                t0 = time.perf_counter()
                items = ds._read_batch(idxs)
                read_ms.append((time.perf_counter() - t0) * 1e3)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                batch = ds._assemble(items, idxs)
                detection.voxelize_batch(batch, 0.025)
                torch.cuda.synchronize()
                assemble_ms.append((time.perf_counter() - t0) * 1e3)
            for _ in range(3):
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    batch = ds._assemble(items, idxs)
                    detection.voxelize_batch(batch, 0.025)
                    torch.cuda.synchronize()
                dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                copies = [e for e in dev if "memcpy" in e.name.lower() or "memset" in e.name.lower()]
                h2d_ms.append(sum(e.time_range.elapsed_us() for e in copies if "htod" in e.name.lower()) / 1e3)
                kernel_ms.append(sum(e.time_range.elapsed_us() for e in dev if e not in copies) / 1e3)
            # one VoteNet training step for scale
            from oracle import det_loss_ref
            step_ms = net = sub = None
            if det_loss_ref.available():
                import importlib
                from pointcontrast_b200 import det_loss, me, pointnet2
                from oracle import detection_ref
                me.install(); pointnet2.install()
                if detection_ref.ROOT not in sys.path:
                    sys.path.insert(0, detection_ref.ROOT)
                votenet = importlib.import_module("models.votenet")
                net = votenet.VoteNet(dc.num_class, dc.num_heading_bin, dc.num_size_cluster, dc.mean_size_arr, input_feature_dim=0,
                                      num_proposal=256, vote_factor=1, sampling="vote_fps", backbone="sparseconv").cuda().train()
                sub = {k2: v[:STEP_SCENES] for k2, v in batch.items() if not k2.startswith("voxel")}
                detection.voxelize_batch(sub, 0.025)
                batch = sub
                times = []
                for i in range(4):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ep = net({k2: batch[k2] for k2 in ("point_clouds", "voxel_coords", "voxel_inds", "voxel_feats")})
                    for k2, v in batch.items():
                        ep.setdefault(k2, v)
                    loss, _ = det_loss.get_loss(ep, dc)
                    loss.backward()
                    torch.cuda.synchronize()
                    if i:
                        times.append((time.perf_counter() - t0) * 1e3)
                step_ms = float(np.median(times))
            res[name] = {"B": B, "num_points": k,
                         "batch_ms_original": [round(w * 1e3, 2) for w in walls["original"]],
                         "batch_ms_library": [round(w * 1e3, 2) for w in walls["library"]],
                         "cpu_s_per_batch_original": [round(c, 3) for c in cpus["original"]],
                         "cpu_s_per_batch_library": [round(c, 3) for c in cpus["library"]],
                         "read_ms_per_batch": [round(v, 1) for v in read_ms],
                         "assemble_ms_per_batch": [round(v, 1) for v in assemble_ms],
                         "kernel_ms_per_batch": [round(v, 3) for v in kernel_ms], "h2d_ms_per_batch": [round(v, 3) for v in h2d_ms],
                         "train_step_ms": step_ms, "train_step_scenes": STEP_SCENES}
            del net, batch, sub
            torch.cuda.empty_cache()
            del ref_loader
    print(json.dumps(res))


if __name__ == "__main__":
    main()
