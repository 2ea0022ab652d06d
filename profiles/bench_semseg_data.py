"""Times the semseg finetune data path (pointcontrast_b200/semseg_data.py) per scene at ScanNet 2 cm sizes and sets it against the
finetune step it feeds.  Prints one JSON line.

    python profiles/bench_semseg_data.py [--sizes 150000 300000] [--batch 6]

* gpu_ms: one training item of `ScannetVoxelization2cmDataset` (PLY read, elastic distortion, rotation / scale / floor, label-aware
  voxelisation, dropout, flip, colour augmentation, label map), synthetic rooms of N raw points written to a temporary directory;
  CUDA events around a window of >= 1 s after warm-up (the pipeline synchronises inside, so the window is wall time on the GPU).
* cpu_oracle_ms: the numpy / scipy oracle (oracle/semseg_data_cpu.py) on the same scene with the draws the GPU run took, once; its
  output is compared with the GPU's (`oracle_match`).
* step_ms: one `SegmentationTrainer.train_step` (Res16UNet34C, 20 classes, iter_size 1) on a batch of `--batch` scenes of the
  smallest size, CUDA events over >= 1 s; `loader_share` = batch x gpu_ms / step_ms (the data path runs on the same GPU).
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import semseg_data_cpu as O  # noqa: E402
from pointcontrast_b200 import semseg, semseg_data as S, synth  # noqa: E402
from pointcontrast_b200.model import load_model  # noqa: E402
from tests import refload  # noqa: E402
from tests.helpers import det_init  # noqa: E402


class RecordingDraws(S.Draws):
    """The default draws, each also kept (device arrays copied to the host) for the oracle's replay."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.rec = []

    def random(self):
        v = super().random(); self.rec.append(("random", v)); return v

    def uniform(self, lo, hi):
        v = super().uniform(lo, hi); self.rec.append(("uniform", v)); return v

    def rand(self, *shape):
        v = super().rand(*shape); self.rec.append(("rand", v)); return v

    def shuffle(self, x):
        perm = list(range(len(x)))
        super().shuffle(perm)
        y = list(x)
        x[:] = [y[i] for i in perm]
        self.rec.append(("shuffle", np.array(perm)))

    def randn(self, shape, dtype):
        v = super().randn(shape, dtype); self.rec.append(("randn", v.cpu().numpy())); return v

    def choice(self, n, k):
        v = super().choice(n, k); self.rec.append(("choice", v.cpu().numpy())); return v


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"name": torch.cuda.get_device_name(), "nvidia_smi": q}


def timed(fn, min_s=1.0, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, t0 = 0, time.perf_counter()
    a.record()
    while time.perf_counter() - t0 < min_s:
        fn()
        n += 1
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[150_000, 300_000])
    ap.add_argument("--batch", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    torch.cuda.set_device(0)
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    cfg = refload.Cfg(data=dict(ignore_label=255, return_transformation=False),
                      augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
                      optimizer=dict(optimizer="SGD", lr=0.8, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=1,
                                     scheduler="PolyLR", max_iter=60000, poly_power=0.9))
    res = {"card": card(), "sizes": {}}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "splits"))
        loaders = {}
        for n in args.sizes:
            names = []
            for k in range(args.batch):
                xyz, rgb, lab = synth.synth_labelled_room(1000 * k + n % 997, n, scale=1.6)       # about 5 x 5 x 3.8 m
                name = f"scene{n}_{k}.ply"
                synth.write_ply(os.path.join(tmp, name), xyz, rgb, lab)
                names.append(name)
            with open(os.path.join(tmp, "splits", "scannetv2_train.txt"), "w") as f:
                f.write("\n".join(names) + "\n")
            cfg["data"]["scannet_path"] = tmp
            draws = RecordingDraws("cuda")
            loader = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "train", shuffle=False, augment_data=True,
                                              batch_size=args.batch, limit_numpoints=0, normalize_color=True, draws=draws,
                                              split_dir=os.path.join(tmp, "splits"))
            ds = loader.dataset
            loaders[n] = loader
            idx = [0]

            def one():
                ds[idx[0] % len(ds)]
                idx[0] += 1

            ms, reps = timed(one)
            # the oracle on scene 0 with the draws of a fresh GPU run
            draws.rec.clear()
            c, f, l = (t.cpu().numpy() for t in ds[0])
            data = S.read_ply(os.path.join(tmp, names[0]))
            xyz = np.array([data["x"], data["y"], data["z"]], np.float32).T
            rgb = np.array([data["red"], data["green"], data["blue"]], np.float32).T
            t0 = time.perf_counter()
            out = O.run_scene(xyz, rgb, np.array(data["label"], np.int32), O.SCANNET_2CM, O.Replay(draws.rec))
            cpu_ms = (time.perf_counter() - t0) * 1e3
            match = bool((out["coords"] == c).all() and (out["labels"] == l).all() and np.array_equal(out["feats"], f)) \
                if out["coords"].shape == c.shape else False
            res["sizes"][str(n)] = {"gpu_ms": round(ms, 3), "gpu_reps": reps, "voxels": int(len(c)), "cpu_oracle_ms": round(cpu_ms, 1),
                                    "oracle_match": match, "gpu_scenes_per_s": round(1e3 / ms, 1)}
        # the finetune step on a batch of the smallest scenes
        n0 = min(args.sizes)
        batch = next(iter(loaders[n0]))
        mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
        net = load_model("Res16UNet34C")(3, 20, mcfg, D=3)
        det_init(net, 0)
        tr = semseg.SegmentationTrainer(net, cfg)
        step_ms, steps = timed(lambda: tr.train_step(batch), warmup=2)
        gpu0 = res["sizes"][str(n0)]["gpu_ms"]
        res.update(step_ms=round(step_ms, 2), step_reps=steps, batch=args.batch, batch_voxels=int(len(batch[0][0])),
                   step_scenes_per_s=round(args.batch * 1e3 / step_ms, 1), loader_share=round(args.batch * gpu0 / step_ms, 3))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
