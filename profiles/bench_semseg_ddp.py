"""Times the data-parallel semantic-segmentation finetune step at `train_scannet.sh`'s shape: Res16UNet34C, 20 classes, `--batch` (6)
synthetic ScanNet-sized rooms per rank at 2 cm, iter_size 1, SGD lr 0.8 under PolyLR.  One JSON line per rank.

    python profiles/bench_semseg_ddp.py [--steps 20] [--warmup 5]                  # one GPU
    torchrun --nproc_per_node N profiles/bench_semseg_ddp.py                       # N GPUs over NCCL, one rank per GPU

* step_ms: `SegmentationTrainer.train_step` on this rank's batch (built once by the GPU data path, reused every step), CUDA events
  around `--steps` steps after `--warmup`;
* world > 1, one instrumented step: allreduce_ms, the time the gradient all-reduces occupy the side stream (the two chunks launched
  during the backward sweep and the tail; includes waiting for the slowest rank), and exposed_wait_plus_sgd_ms, from the end of this
  rank's backward sweep to the end of its step (the tail all-reduce, the wait for every chunk, the SGD kernel).
The card's name and power limit are read in the same run.  `--package DIR` imports `pointcontrast_b200` from DIR instead of this
repository (another checkout to compare with, built).
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"name": torch.cuda.get_device_name(), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=6)
    ap.add_argument("--points", type=int, default=200_000, help="raw points per synthetic room")
    ap.add_argument("--package", default=None, help="directory holding the pointcontrast_b200 package to time")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    if args.package:
        sys.path.insert(0, os.path.abspath(args.package))
    from pointcontrast_b200 import semseg, semseg_data as S, synth
    from pointcontrast_b200.model import load_model
    from tests import refload
    from tests.helpers import det_init
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    world, rank = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    if world > 1:
        dist.init_process_group("nccl")
    random.seed(rank); np.random.seed(rank); torch.manual_seed(rank)            # the augmentation's draws: the same batch every run
    cfg = refload.Cfg(data=dict(ignore_label=255, return_transformation=False),
                      augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
                      optimizer=dict(optimizer="SGD", lr=0.8, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=1,
                                     scheduler="PolyLR", max_iter=60000, poly_power=0.9))
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "splits"))
        names = []
        for k in range(args.batch):
            seed = 1000 * (args.batch * rank + k) + 7
            xyz, rgb, lab = synth.synth_labelled_room(seed, args.points, scale=1.6)         # about 5 x 5 x 3.8 m
            names.append(f"scene{k}.ply")
            synth.write_ply(os.path.join(tmp, names[-1]), xyz, rgb, lab)
        with open(os.path.join(tmp, "splits", "scannetv2_train.txt"), "w") as f:
            f.write("\n".join(names) + "\n")
        cfg["data"]["scannet_path"] = tmp
        loader = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "train", shuffle=False, augment_data=True,
                                          batch_size=args.batch, limit_numpoints=0, normalize_color=True,
                                          split_dir=os.path.join(tmp, "splits"))
        batch = next(iter(loader))
    mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
    net = load_model("Res16UNet34C")(3, 20, mcfg, D=3)
    det_init(net, 0)
    tr = semseg.SegmentationTrainer(net, cfg)
    for _ in range(args.warmup):
        tr.train_step(batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = tr.train_step(batch)
    e1.record()
    e1.synchronize()
    res = {"rank": rank, "world": world, "card": card(), "batch_per_rank": args.batch, "batch_voxels": int(len(batch[0][0])),
           "steps": args.steps, "step_ms": round(e0.elapsed_time(e1) / args.steps, 2), "loss": float(loss),
           "package": os.path.dirname(os.path.dirname(os.path.abspath(semseg.__file__)))}
    if world > 1:
        tr.grads.timing = {}
        tr.train_step(batch)
        end = torch.cuda.Event(enable_timing=True); end.record()
        torch.cuda.synchronize()
        tm = tr.grads.timing
        tr.grads.timing = None
        res.update(allreduce_ms=round(sum(a.elapsed_time(b) for a, b in tm["allreduce"]), 2), allreduces=len(tm["allreduce"]),
                   exposed_wait_plus_sgd_ms=round(tm["tail"][0].elapsed_time(end), 2))
        dist.destroy_process_group()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
