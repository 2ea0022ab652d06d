"""Forward + backward of VoteNet's criterion: the original `loss_helper.get_loss` (where oracle/det_eval_ref.py staged it) against
pointcontrast_b200.det_loss, at ScanNet (NH 1, NS 18, C 18) and SUN RGB-D (NH 12, NS 10, C 10) shapes with B 8, 1024 seeds, 256
proposals and 64 label slots (VoteNet's training batch):

    python profiles/bench_det_loss.py [--iters 200] [--repeats 5] [--warmup 20]

Times each implementation with CUDA events over `iters` calls after warm-up, the two alternating within each of `repeats` rounds
(median and spread over the rounds), counts kernel launches per call in a separate torch.profiler run, checks that the two agree, and
prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointcontrast_b200 import det_loss, synth  # noqa: E402

SHAPES = {"scannet": (1, 18, 18), "sunrgbd": (12, 10, 10)}
KEYS = ("seed_xyz", "seed_inds", "vote_xyz", "aggregated_vote_xyz", "center", "objectness_scores", "heading_scores",
        "heading_residuals_normalized", "size_scores", "size_residuals_normalized", "sem_cls_scores", "center_label", "heading_class_label",
        "heading_residual_label", "size_class_label", "size_residual_label", "sem_cls_label", "box_label_mask", "vote_label",
        "vote_label_mask")


class Config:
    def __init__(self, NH, NS, C, mean_size):
        self.num_heading_bin, self.num_size_cluster, self.num_class, self.mean_size_arr = NH, NS, C, mean_size


def inputs(dname):
    NH, NS, C = SHAPES[dname]
    ms = np.random.default_rng(1).uniform(0.3, 2.0, (NS, 3))
    ep = synth.synth_votenet_loss_batch(1, 8, 20000, 1024, 256, 1, NH, ms, C)
    t = {k: torch.from_numpy(np.ascontiguousarray(ep[k])).cuda() for k in KEYS}
    for k in det_loss.GRAD_INPUTS:
        t[k].requires_grad_(True)
    return t, Config(NH, NS, C, ms)


def step(fn, t, cfg):
    for k in det_loss.GRAD_INPUTS:
        t[k].grad = None
    loss, out = fn(dict(t), cfg)
    loss.backward()
    return out


def timed(fn, t, cfg, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step(fn, t, cfg)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def launches(fn, t, cfg):
    from torch.profiler import ProfilerActivity, profile
    step(fn, t, cfg)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        step(fn, t, cfg)
        torch.cuda.synchronize()
    return sum(1 for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Memcpy")
               and not e.name.startswith("Memset"))


def agree(a, b):
    return max(abs(float(a[k]) - float(b[k])) / max(abs(float(b[k])), 1e-2) for k in det_loss.OUTPUTS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_det_loss needs a GPU"
    from oracle import det_eval_ref
    impls = {"ours": det_loss.get_loss}
    if det_eval_ref.load() is not None:
        import importlib
        impls["original"] = importlib.import_module("models.loss_helper").get_loss
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = {"gpu": q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0), "iters": args.iters, "repeats": args.repeats}
    for dname in SHAPES:
        t, cfg = inputs(dname)
        for fn in impls.values():
            for _ in range(args.warmup):
                step(fn, t, cfg)
        ms = {k: [] for k in impls}
        for _ in range(args.repeats):
            for k, fn in impls.items():
                ms[k].append(timed(fn, t, cfg, args.iters))
        r = {}
        for k, fn in impls.items():
            r[k] = {"ms_median": float(np.median(ms[k])), "ms_min": float(np.min(ms[k])), "ms_max": float(np.max(ms[k])),
                    "launches": launches(fn, t, cfg)}
        if "original" in impls:
            r["max_rel_diff"] = agree(step(impls["ours"], t, cfg), step(impls["original"], t, cfg))
            r["speedup"] = r["original"]["ms_median"] / r["ours"]["ms_median"]
        res[dname] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
