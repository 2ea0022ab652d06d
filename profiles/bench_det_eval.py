"""Times VoteNet's detection evaluation on the library (`det_eval.parse_predictions` + `parse_groundtruths` + `APCalculator`) at the
ScanNet-val shape and prints one JSON line.

    python profiles/bench_det_eval.py [--scenes 312] [--batch 8] [--ref-scenes 16]

Workload: `--scenes` synthetic scenes (ScanNet val has 312) in batches of B = 8, K = 256 proposals, 18 classes, N = 40 000 points,
64 ground-truth slots; both config_dict variants (lib/test.py's: 2-D NMS with empty-box removal; lib/train.py's: 3-D per-class NMS,
per-class proposals), two APCalculators (IoU 0.25 and 0.5) as lib/test.py runs them.  Per variant:
  * batch_ms: parse_predictions + parse_groundtruths + both step() calls per batch, wall time with a device synchronise, after a warm-up
    pass over the same batches;
  * metrics_ms: both compute_metrics() calls;
  * ref: where oracle/det_eval_ref.py staged the original, its unmodified `ap_helper` (numpy, scipy, a pool of 10 processes) on the
    first `--ref-scenes` scenes, timed the same way (per batch and compute_metrics), and our dicts on that same subset: whether they
    have the same keys and the largest difference of their values (NaN equal to NaN).  The full val set would take the original
    minutes per variant, so a stated subset is used.
The card's name and power limit are read in the same run.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import det_eval_ref  # noqa: E402
from pointcontrast_b200 import det_eval  # noqa: E402

VARIANTS = {
    "test": dict(remove_empty_box=True, use_3d_nms=False, nms_iou=0.25, use_old_type_nms=False, cls_nms=False, per_class_proposal=False,
                 conf_thresh=0.05),
    "train": dict(remove_empty_box=False, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=False, cls_nms=True, per_class_proposal=True,
                  conf_thresh=0.05),
}


class ScanNetLike:
    num_class, num_heading_bin, num_size_cluster = 18, 1, 18

    def __init__(self):
        self.mean_size_arr = np.random.default_rng(0).uniform(0.3, 2.0, (18, 3))
        self.class2type = {c: f"class{c}" for c in range(18)}

    def class2angle(self, pred_cls, residual, to_label_format=True):
        return 0

    def class2size(self, pred_cls, residual):
        return self.mean_size_arr[pred_cls, :] + residual


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def batch(seed, B, K=256, C=18, N=40000, K2=64):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, device="cuda")
    n = lambda *s: torch.randn(*s, generator=g, device="cuda")
    gt_center = torch.cat([r(B, K2, 2) * 6 - 3, r(B, K2, 1) * 1.5 + 0.2], -1)
    src = torch.randint(0, K2, (B, K), generator=g, device="cuda")
    center = torch.gather(gt_center, 1, src.unsqueeze(-1).expand(B, K, 3)) + 0.15 * n(B, K, 3)
    sc_l = torch.randint(0, 18, (B, K2), generator=g, device="cuda")
    pts = torch.cat([r(B, N, 2) * 7 - 3.5, r(B, N, 1) * 2, r(B, N, 1)], -1)
    return {
        "center": center, "heading_scores": n(B, K, 1), "heading_residuals": 0.1 * n(B, K, 1), "size_scores": n(B, K, 18),
        "size_residuals": 0.1 * n(B, K, 18, 3), "sem_cls_scores": 2 * n(B, K, C), "objectness_scores": 2 * n(B, K, 2),
        "point_clouds": pts, "center_label": gt_center, "heading_class_label": torch.zeros(B, K2, dtype=torch.int64, device="cuda"),
        "heading_residual_label": torch.zeros(B, K2, device="cuda"), "size_class_label": sc_l,
        "size_residual_label": 0.05 * n(B, K2, 3), "sem_cls_label": sc_l, "box_label_mask": (r(B, K2) < 0.4).float(),
    }


def run(batches, cd, cfg, helper=det_eval):
    calcs = [helper.APCalculator(t, cfg.class2type) for t in (0.25, 0.5)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for ep in batches:
        ep = dict(ep)
        p = helper.parse_predictions(ep, cd)
        gt = helper.parse_groundtruths(ep, cd)
        for c in calcs:
            c.step(p, gt)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    res = [c.compute_metrics() for c in calcs]
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3 / len(batches), (t2 - t1) * 1e3, res


def compare(ours, ref):
    """(same keys, largest |difference| over the values of both thresholds' dicts, NaN equal to NaN)"""
    same = all(list(a) == list(b) for a, b in zip(ours, ref))
    diff = 0.0
    for a, b in zip(ours, ref):
        for k in a:
            x, y = float(a[k]), float(b.get(k, np.nan))
            if not (np.isnan(x) and np.isnan(y)):
                diff = max(diff, abs(x - y)) if not (np.isnan(x) or np.isnan(y)) else np.inf
    return same, diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=312)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--ref-scenes", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det_eval needs a GPU")
    cfg = ScanNetLike()
    nb = (a.scenes + a.batch - 1) // a.batch
    batches = [batch(s, min(a.batch, a.scenes - s * a.batch)) for s in range(nb)]
    ref_helper = det_eval_ref.load()
    ref_batches = batches[:max(1, a.ref_scenes // a.batch)]
    out = {"card": card(), "scenes": a.scenes, "batch": a.batch, "K": 256, "classes": 18, "points": 40000,
           "ref_scenes": sum(b["center"].shape[0] for b in ref_batches) if ref_helper else 0}
    for name, v in VARIANTS.items():
        cd = dict(v, dataset_config=cfg)
        run(batches, cd, cfg)                                                   # warm-up: module load, allocator, every shape
        batch_ms, metrics_ms, res = run(batches, cd, cfg)
        _, _, res2 = run(batches, cd, cfg)
        same = all(json.dumps({k: float(x) for k, x in r1.items()}) == json.dumps({k: float(x) for k, x in r2.items()})
                   for r1, r2 in zip(res, res2))
        out[name] = {"batch_ms": round(batch_ms, 3), "metrics_ms": round(metrics_ms, 3), "mAP@0.25": float(res[0]["mAP"]),
                     "mAP@0.5": float(res[1]["mAP"]), "repeat_identical": same, "ref": "not measured (not staged)"}
        if ref_helper is not None:
            with contextlib.redirect_stdout(io.StringIO()):                     # the original prints per class
                r_batch_ms, r_metrics_ms, r_res = run(ref_batches, cd, cfg, ref_helper)
            o_batch_ms, o_metrics_ms, o_res = run(ref_batches, cd, cfg)
            keys_same, max_diff = compare(o_res, r_res)
            out[name]["ref"] = {"batch_ms": round(r_batch_ms, 1), "metrics_ms": round(r_metrics_ms, 1),
                                "ours_batch_ms": round(o_batch_ms, 3), "ours_metrics_ms": round(o_metrics_ms, 3),
                                "same_keys": keys_same, "max_abs_diff": max_diff}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
