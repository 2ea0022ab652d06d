"""Times the semantic-segmentation evaluation (`semseg.SegmentationMetrics`, `semseg.test`) against the reference's per-batch metric code
(`downstream/semseg/lib/test.py:131-149`).  Prints one JSON line.

    python profiles/bench_semseg_eval.py [--scenes 8] [--n-raw 150000]

* metrics: per batch of logits at ScanNet-val shape (120 k voxels x 20 classes) and S3DIS shape (80 k x 13), about 10 % ignored rows:
  - gpu_ms: `SegmentationMetrics.update` (pcb_seg_metrics + pcb_average_precision), CUDA events over a window of >= 1 s after warm-up
    (nothing in it synchronises);
  - ref_ms: the reference's code on the same logits: torch cross-entropy, `max(1)`, precision@1 and softmax on the GPU, then `.cpu()`,
    numpy `fast_hist` and scikit-learn `label_binarize` + `average_precision_score`, wall time over >= 1 s (it synchronises);
  - the two agree: identical histogram, loss and precision@1 within 1e-6 relative, mAP within 1e-3 (percentage units).
* test: `semseg.test` (Res16UNet34C, 20 classes, batch 1, `det_init` weights) over synthetic ScanNet-like rooms read from PLY, per scene
  (loading and voxelisation included), and the share of it the metric updates take (their CUDA-event time on the same logits).
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pointcontrast_b200 import me as ME, semseg, semseg_data as S, synth  # noqa: E402
from pointcontrast_b200.model import load_model  # noqa: E402
from tests import refload  # noqa: E402
from tests.helpers import det_init  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"name": torch.cuda.get_device_name(), "nvidia_smi": q}


def timed_events(fn, min_s=1.0, warmup=3):
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


def timed_wall(fn, min_s=1.0, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < min_s:
        fn()
        n += 1
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n, n


def reference_batch(output, target, C):
    """`test.py:131-149` (and `utils.py:117-133`) with the model output on the GPU."""
    from sklearn.metrics import average_precision_score
    from sklearn.preprocessing import label_binarize
    target_np = target.cpu().numpy()
    pred = output.max(1)[1].int()
    cross_ent = torch.nn.functional.cross_entropy(output, target.long(), ignore_index=255)
    loss = float(cross_ent)
    p, t = pred.view(1, -1), target.view(1, -1)
    correct = p.eq(t)[t != 255].view(-1)
    score = correct.float().sum(0).mul(100.0 / correct.size(0)).item()
    pn = pred.cpu().numpy().flatten()
    k = (target_np >= 0) & (target_np < C)
    hist = np.bincount(C * target_np[k].astype(int) + pn[k], minlength=C ** 2).reshape(C, C)
    prob = torch.nn.functional.softmax(output, dim=1).cpu().numpy()
    label = label_binarize(target_np, classes=list(range(C)))
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ap = average_precision_score(label, prob, average=None)
    return loss, score, hist, ap


def metric_shapes(res):
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, n, C in (("scannet_val", 120_000, 20), ("s3dis", 80_000, 13)):
        t = torch.randint(0, C, (n,), device="cuda", generator=g)
        x = torch.randn(n, C, device="cuda", generator=g) * 2
        x[torch.arange(n, device="cuda"), t] += 2.0
        t[torch.rand(n, device="cuda", generator=g) < 0.1] = 255
        m = semseg.SegmentationMetrics(C, 255, "cuda")
        gpu_ms, gpu_reps = timed_events(lambda: m.update(x, t))
        ref_ms, ref_reps = timed_wall(lambda: reference_batch(x, t, C))
        m.reset()
        m.update(x, t)
        r = m.result()
        loss, score, hist, ap = reference_batch(x, t, C)
        present = np.bincount(t[t != 255].cpu().numpy(), minlength=C) > 0
        ref_map = float(np.mean(ap[present]) * 100)
        ok = (np.array_equal(r.hist, hist) and abs(r.loss - loss) <= 1e-6 * abs(loss) and abs(r.score - score) <= 1e-6 * abs(score)
              and abs(r.mAP - ref_map) <= 1e-3)
        assert ok, (name, r.loss, loss, r.score, score, r.mAP, ref_map)
        res[name] = {"n": n, "C": C, "gpu_ms": round(gpu_ms, 4), "gpu_reps": gpu_reps, "ref_ms": round(ref_ms, 2), "ref_reps": ref_reps,
                     "speedup": round(ref_ms / gpu_ms, 1), "mAP_gap": float(abs(r.mAP - ref_map))}


def test_pass(res, scenes, n_raw):
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "splits"))
        names = []
        for k in range(scenes):
            xyz, rgb, lab = synth.synth_labelled_room(500 + k, n_raw, scale=1.6)
            names.append(f"scene{k:04d}_00.ply")
            synth.write_ply(os.path.join(tmp, names[-1]), xyz, rgb, lab)
        with open(os.path.join(tmp, "splits", "scannetv2_val.txt"), "w") as f:
            f.write("\n".join(names) + "\n")
        cfg = refload.Cfg(data=dict(scannet_path=tmp, ignore_label=255, return_transformation=False),
                          augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
                          test=dict(test_stat_freq=10 ** 9))
        loader = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "val", shuffle=False, augment_data=False, batch_size=1,
                                          limit_numpoints=0, split_dir=os.path.join(tmp, "splits"), repeat=False)
        mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
        net = load_model("Res16UNet34C")(3, 20, mcfg, D=3).cuda()
        det_init(net, 0)
        semseg.test(net, loader, cfg)                                    # warm-up: allocator, kernel maps
        reps, t0 = 0, time.perf_counter()
        while time.perf_counter() - t0 < 1.0 or reps < 2:
            semseg.test(net, loader, cfg)
            reps += 1
        torch.cuda.synchronize()
        test_ms = (time.perf_counter() - t0) * 1e3 / (reps * scenes)
        # the metric updates alone on the same logits
        net.eval()
        batches = []
        with torch.no_grad():
            for coords, feats, target in loader:
                batches.append((net(ME.SparseTensor(feats, coords).to("cuda")).F.clone(), target.cuda()))
        m = semseg.SegmentationMetrics(20, 255, "cuda")
        metric_ms, _ = timed_events(lambda: [m.update(x, t) for x, t in batches])
        metric_ms /= scenes
        res["test"] = {"scenes": scenes, "n_raw": n_raw, "voxels_per_scene": int(np.mean([len(x) for x, _ in batches])), "reps": reps,
                       "ms_per_scene": round(test_ms, 2), "metric_ms_per_scene": round(metric_ms, 4),
                       "metric_share": round(metric_ms / test_ms, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=8)
    ap.add_argument("--n-raw", type=int, default=150_000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    res = {"card": card()}
    metric_shapes(res)
    test_pass(res, args.scenes, args.n_raw)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
