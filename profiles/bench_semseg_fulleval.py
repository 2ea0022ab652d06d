"""Label transfer to the original point cloud on the GPU (`pcb_nearest` + `pcb_label_transfer`) against the reference's host path
(scipy KD-tree query, the label-map loops and `fast_hist`), at ScanNet size and at the size of a merged S3DIS group:

    python profiles/bench_semseg_fulleval.py [--scannet 150000 120000] [--s3dis 3000000 500000]

Per size (queries n, centres m): the two kernels' time (CUDA events, warmed, windows of at least one second), the reference's path once
on the host (`scipy.spatial.KDTree(leafsize=500).query` as `scannet.py:154-155`, `[label_map[x] for x in ...]` for both label arrays,
`fast_hist`), and whether the GPU's indices equal the oracle's.  Then the time `test.test_original_pointcloud` adds per scene to
`semseg.test`: `PointCloudEvaluator.add` of one ScanNet-size scene with its PLY read and its submission file written (wall clock,
synchronised).  The card's name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import semseg_fulleval_cpu as O  # noqa: E402
from pointcontrast_b200 import semseg, semseg_data as D, synth  # noqa: E402


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def timed(fn, min_s=1.0):
    """Mean ms of fn() over a window of at least min_s seconds (CUDA events), after two warm-up calls."""
    fn(); fn()
    torch.cuda.synchronize()
    reps, total = 0, 0.0
    while total < min_s * 1e3 or reps < 3:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        total += a.elapsed_time(b)
        reps += 1
    return total / reps, reps


def scene(seed, n, m, voxel, scale):
    """n original points of a synthetic room and m voxel centres of it (fp64), with labels."""
    xyz, _, lab = synth.synth_labelled_room(seed, max(n, 4 * m), scale=scale)
    xyz = xyz.astype(np.float64)
    cells = np.unique(np.floor(xyz / voxel), axis=0)
    g = np.random.default_rng(seed)
    ref = (cells[g.permutation(len(cells))[:m]] + 0.5) * voxel
    q = g.permutation(len(xyz))[:n]
    return ref, xyz[q], lab[q].astype(np.int64)


def scannet_maps():
    label_map, used = {}, 0
    for l in range(41):
        if l in D.ScannetVoxelizationDataset.IGNORE_LABELS:
            label_map[l] = 255
        else:
            label_map[l] = used
            used += 1
    label_map[255] = 255
    return label_map, used


def bench_size(name, n, m, voxel, scale, label_map, C, seed):
    ref, query, gt = scene(seed, n, m, voxel, scale)
    g = np.random.default_rng(seed + 1)
    ref_label = O.decode_lut(label_map, C)[g.integers(0, C, len(ref))]
    lut = O.label_lut(label_map)
    r, q = torch.from_numpy(ref).cuda(), torch.from_numpy(query).cuda()
    rl, ql, lt = (torch.from_numpy(a.astype(np.int32)).cuda() for a in (ref_label, gt, lut))
    hist = torch.zeros(C * C, dtype=torch.int64, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")

    def run():
        idx = semseg.nearest(r, q, voxel)           # reads its status: one synchronisation, as in the evaluator
        pl, s = semseg.label_transfer(idx, rl, ql, lt, C, hist)
        st.copy_(s)
        return idx
    ms, reps = timed(run)
    idx = run().cpu().numpy()
    # the reference's host path, once
    from scipy import spatial
    t = time.perf_counter()
    tree = spatial.KDTree(ref, leafsize=500)
    _, result = tree.query(query)
    ptc_pred = ref_label[result].astype(int)
    p = np.array([label_map[x] for x in ptc_pred], dtype=np.int64)
    y = np.array([label_map[x] for x in gt], dtype=np.int64)
    h_ref = O.fast_hist(p, y, C)
    host_s = time.perf_counter() - t
    want = O.nearest(ref, query)
    equal = bool(np.array_equal(idx, want))
    hist.zero_()
    run()
    hist_equal = bool(np.array_equal(hist.cpu().numpy().reshape(C, C), O.label_transfer(want, ref_label, gt, lut, C)[1]))
    log(f"{name}: n {len(query)} m {len(ref)}: gpu {ms:.2f} ms, host {host_s:.2f} s, equal {equal}, hist {hist_equal}")
    return {"queries": len(query), "centres": len(ref), "voxel": voxel, "gpu_ms": round(ms, 3), "gpu_reps": reps,
            "reference_host_s": round(host_s, 3), "kdtree_equals_exact_hist": bool(np.array_equal(h_ref, O.label_transfer(want, ref_label, gt, lut, C)[1])),
            "gpu_idx_equals_oracle": equal, "gpu_hist_equals_oracle": hist_equal}


class _Cfg(dict):
    def __getattr__(self, k):
        v = self[k]
        return _Cfg(v) if isinstance(v, dict) else v


def per_scene_overhead(n, reps=5):
    """Wall time of PointCloudEvaluator.add for one ScanNet-size scene: PLY read, both kernels, the histogram, the .txt write."""
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "splits"))
        xyz, rgb, lab = synth.synth_labelled_room(9, n, scale=1.0)
        synth.write_ply(os.path.join(tmp, "scene0000_00.ply"), xyz, rgb, lab)
        with open(os.path.join(tmp, "splits", "scannetv2_val.txt"), "w") as f:
            f.write("scene0000_00.ply\n")
        cfg = _Cfg(data=dict(scannet_path=tmp, ignore_label=255, return_transformation=True))
        ds = D.ScannetVoxelization2cmDataset(cfg, augment_data=False, phase="val", split_dir=os.path.join(tmp, "splits"))
        coords, _, _, T = ds[0]
        coords = torch.cat([torch.zeros(len(coords), 1, dtype=torch.int32, device=coords.device), coords], 1)
        Trow = torch.from_numpy(np.concatenate([T.reshape(16), [0]]).astype(np.float32))[None]
        pred = torch.randint(0, ds.NUM_LABELS, (len(coords),), dtype=torch.int32, device=coords.device)
        pieces = semseg.prediction_pieces(coords, pred, Trow, ds)
        ts = []
        for k in range(reps + 1):
            ev = semseg.PointCloudEvaluator(ds, "cuda", eval_path=os.path.join(tmp, f"fulleval{k}"))
            torch.cuda.synchronize()
            t = time.perf_counter()
            ev.add(0, *pieces[0])
            ev.result()
            ts.append(time.perf_counter() - t)
        return {"points": n, "centres": len(coords), "ms_per_scene": round(1e3 * float(np.median(ts[1:])), 2), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scannet", type=int, nargs=2, default=[150_000, 120_000])
    ap.add_argument("--s3dis", type=int, nargs=2, default=[3_000_000, 500_000])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_semseg_fulleval needs a GPU"
    torch.cuda.set_device(0)
    label_map, C = scannet_maps()
    out = {"metric": "semseg_fulleval", "card": card()}
    out["scannet"] = bench_size("scannet", *args.scannet, 0.02, 1.0, label_map, C, 1)
    out["s3dis_group"] = bench_size("s3dis_group", *args.s3dis, 0.05, 6.0, label_map, C, 2)
    out["per_scene"] = per_scene_overhead(args.scannet[0])
    out["all_equal"] = all(out[k]["gpu_idx_equals_oracle"] and out[k]["gpu_hist_equals_oracle"] for k in ("scannet", "s3dis_group"))
    print(json.dumps(out))
    return 0 if out["all_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
