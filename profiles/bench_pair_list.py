"""Pair-list construction on the GPU (pointcontrast_b200.pair_list) against the CPU oracle and the reference's per-point loop, on
synthetic scans (`synth.synth_scan_frames`, about 250k fp64 points per frame) of F = 50 / 100 / 200 frames:

    python profiles/bench_pair_list.py [--frames 50 100 200] [--points 250000]

Per scene: `voxel_down_sample` and `overlap_counts` times (CUDA events, warmed, windows of at least one second), the end-to-end wall
time of `compute_full_overlapping` (npz reads, both kernels, the overlap.txt write), the oracle (oracle/pair_list_cpu.py: cKDTree,
vectorised per frame) once, and the reference's loop of one KD-tree query per point (`compute_full_overlapping.py:39-47`, `:67-74`,
restated with one cKDTree query per point) timed on a sample of frame pairs and EXTRAPOLATED to all F (F - 1) ordered pairs.  The GPU
results are checked against the oracle's (points, offsets and counts bit-exact, overlap.txt byte-identical).  The scenes share their
first frames (hard links).  The card's name and power limit are read in the same run.  Prints one JSON line.
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
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pair_list_cpu as O  # noqa: E402
from pointcontrast_b200 import pair_list, synth  # noqa: E402

VOXEL = 0.05


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


def reference_loop_s_per_pair(down, rng, n_pairs):
    """The reference's per-point loop (one KD-tree radius query per point of frame j against frame i's tree), seconds per ordered
    pair, on n_pairs random pairs."""
    F = len(down)
    ts = []
    for _ in range(n_pairs):
        i, j = rng.choice(F, 2, replace=False)
        tree = cKDTree(down[i])
        t = time.perf_counter()
        m = 0
        for p in down[j]:
            m += len(tree.query_ball_point(p, 1.5 * VOXEL)[:1])
        ts.append(time.perf_counter() - t)
    return float(np.mean(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[50, 100, 200])
    ap.add_argument("--points", type=int, default=250_000)
    ap.add_argument("--ref-pairs", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pair_list needs a GPU"
    torch.cuda.set_device(0)
    Fmax = max(args.frames)
    t0 = time.perf_counter()
    log(f"synthesising {Fmax} frames")
    frames = synth.synth_scan_frames(0, Fmax, points_per_frame=args.points)
    gen_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    down_oracle = []
    for k, f in enumerate(frames):
        down_oracle.append(O.voxel_down_sample(f, VOXEL))
        if k % 20 == 19:
            log(f"oracle downsampled {k + 1} / {Fmax} frames")
    oracle_down_s = [time.perf_counter() - t0]
    out = {"metric": "pair_list", "card": card(), "voxel_size": VOXEL, "points_per_frame": args.points, "synth_s": round(gen_s, 1),
           "scenes": []}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        master = os.path.join(tmp, "all")
        os.makedirs(master)
        for k, f in enumerate(frames):
            np.savez(os.path.join(master, f"{k * 25:06d}.npz"), pcd=f)
        for F in args.frames:
            d = os.path.join(tmp, f"scene{F:04d}", "pcd")
            os.makedirs(d)
            for k in range(F):
                src = os.path.join(master, f"{k * 25:06d}.npz")
                try:
                    os.link(src, os.path.join(d, f"{k * 25:06d}.npz"))
                except OSError:
                    import shutil
                    shutil.copyfile(src, os.path.join(d, f"{k * 25:06d}.npz"))
            log(f"scene of {F} frames")
            sizes = np.array([len(f) for f in frames[:F]])
            off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)])).cuda()
            xyz = torch.from_numpy(np.concatenate(frames[:F])).cuda()
            res = {}
            res["down_ms"], _ = timed(lambda: res.__setitem__("down", pair_list.voxel_down_sample(xyz, off, VOXEL)))
            pts, doff, host = res["down"]
            res["overlap_ms"], _ = timed(lambda: res.__setitem__("counts", pair_list.overlap_counts(pts, doff, 1.5 * VOXEL)))
            # end to end: npz reads + both kernels + overlap.txt
            torch.cuda.synchronize()
            t = time.perf_counter()
            M, names = pair_list.compute_full_overlapping(d, VOXEL)
            e2e_s = time.perf_counter() - t
            gpu_txt = open(os.path.join(d, "overlap.txt"), "rb").read()
            # oracle, once
            t = time.perf_counter()
            counts_o = O.frame_overlap_counts(down_oracle[:F], 1.5 * VOXEL)
            oracle_counts_s = time.perf_counter() - t
            want_pts = np.concatenate(down_oracle[:F])
            want_off = np.concatenate([[0], np.cumsum([len(x) for x in down_oracle[:F]])])
            O.write_overlap(os.path.join(d, "overlap.txt"), names, counts_o, [len(x) for x in down_oracle[:F]])
            equal = (host == want_off.tolist() and np.array_equal(pts.cpu().numpy().view(np.uint64), want_pts.view(np.uint64))
                     and np.array_equal(res["counts"].cpu().numpy(), counts_o) and open(os.path.join(d, "overlap.txt"), "rb").read() == gpu_txt)
            log(f"  gpu {res['down_ms']:.1f} + {res['overlap_ms']:.1f} ms, end to end {e2e_s:.1f} s, oracle equal: {equal}")
            per_pair = reference_loop_s_per_pair(down_oracle[:F], rng, args.ref_pairs)
            M_sym = np.maximum(M, M.T)[np.triu_indices(F, 1)]
            out["scenes"].append({
                "frames": F, "raw_points": int(sizes.sum()), "down_points": int(host[F]),
                "voxel_down_sample_ms": round(res["down_ms"], 3), "frame_overlap_ms": round(res["overlap_ms"], 3),
                "end_to_end_s": round(e2e_s, 3),
                "oracle_s": round(oracle_down_s[0] * F / Fmax + oracle_counts_s, 2),
                "reference_loop_s_extrapolated": round(per_pair * F * (F - 1), 1),
                "reference_loop_s_per_pair_sampled": round(per_pair, 3), "reference_pairs_sampled": args.ref_pairs,
                "pairs": F * (F - 1) // 2, "pairs_ge_0.3": int((M_sym >= 0.3).sum()), "gpu_equals_oracle": bool(equal)})
    out["all_equal"] = all(s["gpu_equals_oracle"] for s in out["scenes"])
    print(json.dumps(out))
    return 0 if out["all_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
