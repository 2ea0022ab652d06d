"""`.sens` extraction on the GPU (pointcontrast_b200.pair_list.extract_scene) against the reference's route on the same file:

    python profiles/bench_sens.py [--frames 1500] [--frame_skip 25]

Input: one ScanNet-sized synthetic scan (`synth.synth_sens_scan`: 640 x 480 depth, `--frames` frames, colour payloads of JPEG size)
written by `synth.write_sens` under a temporary directory that is removed afterwards.  The walk turns 1/25 of `synth_scan_frames`'
step per frame, and only the frames the frame skip keeps are rendered (the others repeat them), so the scan is quick to make.

Reports, in one JSON line with the card's name and power limit read in the same run:
* `kernel_ms_per_frame`: `depth_to_points` on a device batch of EXTRACT_CHUNK kept frames (its one synchronising copy of the offsets
  included), CUDA-event mean over windows of at least 1 s after warm-up, divided by the batch;
* `extract_s`: the wall time of one scene, `read_sens` (file reads and zlib inflate) then `extract_scene` ending in a device
  synchronise, and its parts: `gpu` (the device loop with the copies back and the downsampling), `write` (npz writes on the writer
  thread, overlapping the loop), `overlap` (the overlap kernel and overlap.txt);
* `original_s`, run once where `build()` staged the reference's scripts (oracle/sens_ref.py): the staged `reader.py` +
  `point_cloud_extractor.py` with the array codec in place of PNG (which is faster than PNG, so this favours the original), then
  `pair_list overlap` (`compute_full_overlapping`) on the npz files it wrote;
* `npz_equal_oracle`: the extracted npz files are bit-equal to oracle/sens_cpu.py; `same_pairs` / `max_overlap_difference`: the
  overlap.txt files of both routes list the same pairs, and how far their values differ (the original's points differ from ours
  within the bound of its BLAS product, so a downsampled point may move by an ulp).
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sens_cpu, sens_ref  # noqa: E402
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


def pairs(path):
    return {frozenset(os.path.basename(n) for n in line.split()[:2]): line.split()[2] for line in open(path)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1500)
    ap.add_argument("--frame_skip", type=int, default=25)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sens needs a GPU"
    torch.cuda.set_device(0)
    out = {"metric": "sens_extract", "card": card(), "frames": args.frames, "frame_skip": args.frame_skip, "size": "640x480",
           "voxel_size": VOXEL}
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        depth, poses, K = synth.synth_sens_scan(0, args.frames, frames_per_view=25, render_every=args.frame_skip, bad_poses=(args.frame_skip * 3,))
        sens = os.path.join(tmp, "scene0000_00.sens")
        synth.write_sens(sens, depth, poses, K)
        del depth
        out["synth_s"] = round(time.perf_counter() - t, 1)
        out["sens_bytes"] = os.path.getsize(sens)
        log(f"scan written: {out['sens_bytes'] / 1e6:.0f} MB in {out['synth_s']} s")

        # kernel time per frame
        scan = pair_list.read_sens(sens, args.frame_skip)
        F = min(pair_list.EXTRACT_CHUNK, len(scan.frames))
        dev_depth = torch.from_numpy(scan.depth[:F].view(np.int16)).cuda()
        dev_poses = torch.from_numpy(scan.poses[:F]).cuda()
        ms, reps = timed(lambda: pair_list.depth_to_points(dev_depth, scan.intrinsic, dev_poses))
        out["kernel_ms_per_frame"] = round(ms / F, 4)
        out["kernel_batch"] = F
        out["points_per_frame"] = int(np.count_nonzero(scan.depth) / len(scan.frames))
        del dev_depth, dev_poses

        # one scene end to end (the warm-up above loaded the kernels)
        ours = os.path.join(tmp, "ours", "scene0000_00")
        torch.cuda.synchronize()
        t = time.perf_counter()
        scan = pair_list.read_sens(sens, args.frame_skip)
        read_s = time.perf_counter() - t
        M, names, secs = pair_list.extract_scene(sens, ours, args.frame_skip, VOXEL, scan=scan)
        torch.cuda.synchronize()
        total = time.perf_counter() - t
        out["extract_s"] = {"total": round(total, 3), "read_inflate": round(read_s, 3), **{k: round(v, 3) for k, v in secs.items()}}
        out["kept_frames"], out["overlap_frames"] = len(scan.frames), len(names)
        log(f"extract_scene: {out['extract_s']}")
        equal = True
        for k, f in enumerate(scan.frames):
            got = np.load(os.path.join(ours, "pcd", f"{f}.npz"))["pcd"]
            want = sens_cpu.depth_to_points(scan.depth[k], scan.intrinsic, scan.poses[k])
            equal &= got.shape == want.shape and np.array_equal(got.view(np.uint64), want.view(np.uint64))
        out["npz_equal_oracle"] = bool(equal)

        # the original route, once
        if sens_ref.available():
            ref = os.path.join(tmp, "ref", "scene0000_00")
            t = time.perf_counter()
            with contextlib.redirect_stdout(sys.stderr):           # the scripts print as they go
                sens_ref.extract(sens, ref, args.frame_skip)
            ext_s = time.perf_counter() - t
            t = time.perf_counter()
            pair_list.compute_full_overlapping(os.path.join(ref, "pcd"), VOXEL)
            ov_s = time.perf_counter() - t
            out["original_s"] = {"total": round(ext_s + ov_s, 2), "reader_and_extractor": round(ext_s, 2), "pair_list_overlap": round(ov_s, 2)}
            a, b = pairs(os.path.join(ref, "pcd", "overlap.txt")), pairs(os.path.join(ours, "pcd", "overlap.txt"))
            out["same_pairs"] = set(a) == set(b)
            out["max_overlap_difference"] = max((abs(float(a[k]) - float(b[k])) for k in set(a) & set(b)), default=0.0)
            log(f"original: {out['original_s']}")
        else:
            out["original_s"] = "not measured (the reference's scripts are not staged)"
    print(json.dumps(out))
    return 0 if out["npz_equal_oracle"] else 1


if __name__ == "__main__":
    sys.exit(main())
