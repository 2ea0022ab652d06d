"""S3DIS conversion on the GPU (pointcontrast_b200.semseg_prep.convert_stanford) against the host route on the same tree:

    python profiles/bench_semseg_prep.py [--rooms 4] [--points 1000000] [--host_rooms 1]

Input: `synth.write_s3dis_tree` rooms of `--points` points each (S3DIS rooms hold 0.2-9 M points, about 1 M on average) in 6 annotation
files, written under a temporary directory that is removed afterwards.

Reports, in one JSON line with the card's name and power limit read in the same run:
* `gpu_cold` / `gpu_warm`: convert_stanford over every room, with the annotation files dropped from the page cache before the run
  (`posix_fadvise(DONTNEED)` per file after an fsync; no system setting is touched) and then again with them cached; each gives the
  wall seconds, the seconds of file reads on the reader thread, of device work ending in a synchronise (copies back included) and
  of the writes on the writer thread;
* `host_s_per_room`: the host route on the first `--host_rooms` rooms, per room -- the original converter staged by `build()`
  (oracle/semseg_prep_ref.py, its ME call on the oracle's restatement) where it is staged, else oracle/semseg_prep_cpu.py -- warm cache;
* `equal`: the GPU route's files are byte-equal to the host route's for those rooms.
No speed-up is claimed beyond what these numbers show.
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import semseg_prep_cpu, semseg_prep_ref  # noqa: E402
from pointcontrast_b200 import semseg_prep, synth  # noqa: E402


def drop_cache(paths):
    for p in paths:
        fd = os.open(p, os.O_RDONLY)
        try:
            os.fsync(fd)
            os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
        finally:
            os.close(fd)


def gpu_run(src, out):
    t = time.perf_counter()
    secs = semseg_prep.convert_stanford(src, out, log=None)
    torch.cuda.synchronize()
    return dict(wall_s=round(time.perf_counter() - t, 4), **{f"{k}_s": round(v, 4) for k, v in secs.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rooms", type=int, default=4)
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--host_rooms", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "in")
        synth.write_s3dis_tree(src, 0, areas=(1,), rooms_per_area=args.rooms, points_per_room=args.points, empty_room=False)
        ann = glob.glob(os.path.join(src, "*", "*", "Annotations", "*.txt"))
        nbytes = sum(os.path.getsize(p) for p in ann)
        small = os.path.join(d, "warm")                                   # warm-up: module load, allocator, pinned pool
        synth.write_s3dis_tree(small, 1, areas=(1,), rooms_per_area=1, points_per_room=20000, empty_room=False)
        semseg_prep.convert_stanford(small, os.path.join(d, "warm_out"), log=None)
        drop_cache(ann)
        cold = gpu_run(src, os.path.join(d, "gpu_cold"))
        warm = gpu_run(src, os.path.join(d, "gpu_warm"))
        host_in = os.path.join(d, "host_in", "Area_1")
        os.makedirs(host_in)
        rooms = sorted(os.listdir(os.path.join(src, "Area_1")))[:args.host_rooms]
        for r in rooms:
            os.symlink(os.path.join(src, "Area_1", r), os.path.join(host_in, r))
        route = "original" if semseg_prep_ref.available() else "oracle"
        t = time.perf_counter()
        if route == "original":
            semseg_prep_ref.stanford(os.path.dirname(host_in), os.path.join(d, "host_out"), os.path.join(d, "host_cwd"))
        else:
            semseg_prep_cpu.convert_stanford(os.path.dirname(host_in), os.path.join(d, "host_out"))
        host_s = (time.perf_counter() - t) / len(rooms)
        equal = all(open(os.path.join(d, "host_out", "Area_1", r + ".ply"), "rb").read() ==
                    open(os.path.join(d, "gpu_warm", "Area_1", r + ".ply"), "rb").read() for r in rooms)
    print(json.dumps(dict(bench="semseg_prep", gpu=gpu, rooms=args.rooms, points_per_room=args.points, text_bytes=nbytes, gpu_cold=cold,
                          gpu_warm=warm, gpu_warm_s_per_room=round(warm["wall_s"] / args.rooms, 4), host_route=route,
                          host_rooms=len(rooms), host_s_per_room=round(host_s, 3), equal=equal)))


if __name__ == "__main__":
    main()
