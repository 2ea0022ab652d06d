"""VoteNet detection preprocessing on the GPU (pointcontrast_b200.det_prep) against the host route on the same synthetic scenes:

    python profiles/bench_det_prep.py [--scannet 6] [--sunrgbd 16] [--host_scenes 2]

Input, written under a temporary directory that is removed afterwards: `--scannet` ScanNet scenes of 150 000 vertices, 3 000 segments and
40 instances (`synth.write_scannet_det_raw_scene`; released scenes hold 50 k - 500 k vertices), and `--sunrgbd` SUN RGB-D scenes of
300 000 points and 10 boxes (`synth.write_sunrgbd_export`, about the size of a released depth export).

Reports, in one JSON line with the card's name and power limit read in the same run, seconds per scene for each route: the GPU route's
wall time and its read / device / write parts (reads and writes summed over their threads, so they may exceed the wall time), after one
warm-up scene, warm page cache; and the host route on the first `--host_scenes` scenes -- the original scripts staged by `build()`
(oracle/det_prep_ref.py) where they are staged, else oracle/det_prep_cpu.py.  `equal` says the GPU route's arrays equal the host
route's for those scenes under the same seed.  No speed-up is claimed beyond what these numbers show.
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
from oracle import det_prep_cpu, det_prep_ref  # noqa: E402
from pointcontrast_b200 import det_prep, synth  # noqa: E402
from tests.golden.make_det_prep_golden import digests  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scannet", type=int, default=6)
    ap.add_argument("--sunrgbd", type=int, default=16)
    ap.add_argument("--host_scenes", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    staged = det_prep_ref.available()
    out = dict(host_route="original" if staged else "numpy restatement")
    with tempfile.TemporaryDirectory() as d:
        lm = synth.write_scannet_label_map(os.path.join(d, "labels.tsv"))
        names = ["scene%04d_00" % k for k in range(args.scannet + 1)]
        for k, n in enumerate(names):
            synth.write_scannet_det_raw_scene(os.path.join(d, "scans"), n, k, n=150000, n_seg=3000, n_obj=40)
        sun = os.path.join(d, "sun")
        synth.write_sunrgbd_export(sun, 1, n_scenes=args.sunrgbd + 2, n_points=300000, big_points=300000, n_boxes=10)
        with open(os.path.join(sun, "train_data_idx.txt"), "w") as f:       # the warm-up scene alone in val
            f.write("".join("%d\n" % i for i in range(2, args.sunrgbd + 2)))
        with open(os.path.join(sun, "val_data_idx.txt"), "w") as f:
            f.write("1\n")

        det_prep.convert_scannet(os.path.join(d, "scans"), os.path.join(d, "warm"), lm, scan_list=_list(d, names[:1]), log=None)
        np.random.seed(0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        secs = det_prep.convert_scannet(os.path.join(d, "scans"), os.path.join(d, "gpu_sc"), lm, scan_list=_list(d, names[1:]), log=None)
        wall = time.perf_counter() - t
        out["scannet_gpu_s_per_scene"] = dict(wall=wall / args.scannet, **{k: secs[k] / args.scannet for k in ("read", "device", "write")})
        det_prep.convert_sunrgbd(sun, os.path.join(d, "warm_sun"), splits=("val",), log=None)
        np.random.seed(0)
        t = time.perf_counter()
        secs = det_prep.convert_sunrgbd(sun, os.path.join(d, "gpu_sun"), splits=("train",), log=None)
        wall = time.perf_counter() - t
        out["sunrgbd_gpu_s_per_scene"] = dict(wall=wall / args.sunrgbd, **{k: v / args.sunrgbd for k, v in secs.items()})

        h = args.host_scenes
        np.random.seed(0)
        t = time.perf_counter()
        if staged:
            det_prep_ref.scannet(os.path.join(d, "scans"), lm, names[1:1 + h], os.path.join(d, "host_sc"))
        else:
            det_prep_cpu.convert_scannet(os.path.join(d, "scans"), os.path.join(d, "host_sc"), lm, names[1:1 + h])
        out["scannet_host_s_per_scene"] = (time.perf_counter() - t) / h
        with open(os.path.join(sun, "train_data_idx.txt"), "w") as f:
            f.write("".join("%d\n" % i for i in range(2, 2 + h)))
        np.random.seed(0)
        t = time.perf_counter()
        if staged:
            det_prep_ref.sunrgbd(sun, os.path.join(d, "host_sun"), splits=("train",))
        else:
            det_prep_cpu.convert_sunrgbd(sun, os.path.join(d, "host_sun"), splits=("train",))
        out["sunrgbd_host_s_per_scene"] = (time.perf_counter() - t) / h
        g_sc, h_sc = digests(os.path.join(d, "gpu_sc")), digests(os.path.join(d, "host_sc"))
        g_sun, h_sun = digests(os.path.join(d, "gpu_sun")), digests(os.path.join(d, "host_sun"))
        out["equal"] = dict(scannet=all(g_sc.get(k) == v for k, v in h_sc.items()) and len(h_sc) == 4 * h,
                            sunrgbd=all(g_sun.get(k) == v for k, v in h_sun.items()) and len(h_sun) == 3 * h)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                text=True).stdout.strip()
    print(json.dumps(out))


def _list(d, names):
    p = os.path.join(d, "list_%d.txt" % len(os.listdir(d)))
    with open(p, "w") as f:
        f.write("".join(n + "\n" for n in names))
    return p


if __name__ == "__main__":
    main()
