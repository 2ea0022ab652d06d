"""Writes tests/golden/det_data.npz: the original VoteNet detection `__getitem__`s (staged by oracle/stage_ref.py, loaded by
oracle/det_data_ref.py), run unmodified on small synthetic scenes (pointcontrast_b200.synth) from a seeded RandomState, their draws
recorded.

    python tests/golden/make_det_data_golden.py

Cases: ScanNet (N above and below num_points, K = 0 / 5 / 64, the instance-id quirks of synth.write_scannet_detection_scene) x augment x
use_height; SUN RGB-D x augment x use_height x use_color.  Per case: `<case>/<output key>` (the original's item), `<case>/draw_kinds`
(random / choice, in call order) and `<case>/draw<i>`; per scene `<scene>/<file array>`.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import det_data_ref  # noqa: E402
from pointcontrast_b200 import synth  # noqa: E402

NUM_POINTS = 200
SCANNET = (("scene0000_00", 300, 5), ("scene0001_00", 150, 0), ("scene0002_00", 250, 64))
SUNRGBD = (("000001", 300, 6), ("000002", 150, 0), ("000003", 250, 64))


def scannet_cases():
    for s in range(len(SCANNET)):
        for augment in (False, True):
            for use_height in (False, True):
                yield f"scannet_{s}_a{int(augment)}_h{int(use_height)}", s, dict(augment=augment, use_height=use_height, use_color=False)


def sunrgbd_cases():
    for s in range(len(SUNRGBD)):
        for augment in (False, True):
            for use_height in (False, True):
                for use_color in (False, True):
                    yield (f"sunrgbd_{s}_a{int(augment)}_h{int(use_height)}_c{int(use_color)}", s,
                           dict(augment=augment, use_height=use_height, use_color=use_color))


def write_scenes(path):
    for j, (name, n, k) in enumerate(SCANNET):
        synth.write_scannet_detection_scene(path, name, 100 + j, n, k)
    for j, (name, n, k) in enumerate(SUNRGBD):
        synth.write_sunrgbd_detection_scene(path, name, 200 + j, n, k)


def main():
    mods = det_data_ref.load()
    assert mods is not None, "the original is not staged: run oracle/stage_ref.py"
    out = {}
    with tempfile.TemporaryDirectory() as d:
        write_scenes(d)
        for f in sorted(os.listdir(d)):
            stem, ext = os.path.splitext(f)
            if ext == ".npy":
                out[f"files/{stem}"] = np.load(os.path.join(d, f))
            else:
                with np.load(os.path.join(d, f)) as z:
                    for key in z.files:
                        out[f"files/{stem}/{key}"] = z[key]
        rng = np.random.RandomState(7)          # the legacy global generator np.random.* draws from, seeded
        for (cases, cls, scenes) in ((scannet_cases(), mods[0].ScannetDetectionDataset, SCANNET),
                                     (sunrgbd_cases(), mods[1].SunrgbdDetectionVotesDataset, SUNRGBD)):
            for case, s, opt in cases:
                rec = []

                def draws(kind, *a, **kw):
                    v = rng.random_sample(*a) if kind == "random" else rng.choice(*a, **kw)
                    rec.append((kind, v))
                    return v
                item = det_data_ref.item(cls, d, [x[0] for x in scenes], NUM_POINTS, idx=s, draws=draws, **opt)
                for k, v in item.items():
                    out[f"{case}/{k}"] = np.asarray(v)
                out[f"{case}/draw_kinds"] = np.array([k for k, _ in rec])
                for i, (_, v) in enumerate(rec):
                    out[f"{case}/draw{i}"] = np.asarray(v)
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "det_data.npz")
    np.savez_compressed(dst, **out)
    print(dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
