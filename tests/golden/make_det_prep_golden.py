"""Writes tests/golden/det_prep.npz: small synthetic ScanNet and SUN RGB-D inputs (file bytes) and the SHA-256 of every array the staged
original preprocessing (oracle/det_prep_ref.py) writes from them under np.random.seed(SEED), so that tests/test_gpu_det_prep.py checks the
GPU route against the original without the reference tree.

    python tests/golden/make_det_prep_golden.py
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import det_prep_ref as R, stage_ref  # noqa: E402
from pointcontrast_b200 import synth  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "det_prep.npz")
SEED = 11
SCENES = (("scene0100_00", None), ("scene0101_00", "unknown_seg"), ("scene0102_00", None))


def write_inputs(d):
    os.makedirs(d, exist_ok=True)
    synth.write_scannet_label_map(os.path.join(d, "labels.tsv"))
    for k, (name, fault) in enumerate(SCENES):
        synth.write_scannet_det_raw_scene(os.path.join(d, "scans"), name, 40 + k, n=1500, n_seg=40, fault=fault)
    synth.write_sunrgbd_export(os.path.join(d, "sunrgbd_trainval"), 41, n_scenes=4, n_points=600, big_points=900)


def digests(root):
    """{relative path[:member]: sha256 of the array's bytes, dtype and shape} of every .npy / .npz under root."""
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            rel = os.path.relpath(p, root)
            arrays = {"": np.load(p)} if f.endswith(".npy") else dict(np.load(p))
            for k, a in arrays.items():
                out[rel + (":" + k if k else "")] = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()
    return out


def main():
    assert R.available() or "det_prep" in stage_ref.stage(), "the original is not present"
    with tempfile.TemporaryDirectory() as d:
        write_inputs(os.path.join(d, "in"))
        files = sorted(os.path.relpath(os.path.join(a, f), os.path.join(d, "in")) for a, _, fs in os.walk(os.path.join(d, "in")) for f in fs)
        blobs = [open(os.path.join(d, "in", f), "rb").read() for f in files]
        np.random.seed(SEED)
        R.scannet(os.path.join(d, "in", "scans"), os.path.join(d, "in", "labels.tsv"), [n for n, _ in SCENES], os.path.join(d, "out", "scannet"))
        R.sunrgbd(os.path.join(d, "in", "sunrgbd_trainval"), os.path.join(d, "out", "sunrgbd"), v1=True)
        dig = digests(os.path.join(d, "out"))
    off = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    np.savez_compressed(OUT, paths=np.array(files), data=np.frombuffer(b"".join(blobs), np.uint8), off=off, outputs=np.array(sorted(dig)),
                        sha=np.array([dig[k] for k in sorted(dig)]))
    print("wrote", OUT, len(files), "inputs,", len(dig), "output arrays")


if __name__ == "__main__":
    main()
