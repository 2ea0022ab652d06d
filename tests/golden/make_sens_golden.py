"""Generates tests/golden/sens_extract.npz: what the reference's own `reader.py` + `point_cloud_extractor.py`, unmodified, staged by
oracle/stage_ref.py and run by oracle/sens_ref.py with the stand-ins its docstring lists, extract from a small synthetic `.sens` file:

    python oracle/stage_ref.py && python tests/golden/make_sens_golden.py

The scan (`synth.synth_sens_scan`, 64 x 48 depth, 9 frames, frame_skip 2, so 5 frames kept and 4 seeked past) holds zero-depth holes
and depth-65535 pixels in every frame, an all-zero frame (2), a frame with a block of depth 65535 (6) and a frame stored with an
all -inf pose (4, as ScanNet stores a frame without tracking).  The file holds the `.sens` bytes, the kept frame indices, the text of
each `pose/<f>.txt` and of `intrinsic/intrinsic_depth.txt`, and every `pcd/<f>.npz` frame (rows concatenated, `offsets` delimiting
them).  The reference cannot extract a frame with exactly one valid pixel (`.squeeze()` makes it a vector), so there is none here.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "sens_extract.npz")
FRAME_SKIP = 2


def scan():
    """(depth, poses, intrinsic) of the golden's `.sens` file."""
    from pointcontrast_b200 import synth
    depth, poses, K = synth.synth_sens_scan(21, 9, width=64, height=48, holes=0.1, far=0.01, bad_poses=(4,))
    depth[2] = 0
    depth[6, 10:20, 30:50] = 65535
    return depth, poses, K


def main():
    sys.path.insert(0, ROOT)
    from oracle import sens_ref
    from pointcontrast_b200 import synth
    if not sens_ref.available():
        raise SystemExit("the reference's .sens scripts are not staged: run oracle/stage_ref.py")
    depth, poses, K = scan()
    with tempfile.TemporaryDirectory() as tmp:
        sens = os.path.join(tmp, "scene0000_00.sens")
        synth.write_sens(sens, depth, poses, K, color_bytes=(2000, 4000))
        scene = os.path.join(tmp, "scene0000_00")
        sens_ref.extract(sens, scene, FRAME_SKIP)
        frames = list(range(0, len(depth), FRAME_SKIP))
        pcd = [np.load(os.path.join(scene, "pcd", f"{f}.npz"))["pcd"] for f in frames]
        np.savez_compressed(
            OUT, sens=np.frombuffer(open(sens, "rb").read(), np.uint8), frame_skip=FRAME_SKIP, frames=np.array(frames, np.int64),
            pose_text=np.array([open(os.path.join(scene, "pose", f"{f}.txt")).read() for f in frames]),
            intrinsic_text=np.array(open(os.path.join(scene, "intrinsic", "intrinsic_depth.txt")).read()),
            pcd=np.concatenate(pcd), offsets=np.concatenate([[0], np.cumsum([len(p) for p in pcd])]).astype(np.int64))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
