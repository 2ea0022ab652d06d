"""Writes tests/golden/semseg_prep.npz: a small S3DIS tree with adversarial annotation text and the output the original converter
(oracle/semseg_prep_ref.py, staged by `python oracle/stage_ref.py`) writes for it -- each room's PLY bytes and the split files.

    python tests/golden/make_semseg_prep_golden.py

Keys: `paths` (relative input paths), `text` (their bytes concatenated) with `text_off`, `outputs` (relative output paths), `out`
(their bytes concatenated) with `out_off`.  The original's ME call runs on the oracle's restatement (oracle/semseg_prep_ref.py)."""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import semseg_prep_ref as R, stage_ref  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "semseg_prep.npz")


def tree():
    """{relative path: bytes} of the input tree."""
    rng = np.random.default_rng(14)
    files = {}
    adversarial = (b"-0.000 0.005 -0.005 1 2 3\n0.010 -0.010 0.015 4 5 6\r\n1e-3 +.5 5. 7 8 9\r"
                   b"12.345\t6.789\x0b-1.001\x0c10 11 12\x1c\n3.141\x1d2.718\x1e1.414\x1f13 14 15 \n"
                   b"1.2.3 0 0 0 0 0\n1\x102 0 0 0 0 0\n1_0 0.1 0.2 16 17 18\n0.12345678901234567890 1.5 2.5 255.9 0 1\n"
                   b"0.009999 0.019999 -0.0099 200 100 50\n0.005 0.005 -0.005 9 9 9")
    files["Area_1/hall_1/Annotations/wall_1.txt"] = adversarial
    mm = rng.integers(-3000, 3000, size=(4000, 3))
    mm[:1000] = mm[:1000] // 10 * 10
    rgb = rng.integers(0, 256, size=(4000, 3))
    lines = [b"%.3f %.3f %.3f %d %d %d" % (x / 1000, y / 1000, z / 1000, r, g, b) for (x, y, z), (r, g, b) in zip(mm.tolist(), rgb.tolist())]
    files["Area_1/hall_1/Annotations/chair_1.txt"] = b"\n".join(lines[:2500]) + b"\n"
    files["Area_1/hall_1/Annotations/table_2.txt"] = b"\n".join(lines[2000:]) + b"\n" + adversarial[:52]
    files["Area_1/hall_1/Annotations/ceiling_1.txt"] = "0.001 0.002 0.003 1 2 3\n0.004 0.005 0.006 4 5 6\n".encode("utf-8")
    files["Area_1/hall_1/hall_1.txt"] = b"".join(files[k] for k in list(files))
    files["Area_5/office_3/Annotations/floor_1.txt"] = b"\n".join(lines[:300])
    files["Area_5/office_3/Annotations/clutter_1.txt"] = b"\r\n".join(lines[100:200]) + b"\r\n"
    files["Area_5/office_3/office_3.txt"] = b"\n".join(lines[:300])
    files["Area_5/storage_2/storage_2.txt"] = b"0 0 0 0 0 0\n"
    return files


def main():
    assert R.available() or "semseg_prep" in stage_ref.stage(), "the original is not present"
    files = tree()
    with tempfile.TemporaryDirectory() as d:
        for rel, data in files.items():
            os.makedirs(os.path.dirname(os.path.join(d, "in", rel)), exist_ok=True)
            with open(os.path.join(d, "in", rel), "wb") as f:
                f.write(data)
        R.stanford(os.path.join(d, "in"), os.path.join(d, "out"), os.path.join(d, "cwd"))
        outs = {}
        for rel in ("Area_1/hall_1.ply", "Area_5/office_3.ply"):
            outs[rel] = open(os.path.join(d, "out", rel), "rb").read()
        for i in range(1, 7):
            outs[f"splits/area{i}.txt"] = open(os.path.join(d, "cwd", "splits", "stanford", f"area{i}.txt"), "rb").read()
    pack = lambda blobs: (np.frombuffer(b"".join(blobs), np.uint8), np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64))
    text, text_off = pack(list(files.values()))
    out, out_off = pack(list(outs.values()))
    np.savez_compressed(OUT, paths=np.array(list(files)), text=text, text_off=text_off, outputs=np.array(list(outs)), out=out, out_off=out_off)
    print("wrote", OUT, {k: len(v) for k, v in outs.items()})


if __name__ == "__main__":
    main()
