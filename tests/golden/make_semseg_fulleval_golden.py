"""Generates tests/golden/semseg_fulleval.npz: the reference's own `save_predictions` (`downstream/semseg/lib/utils.py:304-349`) and
`test_pointcloud` (`lib/datasets/scannet.py:131-172`, `stanford.py:41-84`), unmodified, staged by oracle/stage_ref.py and run by
oracle/semseg_fulleval_ref.py with the shims its docstring lists, on synthetic rooms:

    python oracle/stage_ref.py && python tests/golden/make_semseg_fulleval_golden.py

* ScanNet: 4 rooms (`synth.synth_labelled_room`), 2 cm voxels, each under its own rotation about z, scale and translation (the float32
  4x4 the voxelizer returns), seeded masked predictions over 20 classes, batch size 1;
* S3DIS: one area of 3 rooms, `hallway_1`, `office_1`, `office_2`, 5 cm voxels, 13 classes; `office_1` repeats some of its own rows and
  `office_2` holds rows of `office_1`, so the office group's de-duplication has work to do.

The original's KD-tree leaves the order of equal distances unspecified, so every original point whose nearest and second-nearest
centre (of its scene or group) are within 1e-6 m of each other is left out of the PLY files: the golden does not depend on a tie
rule.  The file holds the PLY vertices, the collated inputs (batch-first coords, transformation rows, masked predictions), the
reference's `pred_*.npy` arrays, ScanNet's `fulleval/<scene>.txt` bytes and the histograms `test_pointcloud` bins.

`scene(z, kind)` and `write_plys(z, kind, root)` unpack the file for the tests.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "semseg_fulleval.npz")
SCANNET_VALID = (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39)


def label_map(num_labels, ignore):
    """`VoxelizationDataset.__init__`'s label map (original -> masked, ignored -> 255) and the masked class count."""
    m, used = {}, 0
    for l in range(num_labels):
        if l in ignore:
            m[l] = 255
        else:
            m[l] = used
            used += 1
    m[255] = 255
    return m, used


KINDS = {"scannet": label_map(41, set(range(41)) - set(SCANNET_VALID)), "s3dis": label_map(14, {10})}


def _cat(arrs):
    return np.concatenate(arrs) if arrs else np.zeros(0), np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)


def _split(z, key):
    a, off = z[key], z[key + "_off"]
    return [a[off[i]:off[i + 1]] for i in range(len(off) - 1)]


def scene(z, kind):
    """The golden of `kind` as a dict: names, xyz / rgb / label (per file), coords / pred (per item), T [n, 17], npy (per item), hist,
    txt (ScanNet: bytes per file)."""
    p = kind + "_"
    out = {"names": [str(s) for s in z[p + "names"]], "T": z[p + "T"], "hist": z[p + "hist"]}
    for k in ("xyz", "rgb", "label", "coords", "pred", "npy") + (("txt",) if kind == "scannet" else ()):
        out[k] = _split(z, p + k)
    if kind == "scannet":
        out["txt"] = [bytes(t.astype(np.uint8)) for t in out["txt"]]
    return out


def write_plys(z, kind, root):
    """Writes the golden's PLY files and split file under root (ScanNet: `splits/scannetv2_val.txt`; S3DIS: `splits/val.txt`)."""
    from pointcontrast_b200 import synth
    s = scene(z, kind)
    os.makedirs(os.path.join(root, "splits"), exist_ok=True)
    for name, xyz, rgb, lab in zip(s["names"], s["xyz"], s["rgb"], s["label"]):
        os.makedirs(os.path.dirname(os.path.join(root, name)), exist_ok=True)
        synth.write_ply(os.path.join(root, name), xyz.reshape(-1, 3), rgb.reshape(-1, 3).astype(np.uint8), lab.astype(np.uint8))
    split = "scannetv2_val.txt" if kind == "scannet" else "val.txt"
    with open(os.path.join(root, "splits", split), "w") as f:
        f.write("\n".join(s["names"]) + "\n")
    return s


def _transform(rng, voxel, xyz):
    th = rng.uniform(-np.pi, np.pi)
    R = np.eye(4)
    R[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
    V = np.diag([1 / voxel * rng.uniform(0.9, 1.1)] * 3 + [1.0])
    T = R @ V
    c = np.floor(np.hstack([xyz, np.ones((len(xyz), 1))]) @ T[:3].T)
    M = np.eye(4)
    M[:3, 3] = -c.min(0)
    T = M @ T
    coords = np.unique((c - c.min(0)).astype(np.int32), axis=0)
    return T.astype(np.float32), coords


def _tie_free(centres, xyz, margin=1e-6):
    from scipy.spatial import cKDTree
    if len(centres) < 2:
        return np.ones(len(xyz), bool)
    d, _ = cKDTree(centres).query(xyz, k=2)
    return d[:, 1] - d[:, 0] > margin


def build(kind, tmp):
    from pointcontrast_b200 import synth
    from oracle import semseg_fulleval_ref as R
    lm, C = KINDS[kind]
    rng = np.random.default_rng(7 if kind == "scannet" else 8)
    if kind == "scannet":
        names = [f"scene{k:04d}_00_vh_clean_2.ply" for k in range(4)]
        rooms = [synth.synth_labelled_room(500 + k, 4000, scale=0.7 + 0.1 * k) for k in range(4)]
        voxel, groups = 0.02, [[0], [1], [2], [3]]
    else:
        names = [os.path.join("Area_5", f"{r}.ply") for r in ("hallway_1", "office_1", "office_2")]
        rooms = [list(synth.synth_labelled_room(600 + k, 3500, scale=0.7 + 0.1 * k, num_labels=14)) for k in range(3)]
        shared = [a[:600] for a in rooms[1]]
        rooms[1] = [np.concatenate([a, b[:200]]) for a, b in zip(rooms[1], shared)]
        rooms[2] = [np.concatenate([a, b]) for a, b in zip(rooms[2], shared)]
        voxel, groups = 0.05, [[0], [1, 2]]
    Ts, coords, preds = [], [], []
    pred_dir = os.path.join(tmp, kind + "_pred")
    os.makedirs(pred_dir)
    for i, (xyz, _, _) in enumerate(rooms):
        T, c = _transform(rng, voxel, xyz.astype(np.float64))
        p = rng.integers(0, C, len(c))
        Ts.append(np.concatenate([T.reshape(16), [0.0]]).astype(np.float32))
        coords.append(np.hstack([np.zeros((len(c), 1), np.int32), c]))
        preds.append(p)
        ds = R.dataset(kind, os.path.join(tmp, kind), names, lm, C)
        R.save_predictions(coords[-1], p, Ts[-1][None], ds, i, pred_dir)
    npy = [np.load(os.path.join(pred_dir, "pred_%04d_00.npy" % i)) for i in range(len(rooms))]
    for g in groups:
        centres = np.vstack([npy[i][:, :3] for i in g])
        for i in g:
            keep = _tie_free(centres, rooms[i][0].astype(np.float64))
            rooms[i] = [a[keep] for a in rooms[i]]
    root = os.path.join(tmp, kind)
    for name, (xyz, rgb, lab) in zip(names, rooms):
        os.makedirs(os.path.dirname(os.path.join(root, name)), exist_ok=True)
        synth.write_ply(os.path.join(root, name), xyz, rgb, lab)
    hists = R.test_pointcloud(R.dataset(kind, root, names, lm, C), pred_dir)
    z = {f"{kind}_names": np.array(names), f"{kind}_T": np.stack(Ts), f"{kind}_hist": np.sum(hists, 0).astype(np.int64)}
    for key, arrs in (("xyz", [r[0].reshape(-1) for r in rooms]), ("rgb", [r[1].reshape(-1) for r in rooms]),
                      ("label", [r[2] for r in rooms]), ("coords", [c.reshape(-1) for c in coords]),
                      ("pred", [p.astype(np.int32) for p in preds]), ("npy", [a.reshape(-1) for a in npy])):
        z[f"{kind}_{key}"], z[f"{kind}_{key}_off"] = _cat(arrs)
    if kind == "scannet":
        txt = [np.frombuffer(open(os.path.join(pred_dir, "fulleval", n[:12] + ".txt"), "rb").read(), np.uint8) for n in names]
        z["scannet_txt"], z["scannet_txt_off"] = _cat(txt)
    print(kind, "points", [len(r[0]) for r in rooms], "centres", [len(a) for a in npy], "hist total", int(z[f"{kind}_hist"].sum()))
    return z


def main():
    sys.path.insert(0, ROOT)
    z = {}
    with tempfile.TemporaryDirectory() as tmp:
        for kind in ("scannet", "s3dis"):
            z.update(build(kind, tmp))
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
