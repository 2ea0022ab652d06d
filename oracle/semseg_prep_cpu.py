"""numpy restatement of the reference's semantic-segmentation preprocessing (`downstream/semseg/lib/datasets/preprocessing/stanford.py`,
`preprocessing/scannet.py`, the PLY writer of `lib/pc_utils.py:41-70`): the checker of pointcontrast_b200/semseg_prep.py, and the host
route of profiles/bench_semseg_prep.py where the original is not staged.  Nothing under pointcontrast_b200/ imports this."""
import glob
import os
from pathlib import Path

import numpy as np

from oracle import semseg_data_cpu

CLASSES = ['clutter', 'beam', 'board', 'bookcase', 'ceiling', 'chair', 'column', 'door', 'floor', 'sofa', 'stairs', 'table', 'wall',
           'window']
PLY_DTYPE = [('x', 'f4'), ('y', 'f4'), ('z', 'f4'), ('red', 'u1'), ('green', 'u1'), ('blue', 'u1'), ('label', 'u1')]
BUGS = {'train/scene0270_00.ply': 50, 'train/scene0270_02.ply': 50, 'train/scene0384_00.ply': 149}


def write_ply(rows, path):
    """`PlyData([PlyElement.describe(rows, 'vertex')]).write(path)` of the plyfile the original ships: CRLF header, little-endian body."""
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(rows)}"]
    header += [f"property {'float' if rows.dtype[k].kind == 'f' else 'uchar'} {k}" for k in rows.dtype.names]
    with open(path, "wb") as f:
        f.write(("\r\n".join(header + ["end_header"]) + "\r\n").encode("ascii"))
        f.write(rows.astype([(k, "<" + rows.dtype[k].str[1:]) for k in rows.dtype.names]).tobytes())


def save_point_cloud(points_3d, path):
    """`lib/pc_utils.py:41-70` with `with_label=True`: each value through `float` / `int`, then the 7-field vertex table."""
    rows = np.array([tuple(t(v) for t, v in zip((float, float, float, int, int, int, int), r)) for r in points_3d], dtype=PLY_DTYPE)
    write_ply(rows, path)


def parse_lines(f):
    """`stanford.py:50-55`: `[float(t) for t in l.split()]` per line of a text-mode file, a line where it raises skipped."""
    rows = []
    for line in f:
        try:
            rows.append([float(t) for t in line.split()])
        except Exception:
            continue
    return rows


def values(rows):
    """`stanford.py:58-62` on the parsed rows: xyz float32 [N, 3], rgb uint8 [N, 3]; raises where the original's np.array or assert do."""
    a = np.array(rows)
    if a.ndim != 2 or a.shape[1] != 6:
        raise ValueError(f"parsed rows of shape {a.shape}, not (N, 6)")
    a = a.astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        return a[:, :3].astype(np.float32), a[:, 3:].astype(np.uint8)


def read_txt(path):
    with open(path) as f:
        return values(parse_lines(f))


def sparse_quantize(coords, feats=None, labels=None, ignore_label=255, return_index=False, quantization_size=1):
    """`ME.utils.sparse_quantize` (0.4.3, as recalled) with a float quantisation size: cells `floor(float64(coords) / quantization_size)`
    (true fp64 division), then the integer rule of `semseg_data_cpu.sparse_quantize`.  Cells outside +-2^20 raise."""
    c = np.floor(np.asarray(coords).astype(np.float64) / np.float64(quantization_size))
    if not np.isfinite(c).all() or (np.abs(c) >= 1 << 20).any():
        raise ValueError("a cell lies outside +-2^20")
    return semseg_data_cpu.sparse_quantize(c.astype(np.int64), feats, None if labels is None else np.asarray(labels).reshape(-1),
                                           ignore_label=ignore_label, return_index=return_index)


def convert_room(subclouds):
    """The rows `stanford.py:84-106` writes for one room's annotation files (in the given order)."""
    coords, feats, labels = [], [], []
    for sub in subclouds:
        xyz, rgb = read_txt(sub)
        clsidx = CLASSES.index(os.path.basename(sub).split("_")[0])
        coords.append(xyz)
        feats.append(rgb)
        labels.append(np.full((len(xyz), 1), clsidx, np.int32))
    coords, feats, labels = np.concatenate(coords), np.concatenate(feats), np.concatenate(labels)
    inds, collabels = sparse_quantize(coords, feats, labels, return_index=True, ignore_label=255, quantization_size=0.01)
    return np.concatenate((coords[inds], feats[inds], collabels[:, None]), axis=1)


def convert_stanford(in_root, out_root):
    """`Stanford3DDatasetConverter.convert_to_ply` (`stanford.py:66-112`)."""
    for txtfile in glob.glob(os.path.join(in_root, "*/*/*.txt")):
        file_sp = os.path.normpath(txtfile).split(os.path.sep)
        target = os.path.join(out_root, file_sp[-3])
        out_file = os.path.join(target, file_sp[-2] + ".ply")
        if os.path.exists(out_file):
            continue
        subclouds = glob.glob(os.path.join(os.path.dirname(txtfile), "Annotations/*.txt"))
        if subclouds:
            rows = convert_room(subclouds)
            os.makedirs(target, exist_ok=True)
            save_point_cloud(rows, out_file)


def generate_splits(out_root, split_path):
    """`stanford.py:115-127` writing to `split_path`."""
    os.makedirs(split_path, exist_ok=True)
    for i in range(1, 7):
        files = glob.glob(os.path.join(out_root, f"Area_{i}", "*.ply"))
        with open(os.path.join(split_path, f"area{i}.txt"), "w") as f:
            f.write("\n".join(os.path.relpath(p, out_root) for p in files))


def read_plyfile(path):
    """`lib/pc_utils.py` `read_plyfile`: every vertex column cast to their common dtype."""
    from pointcontrast_b200.semseg_data import read_ply
    v = read_ply(path)
    dt = np.result_type(*[v.dtype[k] for k in v.dtype.names])
    return np.stack([v[k].astype(dt) for k in v.dtype.names], 1)


def convert_scannet(raw_root, out_root):
    """`preprocessing/scannet.py` run serially: one write per scene, then the BUGS rewrite."""
    for phase, sub in (("train", "scans"), ("test", "scans_test")):
        out = Path(out_root) / phase
        out.mkdir(parents=True, exist_ok=True)
        for f in (Path(raw_root) / sub).glob("*/*_vh_clean_2.ply"):
            pc = read_plyfile(f)
            assert np.unique(pc[:, -1]).size == 1
            label_f = f.parent / (f.stem + ".labels" + f.suffix)
            if label_f.is_file():
                label = read_plyfile(label_f)
                assert pc.shape[0] == label.shape[0]
                assert np.allclose(pc[:, :3], label[:, :3])
            else:
                label = np.zeros_like(pc)
            save_point_cloud(np.hstack((pc[:, :6], np.array([label[:, -1]]).T)), out / (f.name[:-len("_vh_clean_2.ply")] + f.suffix))
    for name, bug in BUGS.items():
        for f in Path(out_root).glob(name):
            pc = read_plyfile(f)
            pc[pc[:, -1] == bug, -1] = 0
            save_point_cloud(pc, f)
