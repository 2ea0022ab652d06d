"""Semantic-segmentation training PLYs from the released datasets (DESIGN.md 8f-14): the reference's
`downstream/semseg/lib/datasets/preprocessing/stanford.py` (S3DIS) and `preprocessing/scannet.py` (ScanNet), whose output files this
writes byte for byte.

    convert_stanford("Stanford3dDataset_v1.2_Aligned_Version", "stanford")   # <out>/Area_i/<room>.ply, then generate_splits
    generate_splits("stanford")                                              # <out>/splits/area{1..6}.txt
    convert_scannet("ScanNet", "scannet_processed")                          # <out>/{train,test}/<scene>.ply

    python -m pointcontrast_b200.semseg_prep stanford --input <Stanford3dDataset_v1.2_Aligned_Version> --output <dir>
    python -m pointcontrast_b200.semseg_prep scannet --input <ScanNet> --output <dir>

S3DIS runs on the GPU, one room at a time: a reader thread reads the next room's annotation files into pinned memory while the device
finds the lines of the current one (pcb_text_lines), parses them (pcb_s3dis_parse), quantises them to 1 cm with their labels
(pcb_voxelize_labels) and writes the PLY body (pcb_ply_rows); a writer thread writes the files.  The lines the device cannot decide
exactly, and every file holding a non-ASCII byte, are parsed on the host with the original's own expression, so the output is the
original's for any input.  ScanNet needs no GPU: one read, one column stack and one write per scene.

Deliberate differences from the reference (DESIGN.md section 5): the split files go to `<out>/splits/`, where `StanfordDataset` reads
them (the reference writes `./splits/stanford/` under the working directory), and the 1 cm cells are `floor(float64(x) / 0.01)`, the
rule MinkowskiEngine 0.4.3's `sparse_quantize` is recalled to compute and which could not be checked against it.
"""
import argparse
import ctypes
import glob
import os
import queue
import threading
import time
from pathlib import Path

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, ptr, stream, workspace
from .pair_list import _read_ahead
from .semseg_data import read_ply, voxelize_labels

# `stanford.py:39-42`
CLASSES = ('clutter', 'beam', 'board', 'bookcase', 'ceiling', 'chair', 'column', 'door', 'floor', 'sofa', 'stairs', 'table', 'wall',
           'window')
IGNORE_LABEL = 255
QUANTIZATION_SIZE = 0.01
# `lib/pc_utils.py:49-51`; the header is what `PlyData([el]).write` of the plyfile the original ships
# (`pretrain/data_preprocess/scannet_pair/plyfile.py`) writes.  The semseg code imports an unpinned pip plyfile; this pins that copy.
PLY_DTYPE = np.dtype([('x', '<f4'), ('y', '<f4'), ('z', '<f4'), ('red', 'u1'), ('green', 'u1'), ('blue', 'u1'), ('label', 'u1')])
_HEADER = ("ply\r\nformat binary_little_endian 1.0\r\nelement vertex {}\r\nproperty float x\r\nproperty float y\r\nproperty float z\r\n"
           "property uchar red\r\nproperty uchar green\r\nproperty uchar blue\r\nproperty uchar label\r\nend_header\r\n")
# `preprocessing/scannet.py:12-20`
SCANNET_SUBSETS = {'train': 'scans', 'test': 'scans_test'}
SCANNET_POINTCLOUD_FILE = '_vh_clean_2.ply'
SCANNET_BUGS = {'train/scene0270_00.ply': 50, 'train/scene0270_02.ply': 50, 'train/scene0384_00.ply': 149}


def ply_header(n):
    return _HEADER.format(n).encode('ascii')


# ---------------------------------------------------------------------------------------------------------------- S3DIS

def _class_index(path):
    """`stanford.py:91`: the label of an annotation file; an unknown class raises."""
    name = os.path.basename(path).split('_')[0]
    if name not in CLASSES:
        raise ValueError(f"{path}: unknown S3DIS class {name!r} (classes: {', '.join(CLASSES)})")
    return CLASSES.index(name)


def _host_values(rows):
    """xyz float32, rgb uint8 and the int64 1 cm cells of parsed rows [[x, y, z, r, g, b], ...] (`stanford.py:58-62`)."""
    a = np.array(rows, dtype=np.float64).reshape(-1, 6).astype(np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        rgb = a[:, 3:].astype(np.uint8)
        cell = np.floor(a[:, :3].astype(np.float64) / QUANTIZATION_SIZE)
    if not np.isfinite(cell).all() or (np.abs(cell) >= 1 << 20).any():
        raise ValueError("a coordinate is not finite or its 1 cm cell lies outside +-2^20")
    return a[:, :3].copy(), rgb, cell.astype(np.int32)


def _parse_line(line):
    """`stanford.py:51-55` on one line: its values, or None where the original's `except` skips it."""
    try:
        return [float(t) for t in line.split()]
    except Exception:
        return None


def _read_txt_host(path):
    """`stanford.py:47-64` on a whole file, through Python's text mode (files with a non-ASCII byte: their decoding is the original's)."""
    with open(path) as f:
        rows = [r for r in map(_parse_line, f) if r is not None]
    if not rows or any(len(r) != 6 for r in rows):
        raise ValueError(f"{path}: {len(rows)} parsed lines, not all of 6 values (the original raises)")
    return rows


def _load_room(files):
    """The room's annotation files, concatenated into pinned memory (16-byte padded), their offsets and labels."""
    labels = np.array([_class_index(p) for p in files], np.int32)
    sizes = [os.path.getsize(p) for p in files]
    off = np.zeros(len(files) + 1, np.int64)
    np.cumsum(sizes, out=off[1:])
    text = torch.empty(max(16, (int(off[-1]) + 15) // 16 * 16), dtype=torch.uint8, pin_memory=True)
    view = memoryview(text.numpy())
    for p, a, b in zip(files, off[:-1], off[1:]):
        with open(p, 'rb') as f:
            if f.readinto(view[a:b]) != b - a:
                raise OSError(f"{p}: changed size while being read")
    return dict(files=files, labels=labels, off=off, text=text)


def parse_room(room, device):
    """The parsed, kept points of a room loaded by `_load_room`, in file and line order: xyz fp32 [N, 3], rgb uint8 [N, 3], labels int32 [N]
    and 1 cm cells int32 [N, 3], on the device.  Raises where the original's `read_txt` does."""
    files, off, labels = room['files'], room['off'], room['labels']
    F, n = len(files), int(off[-1])
    text = room['text'].to(device, non_blocking=True)
    off_d = torch.from_numpy(off).to(device, non_blocking=True)
    lab_d = torch.from_numpy(labels).to(device, non_blocking=True)
    nchunks = (n + 15) // 16
    chunk_off = torch.empty(nchunks + 1, dtype=torch.int64, device=device)
    flags = torch.empty(F, dtype=torch.int32, device=device)
    L = ctypes.c_int64(0)
    wsb = lib.pcb_text_lines_ws_bytes(n)
    ws = workspace(wsb, device)
    check(lib.pcb_text_lines(ptr(text), n, ptr(off_d), F, ptr(chunk_off), ptr(flags), ctypes.byref(L), ptr(ws), wsb, stream()))
    L = L.value
    line_start = torch.empty(L + 1, dtype=torch.int64, device=device)
    xyz = torch.empty(L, 3, dtype=torch.float32, device=device)
    rgb = torch.empty(L, 3, dtype=torch.uint8, device=device)
    lab = torch.empty(L, dtype=torch.int32, device=device)
    cell = torch.empty(L, 3, dtype=torch.int32, device=device)
    status = torch.empty(L, dtype=torch.uint8, device=device)
    check(lib.pcb_s3dis_parse(ptr(text), n, ptr(off_d), ptr(lab_d), F, ptr(chunk_off), ptr(flags), L, ptr(line_start), ptr(xyz), ptr(rgb),
                              ptr(lab), ptr(cell), ptr(status), stream()))
    line_file = torch.searchsorted(off_d, line_start[:L], right=True) - 1
    status_h = status.cpu().numpy()
    nonascii = np.flatnonzero(flags.cpu().numpy() & _lib.TEXT_NONASCII)
    file_h = line_file.cpu().numpy() if (status_h != _lib.LINE_KEPT).any() else None
    kept_per_file = np.zeros(F, np.int64)
    if file_h is None:
        kept_per_file += np.bincount(line_file.cpu().numpy(), minlength=F)
    else:
        bad = np.flatnonzero((status_h == _lib.LINE_ERROR) & ~np.isin(file_h, nonascii))
        if len(bad):
            raise ValueError(f"{files[file_h[bad[0]]]}: a line without 6 values (the original raises)")
        host = np.flatnonzero((status_h == _lib.LINE_HOST) & ~np.isin(file_h, nonascii))
        if len(host):                                   # lines of ASCII files the device left undecided: Python's float()
            starts = line_start.cpu().numpy()
            raw = room['text'].numpy()
            kept, rows = [], []
            for j in host.tolist():
                b = min(starts[j + 1], off[file_h[j] + 1])
                r = _parse_line(raw[starts[j]:b].tobytes().decode('ascii'))
                if r is None:
                    continue
                if len(r) != 6:
                    raise ValueError(f"{files[file_h[j]]}: a line with {len(r)} values (the original raises)")
                kept.append(j)
                rows.append(r)
            status_h[host] = _lib.LINE_SKIPPED
            if kept:
                status_h[kept] = _lib.LINE_KEPT
                hx, hr, hc = _host_values(rows)
                idx = torch.tensor(kept, dtype=torch.int64, device=device)
                xyz[idx] = torch.from_numpy(hx).to(device)
                rgb[idx] = torch.from_numpy(hr).to(device)
                cell[idx] = torch.from_numpy(hc).to(device)
        status_h[np.isin(file_h, nonascii)] = _lib.LINE_SKIPPED
        kept_per_file += np.bincount(file_h[status_h == _lib.LINE_KEPT], minlength=F)
    keep = torch.from_numpy(np.flatnonzero(status_h == _lib.LINE_KEPT)).to(device)
    parts = [t.index_select(0, keep) for t in (xyz, rgb, lab, cell)]
    if len(nonascii):                                   # whole files through Python's text mode, spliced in at their place
        segs, at = [[] for _ in parts], 0
        kept_start = np.concatenate([[0], np.cumsum(kept_per_file)])
        for f in nonascii.tolist():
            hx, hr, hc = _host_values(_read_txt_host(files[f]))
            kept_per_file[f] = len(hx)
            host_part = [torch.from_numpy(hx), torch.from_numpy(hr), torch.full((len(hx),), int(labels[f]), dtype=torch.int32),
                         torch.from_numpy(hc)]
            cut = int(kept_start[f])
            for s, p, h in zip(segs, parts, host_part):
                s += [p[at:cut], h.to(device)]
            at = cut
        parts = [torch.cat(s + [p[at:]]) for s, p in zip(segs, parts)]
    empty = np.flatnonzero(kept_per_file == 0)
    if len(empty):
        raise ValueError(f"{files[empty[0]]}: no parsed line (the original raises)")
    return parts


def quantize_room(xyz, rgb, labels, cell):
    """`ME.utils.sparse_quantize(coords, feats, labels, return_index=True, ignore_label=255, quantization_size=0.01)` and the rows of
    `stanford.py:106`: the PLY body (uint8 [M * 16], device)."""
    _, sel, vl = voxelize_labels(cell, labels, IGNORE_LABEL)
    sel = sel.int()
    body = torch.empty(len(sel) * 16, dtype=torch.uint8, device=xyz.device)
    check(lib.pcb_ply_rows(ptr(xyz), ptr(rgb), ptr(sel), ptr(vl), len(sel), ptr(body), stream()))
    return body


class _FileWriter:
    """Writes (path, header, body) on a thread, at most `depth` files queued; the first error is raised by `check`."""

    def __init__(self, depth):
        self.q = queue.Queue(maxsize=depth)
        self.err = None
        self.busy_s = 0.0
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()

    def _run(self):
        while (item := self.q.get()) is not None:
            if self.err is None:                        # after an error the queue is drained without writing
                t = time.perf_counter()
                try:
                    path, header, body = item
                    os.makedirs(os.path.dirname(path), exist_ok=True)
                    with open(path, 'wb') as f:
                        f.write(header)
                        f.write(body)
                except BaseException as e:
                    self.err = e
                self.busy_s += time.perf_counter() - t

    def put(self, path, header, body):
        self.check()
        self.q.put((path, header, body))

    def close(self):
        self.q.put(None)
        self.t.join()

    def check(self):
        if self.err is not None:
            raise self.err


def stanford_rooms(in_root, out_root, log=print):
    """`stanford.py:73-92` without the work: [(room text file, output file, annotation files)] of the rooms to convert, in glob order.
    An existing output is skipped (so is a second text file of a room already listed); a room without annotation files is reported."""
    todo, planned = [], set()
    for txtfile in glob.glob(os.path.join(in_root, '*/*/*.txt')):
        file_sp = os.path.normpath(txtfile).split(os.path.sep)
        out_file = os.path.join(out_root, file_sp[-3], file_sp[-2] + '.ply')
        if out_file in planned or os.path.exists(out_file):
            if log:
                log(f"{out_file}  exists")
            continue
        subclouds = glob.glob(os.path.join(os.path.dirname(txtfile), 'Annotations/*.txt'))
        if not subclouds:
            if log:
                log(f"{txtfile}  has 0 files.")
            continue
        planned.add(out_file)
        todo.append((txtfile, out_file, subclouds))
    return todo


def convert_stanford(in_root, out_root, device=None, log=print, splits=True):
    """`Stanford3DDatasetConverter.convert_to_ply(in_root, out_root)` (`stanford.py:66-112`) then `generate_splits(out_root)`.  Returns
    the wall seconds of reading (on the reader thread), of the device work (including the copies back) and of writing (on the writer
    thread).  Every thread has ended when this returns or raises."""
    device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
    todo = stanford_rooms(in_root, out_root, log)
    secs = dict(read=0.0, device=0.0, write=0.0)

    def load(item):
        t = time.perf_counter()
        room = _load_room(item[2])
        secs['read'] += time.perf_counter() - t
        return room

    writer = _FileWriter(2)
    try:
        with torch.cuda.device(device), _read_ahead(todo, load) as rooms:
            for (txtfile, out_file, _), room in rooms:
                t = time.perf_counter()
                xyz, rgb, lab, cell = parse_room(room, device)
                body = quantize_room(xyz, rgb, lab, cell)
                host = torch.empty(body.shape, dtype=torch.uint8, pin_memory=True)
                host.copy_(body, non_blocking=True)
                torch.cuda.current_stream(device).synchronize()
                secs['device'] += time.perf_counter() - t
                writer.put(out_file, ply_header(len(body) // 16), host.numpy())
                if log:
                    log(f"{txtfile}: {len(xyz)} points, {len(body) // 16} voxels -> {out_file}")
    finally:
        writer.close()
    writer.check()
    secs['write'] = writer.busy_s
    if splits:
        generate_splits(out_root)
    return secs


def generate_splits(out_root):
    """`stanford.py:115-127`: `area{i}.txt` = the relative paths of `<out_root>/Area_i/*.ply` in glob order, joined by newlines, written to
    `<out_root>/splits/` (the reference: `./splits/stanford/`), where `semseg_data.StanfordDataset` reads them."""
    split_path = os.path.join(out_root, 'splits')
    os.makedirs(split_path, exist_ok=True)
    for i in range(1, 7):
        files = glob.glob(os.path.join(out_root, f'Area_{i}', '*.ply'))
        with open(os.path.join(split_path, f'area{i}.txt'), 'w') as f:
            f.write('\n'.join(os.path.relpath(p, out_root) for p in files))


# ---------------------------------------------------------------------------------------------------------------- ScanNet

def _table(path):
    """`lib/pc_utils.py` `read_plyfile`: the vertex table with every column cast to their common dtype (pandas' `.values`)."""
    v = read_ply(path)
    dt = np.result_type(*[v.dtype[k] for k in v.dtype.names])
    return np.stack([v[k].astype(dt) for k in v.dtype.names], 1)


def scannet_scene(ply_path, out_dir):
    """`preprocessing/scannet.py:24-42` for one `<scene>_vh_clean_2.ply`, with its BUGS fix (`:55-64`) applied before the one write.
    Raises where the original asserts.  Returns the output path."""
    ply_path, out_dir = Path(ply_path), Path(out_dir)
    pc = _table(ply_path)
    if np.unique(pc[:, -1]).size != 1:
        raise ValueError(f"{ply_path}: the last vertex column (alpha) is not constant")
    label_f = ply_path.parent / (ply_path.stem + '.labels' + ply_path.suffix)
    if label_f.is_file():
        label = _table(label_f)
        if pc.shape[0] != label.shape[0]:
            raise ValueError(f"{label_f}: {label.shape[0]} vertices, {ply_path} has {pc.shape[0]}")
        if not np.allclose(pc[:, :3], label[:, :3]):
            raise ValueError(f"{label_f}: vertices differ from {ply_path}")
        lab = label[:, -1]
    else:                                               # no labels for the test scenes
        lab = np.zeros(len(pc), pc.dtype)
    out_f = out_dir / (ply_path.name[:-len(SCANNET_POINTCLOUD_FILE)] + ply_path.suffix)
    rows = np.empty(len(pc), PLY_DTYPE)
    for k, name in enumerate(('x', 'y', 'z')):
        rows[name] = pc[:, k].astype(np.float64)
    for k, name in enumerate(('red', 'green', 'blue')):
        rows[name] = _uint8(pc[:, 3 + k], ply_path)
    lab = _uint8(lab, ply_path)
    bug = SCANNET_BUGS.get(f"{out_dir.name}/{out_f.name}")
    if bug is not None:
        lab[lab == bug] = 0
    rows['label'] = lab
    with open(out_f, 'wb') as f:
        f.write(ply_header(len(rows)))
        f.write(rows.tobytes())
    return out_f


def _uint8(col, path):
    """`int(v)` stored as u1 (`lib/pc_utils.py:60-63`): truncation toward zero; outside [0, 255] numpy raises, so does this."""
    v = np.trunc(col.astype(np.float64))
    if not np.isfinite(v).all() or (v < 0).any() or (v > 255).any():
        raise ValueError(f"{path}: a colour or label outside [0, 255]")
    return v.astype(np.uint8)


def convert_scannet(raw_root, out_root, log=print):
    """`preprocessing/scannet.py`: every `<raw_root>/scans/*/*_vh_clean_2.ply` to `<out_root>/train/<scene>.ply`, every
    `<raw_root>/scans_test/...` to `<out_root>/test/`, x, y, z, rgb and the `.labels.ply` label (0 where there is none)."""
    out = []
    for phase, sub in SCANNET_SUBSETS.items():
        phase_out = Path(out_root) / phase
        phase_out.mkdir(parents=True, exist_ok=True)
        for f in (Path(raw_root) / sub).glob('*/*' + SCANNET_POINTCLOUD_FILE):
            out.append(scannet_scene(f, phase_out))
            if log:
                log(f"{f} -> {out[-1]}")
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m pointcontrast_b200.semseg_prep", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="dataset", required=True)
    s = sub.add_parser("stanford", help="S3DIS rooms -> <output>/Area_i/<room>.ply and <output>/splits/area{1..6}.txt (on the GPU)")
    s.add_argument("--input", required=True, help="Stanford3dDataset_v1.2_Aligned_Version")
    s.add_argument("--output", required=True)
    c = sub.add_parser("scannet", help="ScanNet scans -> <output>/{train,test}/<scene>.ply")
    c.add_argument("--input", required=True, help="the ScanNet root holding scans/ and scans_test/")
    c.add_argument("--output", required=True)
    args = ap.parse_args(argv)
    if args.dataset == "stanford":
        convert_stanford(args.input, args.output)
    else:
        convert_scannet(args.input, args.output)


if __name__ == "__main__":
    main()
