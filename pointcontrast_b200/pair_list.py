"""The pretraining pair list on the GPU (SURVEY.md 8f-10): from a scene's frames `<scene>/pcd/<frame>.npz` (`pcd` = fp64 world points
[N, 3]) to `<scene>/pcd/overlap.txt`, and from those to the list `overlap-30-full.txt` that `scannet_pairs.ScanNetMatchPairDataset`
reads -- the reference's `pretrain/data_preprocess/scannet_pair/compute_full_overlapping.py` and `generate_list.py`, which downsample
with open3d and make one KD-tree radius query per point for every ordered pair of frames.

    points, offsets, host = voxel_down_sample(xyz, offsets, 0.05)     # every frame of a scene in one call
    counts = overlap_counts(points, offsets, 0.075)                    # [F, F]: points of frame j with a neighbour in frame i
    compute_full_overlapping("scans/scene0000_00/pcd")                 # writes overlap.txt
    generate_list("scans")                                             # writes scans/overlap-30-full.txt

    python -m pointcontrast_b200.pair_list overlap --input_path scans/scene0000_00/pcd [more scene paths ...] [--voxel_size 0.05]
    python -m pointcontrast_b200.pair_list list --target_dir scans

Deliberate differences from the reference (DESIGN.md section 5): frames are taken in sorted file order (the reference uses `glob`
order, which depends on the file system; the unordered pairs and their values are the same), and an empty frame is dropped with the
frames holding a NaN (the reference divides by its zero size).
"""
import argparse
import ctypes
import glob
import os
import queue
import threading

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, ptr, stream
from .me import workspace

MAX_FRAMES = 4096


def _frames_args(xyz, offsets):
    _lib.require_cuda(xyz); _lib.require_cuda(offsets)
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise _lib.PcbError(f"xyz must be [N, 3], got {tuple(xyz.shape)}")
    xyz = xyz.contiguous().double()
    offsets = offsets.to(xyz.device, torch.int64).contiguous()
    return xyz, offsets, xyz.shape[0], offsets.shape[0] - 1


def voxel_down_sample(xyz, offsets, voxel_size):
    """open3d `voxel_down_sample` of every frame.  xyz: fp64 CUDA [N, 3], frame f = rows [offsets[f], offsets[f+1]) (int64 [F + 1]).
    Returns (points fp64 [M, 3] frame-major, ascending voxel index within a frame; offsets int64 [F + 1] on the device; the offsets as
    a host list).  Synchronises once."""
    xyz, offsets, n, F = _frames_args(xyz, offsets)
    out = torch.empty(max(n, 1), 3, dtype=torch.float64, device=xyz.device)
    out_off = torch.empty(max(F + 1, 1), dtype=torch.int64, device=xyz.device)
    host = (ctypes.c_int64 * max(F + 1, 1))()
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_voxel_down_sample_ws_bytes(n, F)
        ws = workspace(wsb, xyz.device, slot=6)
        check(lib.pcb_voxel_down_sample(ptr(xyz), n, ptr(offsets), F, float(voxel_size), ptr(out), ptr(out_off), host, ptr(ws), wsb,
                                        stream()))
    return out[:host[F]], out_off, list(host)


def overlap_counts(points, offsets, radius):
    """counts int64 CUDA [F, F]: counts[i, j] = the number of points of frame j with a point of frame i != j closer than `radius`
    (fp64, exact).  points: fp64 CUDA [N, 3], frames as in `voxel_down_sample`.  Synchronises once, to check the coordinates and
    the offsets."""
    points, offsets, n, F = _frames_args(points, offsets)
    counts = torch.empty(max(F, 1), max(F, 1), dtype=torch.int64, device=points.device)
    status = torch.zeros(1, dtype=torch.int32, device=points.device)
    with torch.cuda.device(points.device):
        wsb = lib.pcb_frame_overlap_ws_bytes(n, F)
        ws = workspace(wsb, points.device, slot=6)
        check(lib.pcb_frame_overlap(ptr(points), n, ptr(offsets), F, float(radius), ptr(counts), ptr(status), ptr(ws), wsb, stream()))
    bits = int(status.item())
    if bits & _lib.FRAMES_OFFSETS:
        raise _lib.PcbError("overlap_counts: offsets must run from 0 to N without decreasing")
    if bits & _lib.FRAMES_RANGE:
        raise _lib.PcbError("overlap_counts: a point lies outside +-2^20 cells of the radius or is not finite")
    return counts


def load_scene(input_path):
    """The frames of `<input_path>/*.npz` in sorted file order -> (names, frames): names as `os.path.join(input_path, file)`, frames
    fp64 [n, 3]; a frame holding a NaN (`:16-17`) or no point is dropped."""
    names, frames = [], []
    for name in sorted(glob.glob(os.path.join(input_path, "*.npz"))):
        xyz = np.asarray(np.load(name)["pcd"], np.float64).reshape(-1, 3)
        if len(xyz) and not np.isnan(xyz).any():
            names.append(name)
            frames.append(xyz)
    return names, frames


def scene_overlap(frames, voxel_size, device=None):
    """frames: fp64 [n_f, 3] arrays -> (overlap matrix M fp64 [F, F], M[i, j] = counts[i, j] / n_j of the downsampled frames; the
    downsampled frame sizes)."""
    F = len(frames)
    if F == 0:
        return np.zeros((0, 0)), np.zeros(0, np.int64)
    if F > MAX_FRAMES:
        raise _lib.PcbError(f"a scene holds at most {MAX_FRAMES} frames, got {F}")
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    sizes = np.array([len(f) for f in frames], np.int64)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)])).to(device)
    xyz = torch.from_numpy(np.concatenate(frames)).to(device)
    points, doff, host = voxel_down_sample(xyz, off, voxel_size)
    counts = overlap_counts(points, doff, 1.5 * voxel_size).cpu().numpy()
    n = np.diff(np.asarray(host, np.int64))
    return counts.astype(np.float64) / n.astype(np.float64)[None, :], n


def write_overlap(path, names, M):
    """`compute_full_overlapping.py:78-83`: "<name_i> <name_j> <max(M[i, j], M[j, i])>" for i < j."""
    with open(path, "w") as f:
        for i in range(len(names)):
            for j in range(i + 1, len(names)):
                f.write("{} {} {}\n".format(names[i], names[j], max(M[i, j], M[j, i])))


def compute_full_overlapping(input_path, voxel_size=0.05, device=None, scene=None):
    """`compute_full_overlapping.py` as a function: writes `<input_path>/overlap.txt` and returns (M, names).  `scene` = an already
    loaded `load_scene(input_path)`."""
    names, frames = scene if scene is not None else load_scene(input_path)
    M, _ = scene_overlap(frames, voxel_size, device)
    write_overlap(os.path.join(input_path, "overlap.txt"), names, M)
    return M, names


def generate_list(target_dir, threshold=0.3):
    """`generate_list.py:20-28`: the pairs of `<target_dir>/*/pcd/overlap.txt` (sorted) with overlap >= threshold ->
    `<target_dir>/overlap-30-full.txt`.  Returns its path."""
    out = os.path.join(target_dir, "overlap-30-full.txt")
    with open(out, "w") as f:
        for fo in sorted(glob.glob(os.path.join(target_dir, "*/pcd/overlap.txt"))):
            for line in open(fo):
                pcd0, pcd1, op = line.strip().split()
                if float(op) >= threshold:
                    print("{} {} {}".format(pcd0, pcd1, op), file=f)
    return out


def compute_scenes(input_paths, voxel_size=0.05, device=None, log=print):
    """`compute_full_overlapping` over several scenes back to back; a reader thread loads the next scene's npz files while the GPU
    works on the current one.  The thread has ended when this returns or raises."""
    input_paths = list(input_paths)
    q = queue.Queue(maxsize=1)
    stop = threading.Event()

    def put(item):
        while not stop.is_set():
            try:
                q.put(item, timeout=0.1)
                return True
            except queue.Full:
                pass
        return False

    def reader():
        for p in input_paths:
            try:
                scene, err = load_scene(p), None
            except Exception as e:                      # handed to the consumer, which raises it
                scene, err = None, e
            if not put((p, scene, err)) or err is not None:
                return

    t = threading.Thread(target=reader, daemon=True)
    t.start()
    try:
        for _ in input_paths:
            p, scene, err = q.get()
            if err is not None:
                raise err
            M, names = compute_full_overlapping(p, voxel_size, device, scene=scene)
            if log:
                log(f"{p}: {len(names)} frames, {len(names) * (len(names) - 1) // 2} pairs -> {os.path.join(p, 'overlap.txt')}")
    finally:
        stop.set()                                      # a reader waiting to hand over a scene gives up; one mid-load finishes it
        t.join()


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m pointcontrast_b200.pair_list", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    o = sub.add_parser("overlap", help="write <input_path>/overlap.txt for each scene")
    o.add_argument("--input_path", required=True, nargs="+", help="directories of a scene's <frame>.npz files")
    o.add_argument("--voxel_size", type=float, default=0.05)
    li = sub.add_parser("list", help="write <target_dir>/overlap-30-full.txt from <target_dir>/*/pcd/overlap.txt")
    li.add_argument("--target_dir", required=True)
    args = ap.parse_args(argv)
    if args.cmd == "overlap":
        compute_scenes(args.input_path, args.voxel_size)
    else:
        print(generate_list(args.target_dir))


if __name__ == "__main__":
    main()
