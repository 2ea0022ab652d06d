"""The pretraining pair list on the GPU (SURVEY.md 8f-10, 8f-11): from a raw ScanNet scan `<scene>.sens` to its frames, and from a
scene's frames `<scene>/pcd/<frame>.npz` (`pcd` = fp64 world points [N, 3]) to `<scene>/pcd/overlap.txt`, and from those to the list
`overlap-30-full.txt` that `scannet_pairs.ScanNetMatchPairDataset` reads -- the reference's `pretrain/data_preprocess/scannet_pair/compute_full_overlapping.py` and `generate_list.py`, which downsample
with open3d and make one KD-tree radius query per point for every ordered pair of frames.

    points, offsets, host = voxel_down_sample(xyz, offsets, 0.05)     # every frame of a scene in one call
    counts = overlap_counts(points, offsets, 0.075)                    # [F, F]: points of frame j with a neighbour in frame i
    compute_full_overlapping("scans/scene0000_00/pcd")                 # writes overlap.txt
    generate_list("scans")                                             # writes scans/overlap-30-full.txt

    scan = read_sens("scene0000_00.sens", frame_skip=25)             # header, kept frames' poses, intrinsics and inflated depth
    points, offsets, host, nan = depth_to_points(depth, scan.intrinsic, poses)    # depth uint16 [F, H, W], poses [F, 4, 4] on the device
    extract_scene("scene0000_00.sens", "scans/scene0000_00", 25)     # writes pcd/<frame>.npz and pcd/overlap.txt

    python -m pointcontrast_b200.pair_list extract --target_dir scans --frame_skip 25 raw/scene*/*.sens [--voxel_size 0.05]
    python -m pointcontrast_b200.pair_list overlap --input_path scans/scene0000_00/pcd [more scene paths ...] [--voxel_size 0.05]
    python -m pointcontrast_b200.pair_list list --target_dir scans

`extract` replaces the reference's `reader.py` + `point_cloud_extractor.py` + `compute_full_overlapping.py` (its README's per-scene
script): the depth is inflated on the host, back-projected and downsampled on the GPU chunk by chunk, and the overlap is computed from
the downsampled points still on the device, so no npz file is read back.

Deliberate differences from the reference (DESIGN.md section 5): frames are taken in sorted file order (the reference uses `glob`
order, which depends on the file system; the unordered pairs and their values are the same), and an empty frame is dropped with the
frames holding a NaN (the reference divides by its zero size).  `extract` writes a frame with one valid pixel as a one-point frame (the
reference's `.squeeze()` makes it a vector and raises), and its overlap covers only the frames it extracts (stale npz files in the
directory are ignored).
"""
import argparse
import contextlib
import ctypes
import dataclasses
import glob
import os
import queue
import struct
import threading
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib
from ._lib import check, lib, ptr, stream, workspace

MAX_FRAMES = 4096
EXTRACT_CHUNK = 32          # frames per device batch of `extract_scene` (each takes up to 7.4 MB of points at 640 x 480)
INFLATE_THREADS = 8         # zlib releases the GIL while it inflates
SENS_VERSION = 4
COMPRESSION_TYPE_COLOR = {-1: "unknown", 0: "raw", 1: "png", 2: "jpeg"}            # `SensorData.py:13-14`
COMPRESSION_TYPE_DEPTH = {-1: "unknown", 0: "raw_ushort", 1: "zlib_ushort", 2: "occi_ushort"}


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
        ws = workspace(wsb, xyz.device)
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
        ws = workspace(wsb, points.device)
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
    device = _device(device)
    sizes = np.array([len(f) for f in frames], np.int64)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)])).to(device)
    xyz = torch.from_numpy(np.concatenate(frames)).to(device)
    points, doff, host = voxel_down_sample(xyz, off, voxel_size)
    n = np.diff(np.asarray(host, np.int64))
    return _overlap_matrix(points, doff, n, voxel_size), n


def _device(device):
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def _overlap_matrix(points, offsets, sizes, voxel_size):
    """M[i, j] = counts[i, j] / n_j (`:74`) of downsampled frames (device points and offsets, host sizes n)."""
    counts = overlap_counts(points, offsets, 1.5 * voxel_size).cpu().numpy()
    return counts.astype(np.float64) / np.asarray(sizes, np.float64)[None, :]


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


@contextlib.contextmanager
def _read_ahead(paths, load):
    """Yields an iterator of (path, load(path)) over `paths`; a reader thread loads the next item while the caller works on the current
    one, and an error of `load` is raised when its item is reached.  The thread has ended when the `with` block is left."""
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
        for p in paths:
            try:
                item, err = load(p), None
            except Exception as e:                      # handed to the consumer, which raises it
                item, err = None, e
            if not put((p, item, err)) or err is not None:
                return

    def items():
        for _ in paths:
            p, item, err = q.get()
            if err is not None:
                raise err
            yield p, item

    t = threading.Thread(target=reader, daemon=True)
    t.start()
    try:
        yield items()
    finally:
        stop.set()                                      # a reader waiting to hand over an item gives up; one mid-load finishes it
        t.join()


def compute_scenes(input_paths, voxel_size=0.05, device=None, log=print):
    """`compute_full_overlapping` over several scenes back to back; a reader thread loads the next scene's npz files while the GPU
    works on the current one.  The thread has ended when this returns or raises."""
    input_paths = list(input_paths)
    with _read_ahead(input_paths, load_scene) as scenes:
        for p, scene in scenes:
            M, names = compute_full_overlapping(p, voxel_size, device, scene=scene)
            if log:
                log(f"{p}: {len(names)} frames, {len(names) * (len(names) - 1) // 2} pairs -> {os.path.join(p, 'overlap.txt')}")


@dataclasses.dataclass
class SensScan:
    """What `read_sens` keeps of a version-4 `.sens` file: the header as `SensorData.load` reads it (`SensorData.py:57-74`), the kept
    frames' indices and poses, and their inflated depth.  `poses` and `intrinsic` are the float32 values after the reference's text round
    trip (`text_round_trip`), the values `point_cloud_extractor.py` computes with."""
    sensor_name: bytes
    intrinsic_color: np.ndarray         # float32 [4, 4], as stored
    extrinsic_color: np.ndarray
    intrinsic_depth: np.ndarray
    extrinsic_depth: np.ndarray
    color_compression_type: str
    depth_compression_type: str
    color_width: int
    color_height: int
    depth_width: int
    depth_height: int
    depth_shift: float                  # read, not used: the reference back-projects with 1000
    num_frames: int
    frames: np.ndarray                  # int64 [K]: the kept frame indices f, f % frame_skip == 0
    camera_to_world: np.ndarray         # float32 [K, 4, 4], as stored
    poses: np.ndarray                   # fp64 [K, 4, 4]: text_round_trip(camera_to_world)
    intrinsic: np.ndarray               # fp64 [4, 4]: text_round_trip(intrinsic_depth)
    depth: np.ndarray                   # uint16 [K, depth_height, depth_width], millimetres


def text_round_trip(a):
    """float32 values -> fp64 as `SensorData.save_mat_to_file` (`np.savetxt(fmt='%f')`) and `np.loadtxt` leave them: float('%f' % x);
    -inf and nan survive it."""
    a = np.asarray(a, np.float32)
    return np.array([float("%f" % x) for x in a.ravel().tolist()], np.float64).reshape(a.shape)


def read_sens(path, frame_skip=1):
    """Parses a version-4 ScanNet `.sens` file (`SensorData.load`), keeping the frames f with f % frame_skip == 0 (`export_*`,
    `SensorData.py:86`).  Colour payloads and dropped frames are seeked past, not read; the kept depth is inflated with zlib on
    INFLATE_THREADS threads.  Raises ValueError for a version other than 4, a depth compression other than `zlib_ushort`, a truncated
    file and a frame whose depth does not inflate to 2 * width * height bytes.  Returns a SensScan."""
    if frame_skip < 1:
        raise ValueError(f"frame_skip must be at least 1, got {frame_skip}")
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        def take(n, what):
            b = f.read(n)
            if len(b) != n:
                raise ValueError(f"{path}: truncated .sens file: {what} needs {n} bytes at offset {f.tell() - len(b)}, "
                                 f"the file has {size}")
            return b

        def skip(n, what):
            if f.tell() + n > size:
                raise ValueError(f"{path}: truncated .sens file: {what} needs {n} bytes at offset {f.tell()}, the file has {size}")
            f.seek(n, os.SEEK_CUR)

        version, = struct.unpack("<I", take(4, "the version"))
        if version != SENS_VERSION:
            raise ValueError(f"{path}: .sens version {version}, only version {SENS_VERSION} is read")
        strlen, = struct.unpack("<Q", take(8, "the sensor name length"))
        sensor_name = take(strlen, "the sensor name")
        mats = np.frombuffer(take(256, "the calibration"), "<f4").reshape(4, 4, 4).astype(np.float32)
        cc, dc, cw, ch, dw, dh, shift, num_frames = struct.unpack("<iiIIIIfQ", take(36, "the image header"))
        if dc not in COMPRESSION_TYPE_DEPTH or cc not in COMPRESSION_TYPE_COLOR:
            raise ValueError(f"{path}: unknown compression type (colour {cc}, depth {dc})")
        if COMPRESSION_TYPE_DEPTH[dc] != "zlib_ushort":
            raise ValueError(f"{path}: depth compression {COMPRESSION_TYPE_DEPTH[dc]!r}, only 'zlib_ushort' is read")
        frames, c2w, blobs = [], [], []
        for i in range(num_frames):
            head = take(96, f"frame {i}'s header")
            color_bytes, depth_bytes = struct.unpack("<QQ", head[80:96])
            if i % frame_skip:
                skip(color_bytes + depth_bytes, f"frame {i}")
                continue
            skip(color_bytes, f"frame {i}'s colour")
            blobs.append(take(depth_bytes, f"frame {i}'s depth"))
            frames.append(i)
            c2w.append(np.frombuffer(head[:64], "<f4").reshape(4, 4))
    depth = np.empty((len(blobs), dh, dw), np.uint16)

    def inflate(k):
        try:
            raw = zlib.decompress(blobs[k])
        except zlib.error as e:
            raise ValueError(f"{path}: frame {frames[k]}'s depth does not inflate: {e}") from None
        if len(raw) != 2 * dw * dh:
            raise ValueError(f"{path}: frame {frames[k]}'s depth inflates to {len(raw)} bytes, not 2 * {dw} * {dh}")
        depth[k] = np.frombuffer(raw, "<u2").reshape(dh, dw)

    with ThreadPoolExecutor(INFLATE_THREADS) as ex:
        list(ex.map(inflate, range(len(blobs))))
    camera_to_world = np.array(c2w, np.float32).reshape(-1, 4, 4)
    return SensScan(sensor_name, mats[0].copy(), mats[1].copy(), mats[2].copy(), mats[3].copy(), COMPRESSION_TYPE_COLOR[cc],
                    COMPRESSION_TYPE_DEPTH[dc], cw, ch, dw, dh, shift, num_frames, np.array(frames, np.int64), camera_to_world,
                    text_round_trip(camera_to_world), text_round_trip(mats[2]), depth)


def depth_to_points(depth, intrinsic, poses):
    """`point_cloud_extractor.py:47-75` for a batch of frames on the device (pcb_depth_to_points).  depth: CUDA uint16 (or int16 with
    the same bits) [F, H, W] in millimetres; intrinsic: the 4 x 4 depth intrinsics (fx = K[0, 0], fy = K[1, 1], cx = K[0, 2],
    cy = K[1, 2], bx = K[0, 3], by = K[1, 3]); poses: fp64 [F, 4, 4] camera-to-world.  Returns (points fp64 CUDA [N, 3]: every pixel
    with nonzero depth, frame-major, row-major within a frame; offsets int64 CUDA [F + 1]; the offsets as a host list; a host list of F
    bools, True where the frame holds a NaN).  Synchronises once."""
    _lib.require_cuda(depth)
    if depth.dim() != 3 or depth.dtype not in (torch.uint16, torch.int16):
        raise _lib.PcbError(f"depth must be uint16 [F, H, W], got {depth.dtype} {tuple(depth.shape)}")
    F, H, W = depth.shape
    K = np.asarray(intrinsic, np.float64)
    poses = torch.as_tensor(poses, dtype=torch.float64).to(depth.device).contiguous()
    if K.shape != (4, 4) or tuple(poses.shape) != (F, 4, 4):
        raise _lib.PcbError(f"intrinsic must be [4, 4] and poses [{F}, 4, 4], got {K.shape} and {tuple(poses.shape)}")
    depth = depth.contiguous()
    out = torch.empty(max(F * H * W, 1), 3, dtype=torch.float64, device=depth.device)
    out_off = torch.empty(F + 1, dtype=torch.int64, device=depth.device)
    host = (ctypes.c_int64 * (F + 1))()
    nan = (ctypes.c_int32 * max(F, 1))()
    if F == 0:
        return out[:0], out_off.zero_(), [0], []
    with torch.cuda.device(depth.device):
        wsb = lib.pcb_depth_to_points_ws_bytes(F, H, W)
        ws = workspace(wsb, depth.device)
        check(lib.pcb_depth_to_points(ptr(depth), F, H, W, K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 3], K[1, 3], ptr(poses), ptr(out),
                                      ptr(out_off), host, nan, ptr(ws), wsb, stream()))
    return out[:host[F]], out_off, list(host), [bool(x) for x in nan[:F]]


class _NpzWriter:
    """Writes `np.savez(name, pcd=points)` on a thread, at most `depth` files queued; the first error is raised by `check`."""

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
                    np.savez(item[0], pcd=item[1])
                except BaseException as e:
                    self.err = e
                self.busy_s += time.perf_counter() - t

    def put(self, name, points):
        self.check()
        self.q.put((name, points))

    def close(self):
        self.q.put(None)
        self.t.join()

    def check(self):
        if self.err is not None:
            raise self.err


def extract_scene(sens_path, output_path, frame_skip, voxel_size=0.05, device=None, scan=None):
    """The reference's per-scene preprocessing (`reader.py --export_depth_images --export_poses --export_intrinsics`,
    `point_cloud_extractor.py --save_npz`, `compute_full_overlapping.py`) from the `.sens` file: writes `<output_path>/pcd/<f>.npz`
    (`pcd` = fp64 [n, 3] world points, f the frame index) for every kept frame and `<output_path>/pcd/overlap.txt`.

    Frames go to the device EXTRACT_CHUNK at a time through a pinned staging buffer; each chunk is back-projected, copied back for
    the npz files (written on a thread) and downsampled at once, so only the downsampled points stay on the device.  Frames that
    `load_scene` would drop (a NaN or no point) are left out of the overlap; its rows are ordered as `load_scene` orders the files.
    `scan` = an already read `read_sens(sens_path, frame_skip)`.  Raises before writing anything when more than MAX_FRAMES frames are
    kept.  Returns (M, names, seconds): the overlap matrix and frame names as `compute_full_overlapping` returns them, and the wall
    time of the device loop ("gpu", including the copies back), of the npz writes on the writer thread ("write", overlapping the
    loop) and of the overlap and its file ("overlap")."""
    scan = scan if scan is not None else read_sens(sens_path, frame_skip)
    K = len(scan.frames)
    if K > MAX_FRAMES:
        raise _lib.PcbError(f"{sens_path}: {K} frames kept at frame_skip {frame_skip}; a scene holds at most {MAX_FRAMES}")
    device = _device(device)
    pcd_dir = os.path.join(output_path, "pcd")
    os.makedirs(pcd_dir, exist_ok=True)
    names = [os.path.join(pcd_dir, f"{f}.npz") for f in scan.frames.tolist()]
    down, secs = {}, {}
    t0 = time.perf_counter()
    chunk = max(1, min(EXTRACT_CHUNK, K))
    writer = _NpzWriter(2 * chunk)
    try:
        if K:
            H, W = scan.depth.shape[1:]
            staging = torch.empty((chunk, H, W), dtype=torch.int16, pin_memory=True)
            poses = torch.from_numpy(scan.poses).to(device)
            for a in range(0, K, chunk):
                b = min(K, a + chunk)
                staging.numpy()[:b - a] = scan.depth[a:b].view(np.int16)
                pts, _, host, nan = depth_to_points(staging[:b - a].to(device, non_blocking=True), scan.intrinsic, poses[a:b])
                pts_host = pts.cpu().numpy()
                for k in range(b - a):
                    writer.put(names[a + k], pts_host[host[k]:host[k + 1]])
                keep = [k for k in range(b - a) if host[k + 1] > host[k] and not nan[k]]
                if keep:
                    sizes = [host[k + 1] - host[k] for k in keep]
                    xyz = torch.cat([pts[host[k]:host[k + 1]] for k in keep]) if len(keep) < b - a else pts
                    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=device)
                    dpts, _, dhost = voxel_down_sample(xyz, off, voxel_size)
                    dpts = dpts.clone()                 # the slice would hold the downsampler's raw-sized buffer
                    for i, k in enumerate(keep):
                        down[a + k] = dpts[dhost[i]:dhost[i + 1]]
        secs["gpu"] = time.perf_counter() - t0
    finally:
        writer.close()
    writer.check()
    secs["write"] = writer.busy_s
    t0 = time.perf_counter()
    rows = [k for k in sorted(range(K), key=names.__getitem__) if k in down]
    if rows:
        sizes = np.array([len(down[k]) for k in rows], np.int64)
        off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)])).to(device)
        M = _overlap_matrix(torch.cat([down[k] for k in rows]), off, sizes, voxel_size)
    else:
        M = np.zeros((0, 0))
    names = [names[k] for k in rows]
    write_overlap(os.path.join(pcd_dir, "overlap.txt"), names, M)
    secs["overlap"] = time.perf_counter() - t0
    return M, names, secs


def extract_scenes(paths, target_dir, frame_skip, voxel_size=0.05, device=None, log=print):
    """`extract_scene` over several `.sens` files back to back: scene `<target_dir>/<file name without its extension>`, as the
    reference's README names `$TARGET_DIR/$scene`.  A reader thread reads and inflates the next scan while the GPU works on the current
    one.  Every thread has ended when this returns or raises."""
    paths = list(paths)
    with _read_ahead(paths, lambda p: read_sens(p, frame_skip)) as scans:
        for p, scan in scans:
            out = os.path.join(target_dir, os.path.splitext(os.path.basename(p))[0])
            M, names, _ = extract_scene(p, out, frame_skip, voxel_size, device, scan=scan)
            if log:
                log(f"{p}: {len(scan.frames)} frames kept of {scan.num_frames}, {len(names)} in the overlap, "
                    f"{len(names) * (len(names) - 1) // 2} pairs -> {os.path.join(out, 'pcd')}")


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m pointcontrast_b200.pair_list", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    o = sub.add_parser("overlap", help="write <input_path>/overlap.txt for each scene")
    o.add_argument("--input_path", required=True, nargs="+", help="directories of a scene's <frame>.npz files")
    o.add_argument("--voxel_size", type=float, default=0.05)
    e = sub.add_parser("extract", help="write <target_dir>/<scene>/pcd/<frame>.npz and overlap.txt for each .sens file")
    e.add_argument("sens", nargs="+", help="ScanNet <scene>.sens files")
    e.add_argument("--target_dir", required=True)
    e.add_argument("--frame_skip", type=int, default=1)
    e.add_argument("--voxel_size", type=float, default=0.05)
    li = sub.add_parser("list", help="write <target_dir>/overlap-30-full.txt from <target_dir>/*/pcd/overlap.txt")
    li.add_argument("--target_dir", required=True)
    args = ap.parse_args(argv)
    if args.cmd == "extract":
        extract_scenes(args.sens, args.target_dir, args.frame_skip, args.voxel_size)
    elif args.cmd == "overlap":
        compute_scenes(args.input_path, args.voxel_size)
    else:
        print(generate_list(args.target_dir))


if __name__ == "__main__":
    main()
