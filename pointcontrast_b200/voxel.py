"""GPU voxelisation and correspondence search (SURVEY.md 8f-2): the per-sample work of the reference's ScanNet-pair loader
(`pretrain/pointcontrast/lib/ddp_data_loaders.py:196-265`), which the reference does on CPU workers with
`ME.utils.sparse_quantize` and one open3d KD-tree radius query per point (`:36-49`, seconds per pair).

    coords, sel = voxelize(xyz, voxel_size)          # one point per voxel: floor(xyz / voxel_size), first point of each voxel
    pairs = radius_pairs(src, dst, radius)           # all (i, j) with |src_i - dst_j| < radius

`make_pair` assembles one sample of the loader's output from two raw point clouds and the ground-truth transform.
"""
import ctypes

import torch

from . import _lib
from ._lib import check, lib, ptr, stream, workspace


def voxelize(xyz, voxel_size):
    """xyz: float32 CUDA [N,3].  Returns (coords int32 [M,3] sorted by (x,y,z), sel int64 [M]: the first point of each voxel)."""
    _lib.require_cuda(xyz)
    xyz = xyz.contiguous().float()
    n = xyz.shape[0]
    coords = torch.empty(n, 3, dtype=torch.int32, device=xyz.device)
    sel = torch.empty(n, dtype=torch.int32, device=xyz.device)
    m = ctypes.c_int64(0)
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_voxelize_ws_bytes(n)
        ws = workspace(wsb, xyz.device)
        check(lib.pcb_voxelize(ptr(xyz), n, float(voxel_size), ptr(coords), ptr(sel), ctypes.byref(m), ptr(ws), wsb, stream()))
    return coords[:m.value], sel[:m.value].long()


def voxelize_scenes(xyz, voxel_size):
    """xyz: float32 CUDA [B,N,3], one scene per row.  Returns (coords int32 [M,4] = (b, x, y, z), inds int32 [M]: the scene-local
    index of each voxel's first point, offsets int64 [B+1] on the device, offsets as a host list).  Rows are scene-major and, within a
    scene, in ascending `inds`.  Synchronises once."""
    _lib.require_cuda(xyz)
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise _lib.PcbError(f"xyz must be [B, N, 3], got {tuple(xyz.shape)}")
    xyz = xyz.contiguous().float()
    B, N, _ = xyz.shape
    coords = torch.empty(B * N, 4, dtype=torch.int32, device=xyz.device)
    inds = torch.empty(B * N, dtype=torch.int32, device=xyz.device)
    offsets = torch.empty(B + 1, dtype=torch.int64, device=xyz.device)
    host = (ctypes.c_int64 * (B + 1))()
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_voxelize_scenes_ws_bytes(B, N)
        ws = workspace(wsb, xyz.device)
        check(lib.pcb_voxelize_scenes(ptr(xyz), B, N, float(voxel_size), ptr(coords), ptr(inds), ptr(offsets), host, ptr(ws), wsb, stream()))
    m = host[B]
    return coords[:m], inds[:m], offsets, list(host)


def radius_pairs(src, dst, radius):
    """src [Ns,3], dst [Nd,3] float32 CUDA.  Returns int32 [P,2]: every (i, j) with |src_i - dst_j| < radius, sorted by (i, j)."""
    _lib.require_cuda(src); _lib.require_cuda(dst)
    src, dst = src.contiguous().float(), dst.contiguous().float()
    ns, nd = src.shape[0], dst.shape[0]
    total = ctypes.c_int64(0)
    with torch.cuda.device(src.device):
        wsb = lib.pcb_radius_pairs_ws_bytes(ns, nd)
        ws = workspace(wsb, src.device)
        cap = max(4 * ns, 1024)                                     # usually enough for one pass (about 1-3 matches per point)
        pairs = torch.empty(cap, 2, dtype=torch.int32, device=src.device)
        check(lib.pcb_radius_pairs(ptr(src), ns, ptr(dst), nd, float(radius), ptr(pairs), cap, ctypes.byref(total), ptr(ws), wsb, stream()))
        if total.value > cap:
            cap = total.value
            pairs = torch.empty(cap, 2, dtype=torch.int32, device=src.device)
            check(lib.pcb_radius_pairs(ptr(src), ns, ptr(dst), nd, float(radius), ptr(pairs), cap, ctypes.byref(total), ptr(ws), wsb, stream()))
    return pairs[:total.value]


def make_pair(xyz0, xyz1, T_gt, voxel_size, search_mult=1.5):
    """One sample of `ddp_data_loaders.py:196-265` on the GPU: voxelise both clouds (`:228-241`), match view 0 (moved by the
    ground-truth transform `T_gt` [4,4]) against view 1 within `search_mult * voxel_size` (`:242-245`), integer coordinates
    `floor(xyz / voxel_size)` (`:258-259`).  Returns a dict with coords0/1 (int32 [N,3]), xyz0/1 (the kept points), corr [P,2]."""
    c0, s0 = voxelize(xyz0, voxel_size)
    c1, s1 = voxelize(xyz1, voxel_size)
    p0, p1 = xyz0[s0].float(), xyz1[s1].float()
    T = torch.as_tensor(T_gt, dtype=torch.float32, device=p0.device)
    moved = p0 @ T[:3, :3].T + T[:3, 3]
    corr = radius_pairs(moved, p1, search_mult * voxel_size)
    return {"coords0": c0, "coords1": c1, "xyz0": p0, "xyz1": p1, "corr": corr}
