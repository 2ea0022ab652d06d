"""PointNet++ operators of the VoteNet detection downstream on libpcb200 (DESIGN.md 8f-5): furthest-point sampling, ball query,
grouping, three-NN interpolation and their backward passes, in place of the reference's separately built torch extension
(`downstream/votenet_det_new/models/backbone/pointnet2/_ext_src`).

    from pointcontrast_b200 import pointnet2
    pointnet2.install()          # `import pointnet2._ext` now resolves here: the reference's pointnet2_utils / pointnet2_modules run unmodified

The nine `_ext` functions keep the reference's names, argument order, shapes and dtypes (xyz fp32 [B, N, 3], features fp32 [B, C, N],
indices int32).  They run on torch's current stream and reject CPU tensors, wrong dtypes and non-contiguous inputs.  Index results are
bit-exact against the reference's arithmetic; furthest-point sampling breaks exact distance ties towards the smallest index; the
backward passes are deterministic (DESIGN.md "Numerics").
"""
import sys
import types

import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib
from ._lib import PcbError, check, lib, ptr, stream, workspace


def _check(t, dtype, name, device=None):
    _lib.require_cuda(t)
    if t.dtype != dtype:
        raise PcbError(f"{name} must be a {dtype} tensor, got {t.dtype}")
    if not t.is_contiguous():
        raise PcbError(f"{name} must be a contiguous tensor")
    if device is not None and t.device != device:
        raise PcbError(f"{name} is on {t.device}, expected {device}")


def _dims(t, n, name, batch=None, last=None):
    if t.dim() != n or (batch is not None and t.shape[0] != batch) or (last is not None and t.shape[-1] != last):
        raise PcbError(f"{name} has shape {tuple(t.shape)}: expected {n} dimensions" + (f", batch {batch}" if batch is not None else "")
                       + (f", last dimension {last}" if last is not None else ""))


# ------------------------------------------------------------------------------------------------ the `_ext` functions
def furthest_point_sampling(points, nsamples):
    """points fp32 [B, N, 3] -> int32 [B, nsamples]."""
    _check(points, torch.float32, "points"); _dims(points, 3, "points", last=3)
    B, N, _ = points.shape
    out = torch.empty(B, int(nsamples), dtype=torch.int32, device=points.device)
    with torch.cuda.device(points.device):
        wsb = lib.pcb_furthest_point_sampling_ws_bytes(B, N)
        ws = workspace(wsb, points.device) if wsb else None
        check(lib.pcb_furthest_point_sampling(ptr(points), B, N, int(nsamples), ptr(out), ptr(ws), wsb, stream()))
    return out


def furthest_point_sampling_ragged(points, offsets, max_n, nsamples):
    """points fp32 [M, 3] grouped by scene, offsets int64 [B + 1] on the same device (scene b is rows [offsets[b], offsets[b+1])),
    max_n an upper bound on every scene's size -> int32 [B, nsamples] of scene-local indices: for every scene what
    `furthest_point_sampling` returns for that scene alone, all scenes in one launch."""
    _check(points, torch.float32, "points"); _check(offsets, torch.int64, "offsets", points.device)
    _dims(points, 2, "points", last=3); _dims(offsets, 1, "offsets")
    M, B = points.shape[0], offsets.shape[0] - 1
    out = torch.empty(B, int(nsamples), dtype=torch.int32, device=points.device)
    with torch.cuda.device(points.device):
        wsb = lib.pcb_furthest_point_sampling_ragged_ws_bytes(B, M, int(max_n))
        ws = workspace(wsb, points.device) if wsb else None
        check(lib.pcb_furthest_point_sampling_ragged(ptr(points), ptr(offsets), B, M, int(max_n), int(nsamples), ptr(out), ptr(ws), wsb,
                                                     stream()))
    return out


def gather_rows_grad(grad_out, idx, m):
    """Adjoint of rows[idx] for rows [m, C]: grad_out fp32 [L, C], idx int32 [L] -> [m, C], each row the sum of its readers'
    gradients in ascending reader order (fp64, deterministic)."""
    _check(grad_out, torch.float32, "grad_out"); _check(idx, torch.int32, "idx", grad_out.device)
    _dims(grad_out, 2, "grad_out"); _dims(idx, 1, "idx")
    L, C = grad_out.shape
    if idx.shape[0] != L:
        raise PcbError(f"idx has {idx.shape[0]} entries, grad_out {L} rows")
    out = torch.empty(int(m), C, dtype=torch.float32, device=grad_out.device)
    with torch.cuda.device(grad_out.device):
        wsb = lib.pcb_points_grad_ws_bytes(1, int(m), L)
        ws = workspace(wsb, grad_out.device)
        check(lib.pcb_gather_rows_grad(ptr(grad_out), ptr(idx), L, C, int(m), ptr(out), ptr(ws), wsb, stream()))
    return out


def gather_points(points, idx):
    """points fp32 [B, C, N], idx int32 [B, M] -> [B, C, M]."""
    _check(points, torch.float32, "points"); _check(idx, torch.int32, "idx", points.device)
    _dims(points, 3, "points"); _dims(idx, 2, "idx", batch=points.shape[0])
    B, C, N = points.shape
    out = torch.empty(B, C, idx.shape[1], dtype=torch.float32, device=points.device)
    with torch.cuda.device(points.device):
        check(lib.pcb_gather_points(ptr(points), ptr(idx), B, C, N, idx.shape[1], ptr(out), stream()))
    return out


def _points_grad(grad_out, idx, weight, B, C, n_src, L):
    out = torch.empty(B, C, int(n_src), dtype=torch.float32, device=grad_out.device)
    with torch.cuda.device(grad_out.device):
        wsb = lib.pcb_points_grad_ws_bytes(B, int(n_src), L)
        ws = workspace(wsb, grad_out.device)
        if weight is None:
            check(lib.pcb_gather_points_grad(ptr(grad_out), ptr(idx), B, C, int(n_src), L, ptr(out), ptr(ws), wsb, stream()))
        else:
            check(lib.pcb_three_interpolate_grad(ptr(grad_out), ptr(idx), ptr(weight), B, C, L // 3, int(n_src), ptr(out), ptr(ws), wsb,
                                                 stream()))
    return out


def gather_points_grad(grad_out, idx, n):
    """grad_out fp32 [B, C, M], idx int32 [B, M] -> [B, C, n]."""
    _check(grad_out, torch.float32, "grad_out"); _check(idx, torch.int32, "idx", grad_out.device)
    _dims(grad_out, 3, "grad_out"); _dims(idx, 2, "idx")
    B, C, M = grad_out.shape
    if tuple(idx.shape) != (B, M):
        raise PcbError(f"idx shape {tuple(idx.shape)} does not match grad_out {tuple(grad_out.shape)}")
    return _points_grad(grad_out, idx, None, B, C, n, M)


def three_nn(unknowns, knows):
    """unknowns fp32 [B, n, 3], knows fp32 [B, m, 3] -> [dist2 fp32 [B, n, 3], idx int32 [B, n, 3]]."""
    _check(unknowns, torch.float32, "unknowns"); _check(knows, torch.float32, "knows", unknowns.device)
    _dims(unknowns, 3, "unknowns", last=3); _dims(knows, 3, "knows", batch=unknowns.shape[0], last=3)
    B, n, _ = unknowns.shape
    dist2 = torch.empty(B, n, 3, dtype=torch.float32, device=unknowns.device)
    idx = torch.empty(B, n, 3, dtype=torch.int32, device=unknowns.device)
    with torch.cuda.device(unknowns.device):
        check(lib.pcb_three_nn(ptr(unknowns), ptr(knows), B, n, knows.shape[1], ptr(dist2), ptr(idx), stream()))
    return [dist2, idx]


def three_interpolate(points, idx, weight):
    """points fp32 [B, C, m], idx int32 [B, n, 3], weight fp32 [B, n, 3] -> [B, C, n]."""
    _check(points, torch.float32, "points"); _check(idx, torch.int32, "idx", points.device)
    _check(weight, torch.float32, "weight", points.device)
    _dims(points, 3, "points"); _dims(idx, 3, "idx", batch=points.shape[0], last=3)
    B, C, m = points.shape
    n = idx.shape[1]
    if tuple(weight.shape) != tuple(idx.shape):
        raise PcbError("weight and idx must have the same shape")
    out = torch.empty(B, C, n, dtype=torch.float32, device=points.device)
    with torch.cuda.device(points.device):
        check(lib.pcb_three_interpolate(ptr(points), ptr(idx), ptr(weight), B, C, m, n, ptr(out), stream()))
    return out


def three_interpolate_grad(grad_out, idx, weight, m):
    """grad_out fp32 [B, C, n], idx int32 / weight fp32 [B, n, 3] -> [B, C, m]."""
    _check(grad_out, torch.float32, "grad_out"); _check(idx, torch.int32, "idx", grad_out.device)
    _check(weight, torch.float32, "weight", grad_out.device)
    _dims(grad_out, 3, "grad_out")
    B, C, n = grad_out.shape
    if tuple(idx.shape) != (B, n, 3) or tuple(weight.shape) != (B, n, 3):
        raise PcbError("idx and weight must be [B, n, 3] matching grad_out [B, C, n]")
    return _points_grad(grad_out, idx, weight, B, C, m, 3 * n)


def ball_query(new_xyz, xyz, radius, nsample):
    """new_xyz fp32 [B, M, 3], xyz fp32 [B, N, 3] -> int32 [B, M, nsample]."""
    _check(new_xyz, torch.float32, "new_xyz"); _check(xyz, torch.float32, "xyz", new_xyz.device)
    _dims(new_xyz, 3, "new_xyz", last=3); _dims(xyz, 3, "xyz", batch=new_xyz.shape[0], last=3)
    B, M, _ = new_xyz.shape
    out = torch.empty(B, M, int(nsample), dtype=torch.int32, device=new_xyz.device)
    with torch.cuda.device(new_xyz.device):
        check(lib.pcb_ball_query(ptr(new_xyz), ptr(xyz), B, M, xyz.shape[1], float(radius), int(nsample), ptr(out), stream()))
    return out


def group_points(points, idx):
    """points fp32 [B, C, N], idx int32 [B, M, S] -> [B, C, M, S]."""
    _check(points, torch.float32, "points"); _check(idx, torch.int32, "idx", points.device)
    _dims(points, 3, "points"); _dims(idx, 3, "idx", batch=points.shape[0])
    B, C, N = points.shape
    _, M, S = idx.shape
    out = torch.empty(B, C, M, S, dtype=torch.float32, device=points.device)
    with torch.cuda.device(points.device):
        check(lib.pcb_gather_points(ptr(points), ptr(idx), B, C, N, M * S, ptr(out), stream()))
    return out


def group_points_grad(grad_out, idx, n):
    """grad_out fp32 [B, C, M, S], idx int32 [B, M, S] -> [B, C, n]."""
    _check(grad_out, torch.float32, "grad_out"); _check(idx, torch.int32, "idx", grad_out.device)
    _dims(grad_out, 4, "grad_out")
    B, C, M, S = grad_out.shape
    if tuple(idx.shape) != (B, M, S):
        raise PcbError(f"idx shape {tuple(idx.shape)} does not match grad_out {tuple(grad_out.shape)}")
    return _points_grad(grad_out, idx, None, B, C, n, M * S)


EXT_FUNCTIONS = ("gather_points", "gather_points_grad", "furthest_point_sampling", "three_nn", "three_interpolate", "three_interpolate_grad",
                 "ball_query", "group_points", "group_points_grad")
# The `_ext` surface as one namespace: below, `three_nn`, `three_interpolate` and `ball_query` become the autograd-level functions of
# pointnet2_utils (same names, different signatures), so the layer above calls the native functions through `ext`.
ext = types.ModuleType("pointnet2._ext")
for _f in EXT_FUNCTIONS:
    setattr(ext, _f, globals()[_f])


# ------------------------------------------------------------------------------------------------ autograd layer (pointnet2_utils)
class FurthestPointSampling(Function):
    @staticmethod
    def forward(ctx, xyz, npoint):
        """xyz [B, N, 3] -> int32 [B, npoint] indices of the furthest-point sample."""
        inds = ext.furthest_point_sampling(xyz, npoint)
        ctx.mark_non_differentiable(inds)
        return inds

    @staticmethod
    def backward(ctx, *grads):
        return None, None


class GatherOperation(Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features [B, C, N], idx [B, npoint] -> [B, C, npoint]."""
        ctx.save_for_backward(idx)
        ctx.n = features.shape[2]
        return ext.gather_points(features, idx)

    @staticmethod
    def backward(ctx, grad_out):
        idx, = ctx.saved_tensors
        return ext.gather_points_grad(grad_out.contiguous(), idx, ctx.n), None


class ThreeNN(Function):
    @staticmethod
    def forward(ctx, unknown, known):
        """unknown [B, n, 3], known [B, m, 3] -> (Euclidean distances [B, n, 3], int32 indices [B, n, 3]) of the three nearest known points."""
        dist2, idx = ext.three_nn(unknown, known)
        ctx.mark_non_differentiable(idx)
        return torch.sqrt(dist2), idx

    @staticmethod
    def backward(ctx, *grads):
        return None, None


class ThreeInterpolate(Function):
    @staticmethod
    def forward(ctx, features, idx, weight):
        """features [B, C, m], idx / weight [B, n, 3] -> [B, C, n] weighted sum of the three indexed features."""
        ctx.save_for_backward(idx, weight)
        ctx.m = features.shape[2]
        return ext.three_interpolate(features, idx, weight)

    @staticmethod
    def backward(ctx, grad_out):
        idx, weight = ctx.saved_tensors
        return ext.three_interpolate_grad(grad_out.contiguous(), idx, weight, ctx.m), None, None


class GroupingOperation(Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features [B, C, N], idx [B, npoint, nsample] -> [B, C, npoint, nsample]."""
        ctx.save_for_backward(idx)
        ctx.n = features.shape[2]
        return ext.group_points(features, idx)

    @staticmethod
    def backward(ctx, grad_out):
        idx, = ctx.saved_tensors
        return ext.group_points_grad(grad_out.contiguous(), idx, ctx.n), None


class BallQuery(Function):
    @staticmethod
    def forward(ctx, radius, nsample, xyz, new_xyz):
        """xyz [B, N, 3], centres new_xyz [B, npoint, 3] -> int32 [B, npoint, nsample] indices of the points in each ball."""
        inds = ext.ball_query(new_xyz, xyz, radius, nsample)
        ctx.mark_non_differentiable(inds)
        return inds

    @staticmethod
    def backward(ctx, *grads):
        return None, None, None, None


furthest_point_sample = FurthestPointSampling.apply
gather_operation = GatherOperation.apply
three_nn = ThreeNN.apply
three_interpolate = ThreeInterpolate.apply
grouping_operation = GroupingOperation.apply
ball_query = BallQuery.apply


class QueryAndGroup(nn.Module):
    """Ball query of `radius` around each centre, then the grouped (relative, optionally radius-normalised) xyz and features:
    forward(xyz [B, N, 3], new_xyz [B, npoint, 3], features [B, C, N] or None) -> [B, 3 + C, npoint, nsample]
    (plus grouped_xyz and / or the unique-neighbour count when asked for)."""

    def __init__(self, radius, nsample, use_xyz=True, ret_grouped_xyz=False, normalize_xyz=False, sample_uniformly=False, ret_unique_cnt=False):
        super().__init__()
        if ret_unique_cnt and not sample_uniformly:
            raise ValueError("ret_unique_cnt needs sample_uniformly")
        self.radius, self.nsample, self.use_xyz = radius, nsample, use_xyz
        self.ret_grouped_xyz, self.normalize_xyz = ret_grouped_xyz, normalize_xyz
        self.sample_uniformly, self.ret_unique_cnt = sample_uniformly, ret_unique_cnt

    def _resample_uniformly(self, idx):
        """Each ball keeps its distinct neighbours and refills the remaining slots with uniform draws among them."""
        cnt = torch.zeros(idx.shape[0], idx.shape[1])
        for b in range(idx.shape[0]):
            for r in range(idx.shape[1]):
                uniq = torch.unique(idx[b, r])
                cnt[b, r] = uniq.numel()
                extra = uniq[torch.randint(0, uniq.numel(), (self.nsample - uniq.numel(),), dtype=torch.long).to(uniq.device)]
                idx[b, r] = torch.cat((uniq, extra))
        return cnt

    def forward(self, xyz, new_xyz, features=None):
        idx = ball_query(self.radius, self.nsample, xyz, new_xyz)
        cnt = self._resample_uniformly(idx) if self.sample_uniformly else None
        grouped_xyz = grouping_operation(xyz.transpose(1, 2).contiguous(), idx) - new_xyz.transpose(1, 2).unsqueeze(-1)
        if self.normalize_xyz:
            grouped_xyz = grouped_xyz / self.radius
        if features is not None:
            grouped = grouping_operation(features, idx)
            new_features = torch.cat([grouped_xyz, grouped], dim=1) if self.use_xyz else grouped
        else:
            if not self.use_xyz:
                raise ValueError("QueryAndGroup without features needs use_xyz=True")
            new_features = grouped_xyz
        ret = [new_features] + ([grouped_xyz] if self.ret_grouped_xyz else []) + ([cnt] if self.ret_unique_cnt else [])
        return ret[0] if len(ret) == 1 else tuple(ret)


class GroupAll(nn.Module):
    """One group holding every point: forward(xyz [B, N, 3], new_xyz (ignored), features [B, C, N] or None) -> [B, 3 + C, 1, N]."""

    def __init__(self, use_xyz=True, ret_grouped_xyz=False):
        super().__init__()
        self.use_xyz, self.ret_grouped_xyz = use_xyz, ret_grouped_xyz

    def forward(self, xyz, new_xyz, features=None):
        grouped_xyz = xyz.transpose(1, 2).unsqueeze(2)
        if features is not None:
            grouped = features.unsqueeze(2)
            new_features = torch.cat([grouped_xyz, grouped], dim=1) if self.use_xyz else grouped
        else:
            new_features = grouped_xyz
        return (new_features, grouped_xyz) if self.ret_grouped_xyz else new_features


def install(name="pointnet2"):
    """Register `name` and `name._ext` (the nine functions above) in sys.modules, so that `import pointnet2._ext as _ext` -- the one
    native import of the reference's pointnet2_utils.py -- resolves to this library.  Returns the `_ext` module."""
    ext.__name__ = name + "._ext"
    pkg = types.ModuleType(name)
    pkg.__path__ = []
    pkg._ext = ext
    sys.modules[name] = pkg
    sys.modules[name + "._ext"] = ext
    return ext
