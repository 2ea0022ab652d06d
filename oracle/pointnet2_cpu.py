"""numpy / torch-CPU restatement of the reference's PointNet++ `_ext` operators
(`downstream/votenet_det_new/models/backbone/pointnet2/_ext_src/src/*`), the checker of pointcontrast_b200/pointnet2.py.

Same names, argument order, shapes and dtypes as `_ext` (torch CPU tensors in and out).  Distances are computed in numpy float32, one
rounding per operation in the reference's operand order, so index results are bit-exact against an fp32 kernel without FMA contraction.
Forward gathers are fp32 copies / the fp32 three-term sum; the backward passes accumulate in fp64.

    oracle.pointnet2_cpu.install()      # `import pointnet2._ext` -> these functions (the reference's modules then run on the CPU)
"""
import sys
import types

import numpy as np
import torch

F32 = np.float32


def _d2(a, b):
    """((dx*dx + dy*dy) + dz*dz) in float32 with dx = a - b; a [..., 3], b broadcastable."""
    d = (a - b).astype(F32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def furthest_point_sampling(points, nsamples):
    """`sampling_gpu.cu:74-178` + `sampling.cpp:71-92`: idx[0] = 0; the running min-distance starts at 1e10 (`sampling.cpp:80`); points with
    x^2 + y^2 + z^2 <= 1e-3 (float against the double literal) are never candidates; d = ((dx dx + dy dy) + dz dz) with dx = p_k - p_sel;
    the next pick is the candidate of largest running distance, the SMALLEST index among exact ties (the reference's tie winner
    depends on its block size), and index 0 when there is no candidate."""
    xyz = points.detach().cpu().numpy().astype(F32)
    B, N, _ = xyz.shape
    out = np.zeros((B, int(nsamples)), dtype=np.int32)
    for b in range(B):
        p = xyz[b]
        mag = (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]
        cand = ~(mag.astype(np.float64) <= 1e-3)
        temp = np.full(N, 1e10, dtype=F32)
        old = 0
        for j in range(1, int(nsamples)):
            d = _d2(p, p[old])
            temp = np.where(cand, np.minimum(d, temp), temp)
            score = np.where(cand, temp, F32(-1))
            old = int(np.argmax(score))              # first maximum: smallest index; all -1 (no candidate): 0
            out[b, j] = old
    return torch.from_numpy(out)


def ball_query(new_xyz, xyz, radius, nsample):
    """`ball_query_gpu.cu:14-49` + `ball_query.cpp:24-26`: the first nsample k in ascending order with d < radius * radius (fp32, strict,
    d from new - p); the remaining slots repeat the first hit; no hit: the row stays zero."""
    q = new_xyz.detach().cpu().numpy().astype(F32)
    p = xyz.detach().cpu().numpy().astype(F32)
    B, M, _ = q.shape
    S = int(nsample)
    r2 = F32(radius) * F32(radius)
    out = np.zeros((B, M, S), dtype=np.int32)
    for b in range(B):
        for m0 in range(0, M, 128):
            hit = _d2(q[b, m0:m0 + 128, None, :], p[b][None]) < r2
            pos = np.cumsum(hit, axis=1)
            rows, ks = np.nonzero(hit & (pos <= S))
            slot = pos[rows, ks] - 1
            blk = out[b, m0:m0 + 128]
            first = np.where(hit.any(1), hit.argmax(1), 0)
            blk[:] = first[:, None]
            blk[rows, slot] = ks
    return torch.from_numpy(out)


def three_nn(unknowns, knows):
    """`interpolate_gpu.cu:14-64`: the three smallest d = ((dx dx + dy dy) + dz dz), dx = u - k, by sequential insertion with strict <
    (ties keep the earlier k == a stable sort); squared distances; with m < 3 the missing entries are float(1e40) = inf, index 0."""
    u = unknowns.detach().cpu().numpy().astype(F32)
    k = knows.detach().cpu().numpy().astype(F32)
    B, n, _ = u.shape
    m = k.shape[1]
    dist2 = np.full((B, n, 3), np.inf, dtype=F32)
    idx = np.zeros((B, n, 3), dtype=np.int32)
    t = min(3, m)
    for b in range(B):
        for j0 in range(0, n, 256):
            d = _d2(u[b, j0:j0 + 256, None, :], k[b][None])
            o = np.argsort(d, axis=1, kind="stable")[:, :t]
            dist2[b, j0:j0 + 256, :t] = np.take_along_axis(d, o, 1)
            idx[b, j0:j0 + 256, :t] = o
    return [torch.from_numpy(dist2), torch.from_numpy(idx)]


def gather_points(points, idx):
    """`sampling_gpu.cu:13-25`: out[b, c, j] = points[b, c, idx[b, j]]."""
    return torch.gather(points, 2, idx.long().unsqueeze(1).expand(-1, points.shape[1], -1))


def group_points(points, idx):
    """`group_points_gpu.cu:13-33`: out[b, c, m, s] = points[b, c, idx[b, m, s]]."""
    B, M, S = idx.shape
    return gather_points(points, idx.reshape(B, M * S)).reshape(B, points.shape[1], M, S)


def three_interpolate(points, idx, weight):
    """`interpolate_gpu.cu:77-106`: (f1 w1 + f2 w2) + f3 w3, in the features' dtype (fp32: one rounding per operation)."""
    f = points.detach().cpu().numpy()
    i = idx.cpu().numpy().astype(np.int64)
    w = weight.detach().cpu().numpy().astype(f.dtype)
    g = np.stack([np.take_along_axis(f, np.broadcast_to(i[:, None, :, t], (f.shape[0], f.shape[1], i.shape[1])), 2) for t in range(3)])
    ww = w.transpose(2, 0, 1)[:, :, None, :]
    return torch.from_numpy((g[0] * ww[0] + g[1] * ww[1]) + g[2] * ww[2])


def _scatter(vals, idx, n):
    """out[b, c, a] = sum of vals[b, c, p] over p with idx[b, p] == a, in fp64; vals [B, C, L], idx [B, L]."""
    v = np.asarray(vals, dtype=np.float64)
    B, C, L = v.shape
    out = np.zeros((B, C, int(n)), dtype=np.float64)
    for b in range(B):
        np.add.at(out[b].T, idx[b], v[b].T)
    return out


def gather_points_grad(grad_out, idx, n, absolute=False):
    """Adjoint of gather_points (`sampling_gpu.cu:39-52`), fp64; absolute=True sums |terms| (the scale of the rounding error)."""
    g = grad_out.detach().cpu().double().numpy()
    return torch.from_numpy(_scatter(np.abs(g) if absolute else g, idx.cpu().numpy().astype(np.int64), n))


def group_points_grad(grad_out, idx, n, absolute=False):
    """Adjoint of group_points (`group_points_gpu.cu:48-69`), fp64."""
    B, C, M, S = grad_out.shape
    return gather_points_grad(grad_out.reshape(B, C, M * S), idx.reshape(B, M * S), n, absolute)


def three_interpolate_grad(grad_out, idx, weight, m, absolute=False):
    """Adjoint of three_interpolate (`interpolate_gpu.cu:121-148`): grad_out[b, c, j] * w[b, j, t] scattered to idx[b, j, t], fp64."""
    g = grad_out.detach().cpu().double().numpy()
    w = weight.detach().cpu().double().numpy()
    B, C, n = g.shape
    terms = (g[:, :, :, None] * w[:, None, :, :]).reshape(B, C, 3 * n)
    return torch.from_numpy(_scatter(np.abs(terms) if absolute else terms, idx.cpu().numpy().astype(np.int64).reshape(B, 3 * n), m))


EXT_FUNCTIONS = ("gather_points", "gather_points_grad", "furthest_point_sampling", "three_nn", "three_interpolate", "three_interpolate_grad",
                 "ball_query", "group_points", "group_points_grad")


def _dtype_preserving(f):
    """The reference's modules call the backward functions on whatever dtype autograd hands them (fp64 in the drop-in comparison)."""
    def g(*a):
        ref = next(x for x in a if torch.is_tensor(x) and x.is_floating_point())
        r = f(*a)
        return [x.to(ref.dtype) if x.is_floating_point() else x for x in r] if isinstance(r, list) else (r.to(ref.dtype) if r.is_floating_point() else r)
    return g


def install(name="pointnet2"):
    """Register `name._ext` = these functions (CPU tensors), so the reference's unmodified pointnet2_utils.py runs on the oracle."""
    ext = types.ModuleType(name + "._ext")
    for f in EXT_FUNCTIONS:
        setattr(ext, f, _dtype_preserving(globals()[f]) if f not in ("furthest_point_sampling", "ball_query", "three_nn") else globals()[f])
    pkg = types.ModuleType(name)
    pkg.__path__ = []
    pkg._ext = ext
    sys.modules[name] = pkg
    sys.modules[name + "._ext"] = ext
    return ext
