"""CPU oracle of the `.sens` -> frame stage (pointcontrast_b200.pair_list.depth_to_points / extract_scene), restating the reference's
`pretrain/data_preprocess/scannet_pair/point_cloud_extractor.py:47-75` and the text files `reader.py` writes in numpy:

    text_round_trip(a)                           `SensorData.save_mat_to_file` (`np.savetxt(fmt='%f')`) read back by `np.loadtxt`
    depth_to_points(depth, intrinsic, pose)      one frame's world points, elementwise in a fixed order
    dot_bound(depth, intrinsic, pose)            how far the reference's BLAS product may lie from that order

The reference ends with `np.dot(points, pose.T)`, a BLAS product whose summation order and FMA use are not specified.  This
restatement fixes the order, w_r = ((X P[r,0] + Y P[r,1]) + Z P[r,2]) + P[r,3], one rounding per operation (numpy does not contract to
FMA), so the GPU kernel is held to it bit for bit.  Both this order and any BLAS order or FMA use compute the 4-term dot product with
an error of at most gamma_4 = 4u / (1 - 4u) (u = 2^-53) times sum_c |x_c P[r,c]| (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., (3.5)); so the two lie within twice that of each other.  Everything before the product (d, X, Y) is the
reference's own elementwise expression and is exact against it.
"""
import io

import numpy as np

U = 2.0 ** -53
GAMMA4 = 4 * U / (1 - 4 * U)


def text_round_trip(a):
    """float32 [..., 4] -> fp64: each row through `np.savetxt(f, row[np.newaxis], fmt='%f')` and `np.loadtxt` of the file."""
    a = np.asarray(a, np.float32)
    f = io.StringIO()
    for line in a.reshape(-1, 4):
        np.savetxt(f, line[np.newaxis], fmt="%f")
    f.seek(0)
    return np.loadtxt(f).reshape(a.shape)


def _homogeneous(depth, intrinsic):
    """(X, Y, Z) of the pixels with nonzero depth, in row-major pixel order (`:52-74`)."""
    depth = np.asarray(depth)
    H, W = depth.shape
    v, u = np.divmod(np.arange(H * W, dtype=np.int64), W)
    z = depth.reshape(-1)
    sel = np.flatnonzero(z != 0)
    d = z[sel] / 1000.0
    K = np.asarray(intrinsic, np.float64)
    fx, fy, cx, cy, bx, by = K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 3], K[1, 3]
    X = (u[sel].astype(np.float64) - cx) * d / fx + bx
    Y = (v[sel].astype(np.float64) - cy) * d / fy + by
    return X, Y, d


def depth_to_points(depth, intrinsic, pose):
    """depth uint16 [H, W], intrinsic [4, 4], pose fp64 [4, 4] -> fp64 [n, 3] world points of the nonzero pixels."""
    X, Y, Z = _homogeneous(depth, intrinsic)
    P = np.asarray(pose, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.stack([((X * P[r, 0] + Y * P[r, 1]) + Z * P[r, 2]) + P[r, 3] for r in range(3)], 1)


def dot_bound(depth, intrinsic, pose):
    """fp64 [n, 3]: 2 gamma_4 (|X P[r,0]| + |Y P[r,1]| + |Z P[r,2]| + |P[r,3]|), the largest difference between `depth_to_points` and
    any summation order of `np.dot(points, pose.T)`, with or without FMA."""
    X, Y, Z = _homogeneous(depth, intrinsic)
    P = np.asarray(pose, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.stack([np.abs(X * P[r, 0]) + np.abs(Y * P[r, 1]) + np.abs(Z * P[r, 2]) + np.abs(P[r, 3]) for r in range(3)], 1)
    return 2 * GAMMA4 * s * (1 + 4 * U)         # the sum of magnitudes is itself rounded: a margin of 4 ulp covers it


def within_bound(got, want, bound):
    """got and want agree: equal where either is not finite (NaN equal to NaN), within `bound` elsewhere."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if got.shape != want.shape:
        return False
    fin = np.isfinite(got) & np.isfinite(want)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    with np.errstate(invalid="ignore"):
        return bool(np.all(np.where(fin, np.abs(got - want) <= bound, same)))
