"""CPU oracle of the pretraining pair list (pointcontrast_b200.pair_list), restating the reference's
`pretrain/data_preprocess/scannet_pair/compute_full_overlapping.py` and `generate_list.py` in numpy / scipy:

    voxel_down_sample(xyz, voxel_size)          open3d `PointCloud.voxel_down_sample` (`:15-26`, `:59-63`)
    frame_overlap_counts(frames, radius)        counts[i, j] = len(get_matching_indices(pcd_j, tree_i, radius, K=1)) (`:39-47`, `:67-74`)
    write_overlap(path, names, counts, sizes)   `:76-83`
    write_list(target_dir, overlap_files)       `generate_list.py:20-28`

open3d is not installed, so its semantics are restated as recalled (DESIGN.md section 5): `VoxelDownSample` puts a point in voxel
floor((p - (min - voxel_size / 2)) / voxel_size), sums the points of a voxel in ascending index and divides by their number; the radius
search keeps a point when its squared distance is below radius^2.  fp64 throughout, as the npz frames and open3d.
"""
import os

import numpy as np
from scipy.spatial import cKDTree


def voxel_down_sample(xyz, voxel_size):
    """fp64 [n, 3] -> the voxel averages [m, 3], in ascending (x, y, z) voxel index."""
    xyz = np.asarray(xyz, np.float64)
    if len(xyz) == 0:
        return np.zeros((0, 3))
    lo = xyz.min(0) - voxel_size * 0.5
    idx = np.floor((xyz - lo) / voxel_size).astype(np.int64)         # >= 0
    ext = idx.max(0) + 1
    if float(ext[0]) * float(ext[1]) * float(ext[2]) < 2.0 ** 62:     # one int64 key in (x, y, z) order: same runs, faster
        _, inv = np.unique((idx[:, 0] * ext[1] + idx[:, 1]) * ext[2] + idx[:, 2], return_inverse=True)
    else:
        _, inv = np.unique(idx, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    sums = np.zeros((inv.max() + 1, 3))
    np.add.at(sums, inv, xyz)                    # unbuffered, in index order: open3d's AddPoint sequence
    return sums / np.bincount(inv).astype(np.float64)[:, None]


def within(p, q, radius):
    """The decision of the GPU kernel: ((dx dx + dy dy) + dz dz) < radius^2 in fp64 (numpy does not contract to FMA)."""
    d = np.asarray(p, np.float64) - np.asarray(q, np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2] < radius * radius


def frame_overlap_counts(frames, radius):
    """frames: list of fp64 [n_f, 3].  counts[i, j] (int64 [F, F], diagonal 0) = the number of points of frame j with a point of frame
    i != j within `radius`.  Candidates come from cKDTree at radius (1 + 1e-9), the decision from `within`."""
    F = len(frames)
    counts = np.zeros((F, F), np.int64)
    sizes = [len(f) for f in frames]
    if sum(sizes) == 0:
        return counts
    allp = np.concatenate([np.asarray(f, np.float64).reshape(-1, 3) for f in frames])
    frame = np.repeat(np.arange(F), sizes)
    tree = cKDTree(allp)
    start = np.concatenate([[0], np.cumsum(sizes)])
    for j in range(F):
        if sizes[j] == 0:
            continue
        cand = cKDTree(allp[start[j]:start[j + 1]]).sparse_distance_matrix(tree, radius * (1 + 1e-9), output_type="ndarray")
        q, p = cand["i"].astype(np.int64), cand["j"].astype(np.int64)
        keep = (frame[p] != j) & within(allp[start[j] + q], allp[p], radius)
        hit = np.unique(q[keep] * F + frame[p[keep]])
        counts[:, j] = np.bincount(hit % F, minlength=F)
    return counts


def overlap_matrix(counts, sizes):
    """M[i, j] = counts[i, j] / n_j in fp64 (`:74`)."""
    return counts.astype(np.float64) / np.asarray(sizes, np.float64)[None, :]


def write_overlap(path, names, counts, sizes):
    """`:78-83`: "<name_i> <name_j> <max(M[i, j], M[j, i])>" for i < j."""
    M = overlap_matrix(counts, sizes)
    with open(path, "w") as f:
        for i in range(len(names)):
            for j in range(i + 1, len(names)):
                f.write("{} {} {}\n".format(names[i], names[j], max(M[i, j], M[j, i])))


def write_list(target_dir, overlap_files, threshold=0.3):
    """`generate_list.py:20-28` over the given overlap.txt files, in the given order."""
    with open(os.path.join(target_dir, "overlap-30-full.txt"), "w") as f:
        for fo in overlap_files:
            for line in open(fo):
                pcd0, pcd1, op = line.strip().split()
                if float(op) >= threshold:
                    print("{} {} {}".format(pcd0, pcd1, op), file=f)
