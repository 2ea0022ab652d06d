"""numpy restatement of the sparse-conv detection backbone's data steps, the checker of pointcontrast_b200/detection.py:

  * voxelize_scenes: `downstream/votenet_det_new/models/backbone/sparseconv/voxelized_dataset.py:33-65` -- per scene
    `np.floor(point_clouds / VOXEL_SIZE)` in float32 and `sparse_quantize(coords, return_index=True)` (here `np.unique(...,
    return_index=True)`: the first point of each voxel), the rows in ascending first index, then `collate_fn`'s batch column;
  * sample_seeds: `models/backbone_module.py:160-178` -- per scene furthest-point sampling of the voxel points
    (oracle.pointnet2_cpu.furthest_point_sampling) and the gathers of indices, points and features.
"""
import numpy as np
import torch

from oracle import pointnet2_cpu


def voxelize_scenes(xyz, voxel_size):
    """xyz float32 [B, N, 3] -> (coords int32 [M, 4] = (b, x, y, z), inds int32 [M], offsets int64 [B + 1])."""
    xyz = np.asarray(xyz, dtype=np.float32)
    coords, inds, offsets = [], [], [0]
    for b in range(xyz.shape[0]):
        cells = np.floor(xyz[b] / np.float32(voxel_size)).astype(np.int64)          # `voxelized_dataset.py:33`
        _, first = np.unique(cells, axis=0, return_index=True)                      # `:34`
        first = np.sort(first)
        coords.append(np.concatenate([np.full((len(first), 1), b, np.int64), cells[first]], 1).astype(np.int32))   # `:35`, `:54-55`
        inds.append(first.astype(np.int32))
        offsets.append(offsets[-1] + len(first))
    return np.concatenate(coords), np.concatenate(inds), np.asarray(offsets, np.int64)


def sample_seeds(points, coords, inds, features, num_seed):
    """points float32 [B, N, 3], coords [M, 4], inds [M], features [M, C] (torch, any float dtype) -> (fp2_features [B, C, num_seed],
    fp2_xyz [B, num_seed, 3], fp2_inds int32 [B, num_seed]) as the original's per-scene loop computes them."""
    points = np.asarray(points, dtype=np.float32)
    B, N, _ = points.shape
    flat = points.reshape(-1, 3)
    batch_ids = np.asarray(coords)[:, 0]
    inds = np.asarray(inds)
    voxel_ids = inds.astype(np.int64) + batch_ids.astype(np.int64) * N                          # `backbone_module.py:166`
    f_out, x_out, i_out = [], [], []
    for b in range(B):
        m = batch_ids == b
        p = flat[voxel_ids[m]]
        sid = pointnet2_cpu.furthest_point_sampling(torch.from_numpy(p[None]), num_seed)[0].numpy().astype(np.int64)   # `:169-171`
        i_out.append(inds[m][sid])                                                               # `:173`
        f_out.append(features[torch.from_numpy(np.nonzero(m)[0][sid])])                         # `:174`
        x_out.append(p[sid])                                                                     # `:175`
    return torch.stack(f_out, 0).transpose(1, 2), torch.from_numpy(np.stack(x_out)), torch.from_numpy(np.stack(i_out).astype(np.int32))
