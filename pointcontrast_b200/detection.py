"""VoteNet's sparse-conv detection backbone on libpcb200 (DESIGN.md 8f-7): the pretrained Res16UNet34C with a 256-wide head, which
PointContrast's detection results use (`downstream/votenet_det_new/scripts/train_scannet.sh`, `train_sunrgbd.sh`:
`net.backbone=sparseconv data.voxelization=True data.voxel_size=0.025`).

    batch = {k: v.cuda() for k, v in default_collate(samples).items()}       # `lib/train.py:63-64`
    voxelize_batch(batch, 0.025)                                               # + voxel_coords / voxel_inds / voxel_feats
    backbone = SparseConvBackbone().cuda()
    end_points = backbone(batch["point_clouds"], batch["voxel_coords"], batch["voxel_feats"], batch["voxel_inds"], {})

`voxelize_batch` replaces the reference's CPU voxelisation in the DataLoader workers (`models/backbone/sparseconv/
voxelized_dataset.py:33-65`, `ME.utils.sparse_quantize(coords, return_index=True)` per scene) and its `collate_fn`: one batched
kernel call on the collated batch.  `SparseConvBackbone` mirrors `models/backbone_module.py:134-180`: the network runs as one fused
pass, and the 1024 seeds of every scene come from ONE ragged furthest-point-sampling launch instead of a per-scene Python loop with
boolean-mask gathers and host synchronisations.  Seeds, their coordinates and indices are bit-identical to the per-scene loop; the
seed gather's backward is deterministic (a fixed-order fp64 adjoint, not atomics).
"""
import torch
import torch.nn as nn
from torch.autograd import Function

from . import me as ME
from . import pointnet2, voxel
from ._lib import PcbError, require_cuda
from .config import default_config
from .model import load_model


def voxelize_batch(batch, voxel_size):
    """Adds to a collated batch on the device what the reference's `VoxelizationDataset` + `collate_fn` produce: voxel_coords int32
    [M, 4] = (scene, x, y, z) with x = floor(point / voxel_size) in fp32, voxel_inds int32 [M] (the scene-local index of each voxel's
    first point), voxel_feats fp32 ones [M, 3].  Rows are scene-major, within a scene in ascending voxel_inds.  `point_clouds` must be
    fp32 [B, N, 3] (`no_height=True`, `use_color=False`, what both detection scripts set).  Returns the batch."""
    xyz = batch["point_clouds"]
    require_cuda(xyz)
    if xyz.dim() != 3 or xyz.shape[2] != 3 or xyz.dtype != torch.float32:
        raise PcbError(f"point_clouds must be fp32 [B, N, 3], got {xyz.dtype} {tuple(xyz.shape)}")
    coords, inds, _, _ = voxel.voxelize_scenes(xyz, voxel_size)
    batch["voxel_coords"] = coords
    batch["voxel_inds"] = inds
    batch["voxel_feats"] = xyz.new_ones(coords.shape[0], 3)
    return batch


def backbone_config(model="Res16UNet34C"):
    """The sparse-conv `config.py` defaults the network reads: conv1_kernel_size 3, bn_momentum 0.02, no feature normalisation."""
    return default_config([f"net.model={model}", "net.conv1_kernel_size=3", "net.normalize_feature=False", "opt.bn_momentum=0.02"])


class _SeedGather(Function):
    """rows [M, C] -> rows[idx] [L, C]; the backward sums each row's readers in ascending order in fp64 (`pcb_gather_rows_grad`), so a
    seed repeated by furthest-point sampling (a scene with fewer voxels than seeds) gets the same gradient on every run."""

    @staticmethod
    def forward(ctx, rows, idx):
        ctx.save_for_backward(idx)
        ctx.m = rows.shape[0]
        return rows.index_select(0, idx)

    @staticmethod
    def backward(ctx, grad):
        idx, = ctx.saved_tensors
        return pointnet2.gather_rows_grad(grad.contiguous(), idx, ctx.m), None


def scene_offsets(batch_col, B):
    """int64 [B + 1]: rows of scene b are [offsets[b], offsets[b+1]) of a scene-major batch column, on the device."""
    batch_col = batch_col.contiguous()
    return torch.searchsorted(batch_col, torch.arange(B + 1, dtype=batch_col.dtype, device=batch_col.device))


def sample_seeds(points, coords, inds, features, num_seed):
    """`models/backbone_module.py:160-178` in one pass: furthest-point sampling of every scene's voxel points (points[b, inds]) in one
    ragged launch, then the gathers.  Returns (fp2_features [B, C, num_seed], fp2_xyz [B, num_seed, 3], fp2_inds int32 [B, num_seed])."""
    B, N, _ = points.shape
    batch_col = coords[:, 0]
    offsets = scene_offsets(batch_col, B)
    vxyz = points.reshape(-1, 3)[inds.long() + batch_col.long() * N].contiguous()
    sel = pointnet2.furthest_point_sampling_ragged(vxyz, offsets, N, num_seed)       # a scene has at most N voxels
    rows = (offsets[:B, None] + sel).reshape(-1)
    fp2_inds = inds[rows].view(B, num_seed)
    fp2_xyz = vxyz[rows].view(B, num_seed, 3)
    fp2_features = _SeedGather.apply(features, rows.to(torch.int32)).view(B, num_seed, -1).transpose(1, 2)
    return fp2_features, fp2_xyz, fp2_inds


class SparseConvBackbone(nn.Module):
    """`models/backbone_module.py:134-180`: same constructor, forward signature, `end_points` entries and state_dict (`net.` + the
    Res16UNet34C keys), so `semseg.load_state_with_same_shape(backbone.net, ckpt["state_dict"])` loads pretraining checkpoints as
    `ddp_main.py:146-156` does.  Like the original, `config` is accepted and ignored: the network takes the sparse-conv defaults."""

    def __init__(self, input_feature_dim=3, output_feature_dim=256, num_seed=1024, model="Res16UNet34C", config=None):
        super().__init__()
        self.net = load_model(model)(input_feature_dim, output_feature_dim, backbone_config(model), D=3)
        self.num_seed = num_seed

    def forward(self, points, coords, feats, inds, end_points=None):
        """points fp32 [B, N, 3], coords int32 [M, 4] scene-major, feats fp32 [M, 3], inds int32 [M] (`voxelize_batch`), all on the
        device -> end_points with fp2_features fp32 [B, 256, num_seed], fp2_xyz [B, num_seed, 3], fp2_inds int32 [B, num_seed]."""
        if end_points is None:
            end_points = {}
        for t in (points, coords, feats, inds):
            require_cuda(t)
        features = self.net(ME.SparseTensor(feats, coords=coords.int())).F
        f, xyz, ind = sample_seeds(points.contiguous(), coords, inds, features, self.num_seed)
        end_points["fp2_features"] = f
        end_points["fp2_xyz"] = xyz
        end_points["fp2_inds"] = ind
        return end_points
