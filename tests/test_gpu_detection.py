"""Sparse-conv detection backbone on the GPU (pointcontrast_b200/detection.py, csrc/voxel.cu, csrc/pointnet2.cu, DESIGN.md 8f-7):
batched voxelisation and ragged furthest-point sampling bit-exact against the per-scene entry points and the numpy oracle, the backbone
end to end against the fp64 oracle, the original unmodified module as a drop-in, determinism, BatchNorm momentum updates and the
fused eval path."""
import numpy as np
import pytest
import torch

from oracle import detection_cpu, me_cpu as OR
from oracle import pointnet2_cpu
from tests.helpers import det_init, max_rel_err, model_backend, pinned_relu, rel_err
from tests.test_host_detection import original_backbone_module

pytestmark = pytest.mark.gpu
VOXEL = 0.025
TOL = 1e-3


def special_scenes(rng, B, N):
    xyz = np.empty((B, N, 3), np.float32)
    for b in range(B):
        xyz[b] = (rng.random((N, 3)) * np.array([4.0, 4.0, 2.0]) - np.array([2.0, 2.0, 0.0])).astype(np.float32)
    if B > 1:
        xyz[0] = (np.float32(0.003) + rng.random((N, 3)).astype(np.float32) * np.float32(0.02))     # one voxel
        xyz[1] = xyz[1, rng.integers(0, max(1, N // 50), N)]                                         # heavy duplicates
    if B > 2:
        xyz[2] = (rng.integers(-40, 40, (N, 3)) * VOXEL).astype(np.float32)                          # on cell boundaries
    return xyz


@pytest.mark.parametrize("B", [1, 8, 32])
@pytest.mark.parametrize("N", [1, 1000, 40000])
def test_voxelize_batch_per_scene_and_oracle(B, N):
    from pointcontrast_b200 import detection, voxel
    xyz = special_scenes(np.random.default_rng(B * 7 + N), B, N)
    batch = detection.voxelize_batch({"point_clouds": torch.from_numpy(xyz).cuda()}, VOXEL)
    coords, inds, feats = batch["voxel_coords"].cpu(), batch["voxel_inds"].cpu(), batch["voxel_feats"]
    assert coords.dtype == torch.int32 and inds.dtype == torch.int32 and feats.dtype == torch.float32
    assert torch.equal(feats, torch.ones_like(feats))
    _, _, offsets, host = voxel.voxelize_scenes(torch.from_numpy(xyz).cuda(), VOXEL)
    assert offsets.cpu().tolist() == host and host[-1] == len(coords)
    for b in range(B):
        rows = slice(host[b], host[b + 1])
        assert (coords[rows, 0] == b).all()
        c1, s1 = voxel.voxelize(torch.from_numpy(xyz[b]).cuda(), VOXEL)        # the scene alone, rows in (x, y, z) order
        order = torch.argsort(s1.cpu())
        assert torch.equal(coords[rows, 1:], c1.cpu()[order]) and torch.equal(inds[rows].long(), s1.cpu()[order])
    oc, oi, oo = detection_cpu.voxelize_scenes(xyz, VOXEL)
    assert np.array_equal(coords.numpy(), oc) and np.array_equal(inds.numpy(), oi) and host == oo.tolist()
    if B > 1 and N > 1:
        assert host[1] - host[0] == 1


def ragged_scenes():
    rng = np.random.default_rng(11)
    sizes = [1, 500, 1024, 5000, 30000, 110000] * 5
    scenes = [(rng.random((n, 3)) * np.array([6.0, 6.0, 2.5]) - np.array([3.0, 3.0, 0.5])).astype(np.float32) for n in sizes]
    skip = scenes[1].copy()
    skip[:200] *= np.float32(0.01)                          # inside the 1e-3 origin skip radius
    ties = np.repeat(scenes[2][:64], 16, axis=0)            # exact ties
    return scenes + [skip, ties]


def test_ragged_fps_matches_per_scene_and_oracle():
    from pointcontrast_b200 import pointnet2
    scenes = ragged_scenes()
    assert len(scenes) == 32
    pts = torch.from_numpy(np.concatenate(scenes)).cuda()
    offsets = torch.tensor(np.cumsum([0] + [len(s) for s in scenes]), dtype=torch.int64, device="cuda")
    max_n = max(len(s) for s in scenes)
    from pointcontrast_b200 import _lib
    assert _lib.lib.pcb_furthest_point_sampling_ragged_ws_bytes(32, pts.shape[0], max_n) > 0      # the largest scenes spill
    got = pointnet2.furthest_point_sampling_ragged(pts, offsets, max_n, 1024).cpu()
    again = pointnet2.furthest_point_sampling_ragged(pts, offsets, max_n + 5000, 1024).cpu()       # a looser bound: same result
    assert torch.equal(got, again)
    for b, s in enumerate(scenes):
        one = pointnet2.furthest_point_sampling(torch.from_numpy(s[None]).cuda(), 1024).cpu()[0]
        assert torch.equal(got[b], one), b
        if len(s) <= 30000:
            assert torch.equal(got[b], pointnet2_cpu.furthest_point_sampling(torch.from_numpy(s[None]), 1024)[0]), b
    big = [b for b, s in enumerate(scenes) if len(s) == 110000][:1]
    for b in big:
        assert torch.equal(got[b], pointnet2_cpu.furthest_point_sampling(torch.from_numpy(scenes[b][None]), 1024)[0])


def make_batch(B, N, seed=0):
    from pointcontrast_b200 import detection, synth
    xyz = torch.from_numpy(synth.synth_votenet_batch(seed, B, N)).cuda()
    return detection.voxelize_batch({"point_clouds": xyz}, VOXEL)


def run_backbone(bb, batch, w=None):
    ep = bb(batch["point_clouds"], batch["voxel_coords"], batch["voxel_feats"], batch["voxel_inds"], {})
    if w is not None:
        (ep["fp2_features"] * w).sum().backward()
    return ep


@pytest.mark.parametrize("N", [20000, 40000])
def test_backbone_end_to_end_against_fp64_oracle(N):
    from pointcontrast_b200 import detection, fused
    batch = make_batch(2, N, seed=N)
    bb = detection.SparseConvBackbone()
    det_init(bb.net, 9)
    state = {k: v.clone() for k, v in bb.net.state_dict().items()}
    bb = bb.cuda().train()
    w = torch.from_numpy(np.random.default_rng(N).standard_normal((2, 256, 1024)).astype(np.float32)).cuda()
    fused.CAPTURE_RELU = cap = []
    try:
        ep = run_backbone(bb, batch, w)
    finally:
        fused.CAPTURE_RELU = None
    assert "_fused_runner" in bb.net.__dict__ and len(cap) > 0
    masks = [m.cpu() for _, m in cap]
    coords, inds = batch["voxel_coords"].cpu(), batch["voxel_inds"].cpu()
    flips = []
    with pinned_relu(OR, masks, flips), model_backend(OR) as mod:
        onet = mod.Res16UNet34C(3, 256, detection.backbone_config(), D=3).double()
        onet.load_state_dict({k: (v.double() if v.dtype.is_floating_point else v) for k, v in state.items()})
        onet.train()
        Fo = onet(OR.SparseTensor(torch.ones(len(coords), 3, dtype=torch.float64), coords=coords)).F
    of, ox, oi = detection_cpu.sample_seeds(batch["point_clouds"].cpu().numpy(), coords.numpy(), inds.numpy(), Fo, 1024)
    (of * w.cpu().double()).sum().backward()
    assert torch.equal(ep["fp2_inds"].cpu(), oi) and torch.equal(ep["fp2_xyz"].cpu(), ox)
    assert max_rel_err(ep["fp2_features"], of) < TOL
    assert sum(flips) <= 1e-4 * sum(m.numel() for m in masks)
    og = dict(onet.named_parameters())
    errs = {k: rel_err(p.grad, og[k].grad) for k, p in bb.net.named_parameters()}
    assert len(errs) == len(og) and max(errs.values()) < TOL, sorted(errs.items(), key=lambda t: -t[1])[:5]


def test_original_module_is_a_drop_in():
    from pointcontrast_b200 import detection
    bm = original_backbone_module()
    batch = make_batch(4, 20000, seed=3)
    ours = detection.SparseConvBackbone()
    det_init(ours.net, 4)
    ref = bm.SparseConvBackbone()
    ref.load_state_dict(ours.state_dict())
    ours, ref = ours.cuda().train(), ref.cuda().train()
    w = torch.from_numpy(np.random.default_rng(5).standard_normal((4, 256, 1024)).astype(np.float32)).cuda()
    a, b = run_backbone(ours, batch, w), run_backbone(ref, batch, w)
    assert "_fused_runner" in ref.net.__dict__
    for k in ("fp2_features", "fp2_xyz", "fp2_inds"):
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
    gb = dict(ref.named_parameters())
    for k, p in ours.named_parameters():
        assert torch.equal(p.grad, gb[k].grad), k


def test_two_runs_are_bit_identical_with_a_small_scene():
    from pointcontrast_b200 import detection
    batch = make_batch(3, 20000, seed=5)
    small = make_batch(1, 300, seed=6)["point_clouds"]                     # fewer voxels than seeds: FPS repeats an index
    pc = batch["point_clouds"].clone()
    pc[1, :300] = small[0]
    pc[1, 300:] = small[0, :1]
    batch = detection.voxelize_batch({"point_clouds": pc}, VOXEL)
    counts = torch.bincount(batch["voxel_coords"][:, 0].long()).tolist()
    assert counts[1] < 1024
    bb = detection.SparseConvBackbone()
    det_init(bb.net, 2)
    bb = bb.cuda().train()
    w = torch.from_numpy(np.random.default_rng(1).standard_normal((3, 256, 1024)).astype(np.float32)).cuda()
    runs = []
    for _ in range(2):
        bb.zero_grad(set_to_none=True)
        ep = run_backbone(bb, batch, w)
        runs.append(({k: v.detach().clone() for k, v in ep.items()}, {k: p.grad.clone() for k, p in bb.named_parameters()}))
    assert len(set(runs[0][0]["fp2_inds"][1].tolist())) <= counts[1]           # repeated seeds share one feature row
    for k in runs[0][0]:
        assert torch.equal(runs[0][0][k], runs[1][0][k]), k
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k


def test_assigned_bn_momentum_is_used_by_the_next_step():
    """`pytorch_utils.BNMomentumScheduler` assigns `momentum` on the inner nn.BatchNorm1d between steps."""
    from pointcontrast_b200 import detection, me
    batch = make_batch(2, 20000, seed=8)
    bb = detection.SparseConvBackbone()
    det_init(bb.net, 3)
    bb = bb.cuda().train()
    bns = [m.bn for m in bb.modules() if isinstance(m, me.MinkowskiBatchNorm)]
    init = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in bns]

    def step(momentum):
        for bn, (m, v) in zip(bns, init):
            bn.momentum = momentum
            bn.running_mean.copy_(m); bn.running_var.copy_(v)
        run_backbone(bb, batch)
        return [(bn.running_mean - m).double() for bn, (m, _) in zip(bns, init)]

    assert all(float(d.abs().max()) == 0.0 for d in step(0.0))
    half, quarter = step(0.5), step(0.25)
    for h, q in zip(half, quarter):
        assert float(h.abs().max()) > 0 and float((h - 2 * q).abs().max()) <= 1e-5 * float(h.abs().max()) + 1e-12


def test_eval_takes_the_fused_eval_path_with_the_training_seeds():
    from pointcontrast_b200 import detection, fused, me
    batch = make_batch(2, 20000, seed=9)
    bb = detection.SparseConvBackbone()
    det_init(bb.net, 6)
    bb = bb.cuda()
    train = run_backbone(bb.train(), batch)
    bb.eval()
    with torch.no_grad():
        st = me.SparseTensor(batch["voxel_feats"], coords=batch["voxel_coords"])
        assert fused.applicable_eval(bb.net, st)
        ev = run_backbone(bb, batch)
    assert torch.equal(ev["fp2_inds"], train["fp2_inds"]) and torch.equal(ev["fp2_xyz"], train["fp2_xyz"])
    assert torch.isfinite(ev["fp2_features"]).all() and ev["fp2_features"].shape == (2, 256, 1024)
