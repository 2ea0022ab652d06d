"""VotingModule / ProposalModule on the library (pointcontrast_b200/det_heads.py, csrc/det_head.cu, DESIGN.md 8f-18) against the fp64
oracle (oracle/det_heads_cpu.py) at ScanNet's and SUN RGB-D's widths, vote_factor 1 and 2, a small batch and the training scripts'
batch, in training and eval mode:
  * outputs within 1e-4 of fp64 relative to their largest magnitude;
  * gradients of the inputs and every parameter within tests/test_gpu_pointnet2_modules.py's GRAD_TOL (norm-relative; the conv biases
    in front of a BatchNorm, whose gradient is zero up to rounding, against a floor of 1e-4 of the largest gradient), running statistics
    and num_batches_tracked;
  * two calls give the same bits; the epilogues bit-identical to the original's torch expressions on the same z;
  * weights updated in place between two calls are picked up; eval mode is forward only;
  * the unmodified VoteNet after det_heads.install() against its torch heads, both backbones (the drop-in test)."""
import copy

import numpy as np
import pytest
import torch

from oracle import det_heads_cpu as H
from tests.test_gpu_pointnet2_modules import GRAD_TOL

pytestmark = pytest.mark.gpu
D = torch.float64
DATASETS = {"scannet": (1, 18, 18, 32), "sunrgbd": (12, 10, 10, 64)}        # NH, NS, C, scenes per batch in the training script
BIASES_BEFORE_BN = (1, 3)                                                     # conv1.bias, conv2.bias in registration order


@pytest.fixture(scope="module")
def M():
    from pointcontrast_b200 import det_heads
    return det_heads


def perturb_bn(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in (mod.bn1, mod.bn2):
            m.weight.copy_(torch.randn(m.num_features, generator=g))
            m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)


def point_major(B, C, P, seed):
    """Features [B, C, P] as the backbones and the vote aggregation return them: a channel-major view of point-major storage."""
    x = torch.from_numpy(np.random.default_rng(seed).standard_normal((B, P, C)).astype(np.float32))
    return x.cuda().transpose(1, 2)


def max_rel(a, b):
    return float((a.double().cpu() - b.detach()).abs().max() / b.detach().abs().max())


def grad_errs(ours, want):
    """Norm-relative gradient errors; the biases in front of a BatchNorm against 1e-4 of the largest gradient at least."""
    floor = 1e-4 * max(float(b.norm()) for b in want if b is not None)
    errs = {}
    for i, (a, b) in enumerate(zip(ours, want)):
        den = float(b.norm())
        if i - 2 in BIASES_BEFORE_BN:
            den = max(den, floor)
        errs[i] = float((a.double().cpu().reshape(b.shape) - b).norm()) / den
    return errs


class _View:
    def __init__(self, p, n, ld):
        self.__cuda_array_interface__ = {"shape": (n, ld), "strides": (4 * ld, 4), "typestr": "<f4", "data": (p, False), "version": 2}


class _CaptureZ:
    """Stands in for det_heads' `lib` and copies the z [rows, ldz] each epilogue call reads."""

    def __init__(self, lib):
        self.lib, self.z = lib, None

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if name not in ("pcb_vote_epilogue", "pcb_proposal_epilogue"):
            return f

        def call(*a):
            rc = f(*a)
            if name == "pcb_vote_epilogue":
                z, ldz, n = a[3], a[4], a[5] * a[6]
            else:
                z, ldz, n = a[0], a[1], a[3] * a[4]
            self.z = torch.as_tensor(_View(z, n, ldz), device="cuda").clone()
            return rc
        return call


def _params(mod):
    return [mod.conv1.weight, mod.conv1.bias, mod.conv2.weight, mod.conv2.bias, mod.conv3.weight, mod.conv3.bias, mod.bn1.weight,
            mod.bn1.bias, mod.bn2.weight, mod.bn2.bias]


# ------------------------------------------------------------------------------------------------ voting
def _vote_run(M, mod, xyz, f, train, gx, gf, monkeypatch):
    cap = _CaptureZ(M.lib)
    monkeypatch.setattr(M, "lib", cap)
    mod.train(train)
    x = xyz.clone().requires_grad_(train)
    ff = f.detach().clone().requires_grad_(train) if train else f
    with torch.set_grad_enabled(train):
        vx, vf = mod(x, ff)
        if train:
            ((vx * gx).sum() + (vf * gf).sum()).backward()
    monkeypatch.setattr(M, "lib", cap.lib)
    grads = [x.grad, ff.grad] + [p.grad for p in _params(mod)] if train else []
    return vx.detach(), vf.detach(), grads, cap.z


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("B", [2, 64])
@pytest.mark.parametrize("V", [1, 2])
def test_voting_matches_oracle(M, V, B, train, monkeypatch):
    S, C = 1024, 256
    torch.manual_seed(0)
    mod = M.VotingModule(V, C)
    perturb_bn(mod, 1)
    mod = mod.cuda()
    twin = copy.deepcopy(mod)
    p = H.head_params(mod.state_dict())
    xyz = torch.from_numpy(np.random.default_rng(2).uniform(-3, 3, (B, S, 3)).astype(np.float32)).cuda()
    f = point_major(B, C, S, 3)
    gx = torch.randn(B, S * V, 3, generator=torch.Generator().manual_seed(4)).cuda()
    gf = torch.randn(B, C, S * V, generator=torch.Generator().manual_seed(5)).cuda()
    stats0 = {k: v.clone() for k, v in mod.state_dict().items()}
    vx, vf, grads, z = _vote_run(M, mod, xyz, f, train, gx, gf, monkeypatch)
    assert vx.is_contiguous() and vf.shape == (B, C, S * V) and vf.stride() == (S * V * C, 1, C)
    if not train:
        assert all(torch.equal(v, stats0[k]) for k, v in mod.state_dict().items())
    again = _vote_run(M, twin, xyz, f, train, gx, gf, monkeypatch)
    assert torch.equal(vx, again[0]) and torch.equal(vf, again[1])
    assert all(torch.equal(a, b) for a, b in zip(grads, again[2]))
    # the epilogue: the original's torch expressions on the same z
    net = z[:, :(3 + C) * V].view(B, S, V, 3 + C)
    assert torch.equal(vx, (xyz.unsqueeze(2) + net[..., :3]).contiguous().view(B, S * V, 3))
    want_f = (f.transpose(2, 1).unsqueeze(2) + net[..., 3:]).contiguous().view(B, S * V, C).transpose(2, 1)
    assert torch.equal(vf, want_f)
    xo, fo = xyz.double().cpu().requires_grad_(), f.double().cpu().requires_grad_()
    ox, of = H.voting(xo, fo, p, V, train)
    errs = (max_rel(vx, ox), max_rel(vf, of))
    assert max(errs) < 1e-4, errs
    if not train:
        return
    ((ox * gx.double().cpu()).sum() + (of * gf.double().cpu()).sum()).backward()
    e = grad_errs(grads, [xo.grad, fo.grad] + H.grads(p))
    print("voting V", V, "B", B, "output errs", errs, "grad errs", {k: f"{v:.2e}" for k, v in e.items()})
    assert max(e.values()) < GRAD_TOL, e
    for c in ("bn1", "bn2"):
        bn = getattr(mod, c)
        assert max_rel(bn.running_mean, p[c]["running_mean"]) < 1e-4 and max_rel(bn.running_var, p[c]["running_var"]) < 1e-4
        assert int(bn.num_batches_tracked) == 1


def test_voting_partial_gradients(M):
    """Only vote_features reach the loss (vote_xyz's gradient absent), through a strided gradient: the same as a zero vote_xyz
    gradient; seed_xyz then gets zeros."""
    torch.manual_seed(0)
    mod = M.VotingModule(2, 64).cuda()
    twin = copy.deepcopy(mod)
    xyz = torch.rand(2, 64, 3, device="cuda")
    f = point_major(2, 64, 64, 7)
    res = []
    for m, with_xyz in ((mod, False), (twin, True)):
        x, ff = xyz.clone().requires_grad_(), f.detach().clone().requires_grad_()
        vx, vf = m(x, ff)
        loss = (vf * vf).sum() + (0 * vx.sum() if with_xyz else 0)
        loss.backward()
        res.append([x.grad, ff.grad] + [p.grad for p in _params(m)])
    assert all(torch.equal(a, b) for a, b in zip(*res))
    assert torch.equal(res[0][0], torch.zeros_like(xyz))


# ------------------------------------------------------------------------------------------------ proposal head
class _Aggregation(torch.nn.Module):
    """Stands in for the vote aggregation (tested on its own in tests/test_gpu_pointnet2_modules.py): returns the given outputs."""

    def __init__(self, out):
        super().__init__()
        self.out = out

    def forward(self, *args):
        return self.out


def _proposal_run(M, mod, agg, f, train, gs, monkeypatch):
    cap = _CaptureZ(M.lib)
    monkeypatch.setattr(M, "lib", cap)
    mod.train(train)
    a = agg.clone().requires_grad_(train)
    ff = f.detach().clone().requires_grad_(train) if train else f
    inds = torch.zeros(agg.shape[:2], dtype=torch.int32, device="cuda")
    mod.vote_aggregation = _Aggregation((a, ff, inds))
    with torch.set_grad_enabled(train):
        ep = mod(None, None, {})
        if train:
            sum((ep[k] * g).sum() for k, g in zip(H.DECODE, gs)).backward()
    monkeypatch.setattr(M, "lib", cap.lib)
    grads = [a.grad, ff.grad] + [p.grad for p in _params(mod)] if train else []
    return {k: ep[k].detach() for k in H.DECODE}, grads, cap.z


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("size", ["small", "script"])
@pytest.mark.parametrize("dataset", list(DATASETS))
def test_proposal_matches_oracle(M, dataset, size, train, monkeypatch):
    NH, NS, C, B_script = DATASETS[dataset]
    B, K = (2 if size == "small" else B_script), 256
    ms = np.random.default_rng(6).uniform(0.3, 2.0, (NS, 3))
    torch.manual_seed(0)
    mod = M.ProposalModule(C, NH, NS, ms, K, "vote_fps")
    perturb_bn(mod, 2)
    mod = mod.cuda()
    twin = copy.deepcopy(mod)
    p = H.head_params(mod.state_dict())
    agg = torch.from_numpy(np.random.default_rng(7).uniform(-3, 3, (B, K, 3)).astype(np.float32)).cuda()
    f = torch.relu(point_major(B, 128, K, 8))
    shapes = {k: v.shape for k, v in H.decode(torch.zeros(B, K, 5 + 2 * NH + 4 * NS + C, dtype=D), torch.zeros(B, K, 3, dtype=D), NH, NS,
                                                 ms).items()}
    gs = [torch.randn(shapes[k], generator=torch.Generator().manual_seed(20 + i)).cuda() for i, k in enumerate(H.DECODE)]
    stats0 = {k: v.clone() for k, v in mod.state_dict().items()}
    ep, grads, z = _proposal_run(M, mod, agg, f, train, gs, monkeypatch)
    if not train:
        assert all(torch.equal(v, stats0[k]) for k, v in mod.state_dict().items())
    again = _proposal_run(M, twin, agg, f, train, gs, monkeypatch)
    assert all(torch.equal(ep[k], again[0][k]) for k in H.DECODE)
    assert all(torch.equal(a, b) for a, b in zip(grads, again[1]))
    # the epilogue: decode_scores' torch expressions on the same z
    net_t = z.view(B, K, -1)[:, :, :5 + 2 * NH + 4 * NS + C]
    s0 = 5 + 2 * NH
    assert torch.equal(ep["center"], agg + net_t[:, :, 2:5])
    assert torch.equal(ep["heading_residuals"], net_t[:, :, 5 + NH:s0] * (np.pi / NH))
    srn = net_t[:, :, s0 + NS:s0 + 4 * NS].view(B, K, NS, 3)
    assert torch.equal(ep["size_residuals"], srn * torch.from_numpy(ms.astype(np.float32)).cuda().unsqueeze(0).unsqueeze(0))
    for k, t in (("objectness_scores", net_t[:, :, 0:2]), ("sem_cls_scores", net_t[:, :, s0 + 4 * NS:]), ("size_residuals_normalized", srn)):
        assert torch.equal(ep[k], t), k
    ao, fo = agg.double().cpu().requires_grad_(), f.detach().double().cpu().requires_grad_()
    want = H.proposal(ao, fo, p, NH, NS, ms, train)
    errs = {k: max_rel(ep[k], want[k]) for k in H.DECODE}
    assert max(errs.values()) < 1e-4, errs
    if not train:
        return
    sum((want[k] * g.double().cpu()).sum() for k, g in zip(H.DECODE, gs)).backward()
    e = grad_errs(grads, [ao.grad, fo.grad] + H.grads(p))
    print("proposal", dataset, "B", B, "output err", max(errs.values()), "grad errs", {k: f"{v:.2e}" for k, v in e.items()})
    assert max(e.values()) < GRAD_TOL, e
    for c in ("bn1", "bn2"):
        bn = getattr(mod, c)
        assert max_rel(bn.running_mean, p[c]["running_mean"]) < 1e-4 and max_rel(bn.running_var, p[c]["running_var"]) < 1e-4
        assert int(bn.num_batches_tracked) == 1


def test_decode_scores_matches_the_original_expressions(M):
    """The stand-alone decode_scores on a channel-major net: the torch expressions' values, and autograd's gradient of net and of
    aggregated_vote_xyz."""
    NH, NS, C = 12, 10, 10
    B, K, X = 2, 64, 5 + 2 * NH + 4 * NS + C
    ms = np.random.default_rng(9).uniform(0.3, 2.0, (NS, 3))
    net = torch.randn(B, X, K, device="cuda", requires_grad=True)
    agg = torch.randn(B, K, 3, device="cuda", requires_grad=True)
    ep = M.decode_scores(net, {"aggregated_vote_xyz": agg}, C, NH, NS, ms)
    net2, agg2 = net.detach().clone().requires_grad_(), agg.detach().clone().requires_grad_()
    nt = net2.transpose(2, 1)
    s0 = 5 + 2 * NH
    srn = nt[:, :, s0 + NS:s0 + 4 * NS].reshape(B, K, NS, 3)
    want = dict(objectness_scores=nt[:, :, 0:2], center=agg2 + nt[:, :, 2:5], heading_scores=nt[:, :, 5:5 + NH],
                heading_residuals_normalized=nt[:, :, 5 + NH:s0], heading_residuals=nt[:, :, 5 + NH:s0] * (np.pi / NH),
                size_scores=nt[:, :, s0:s0 + NS], size_residuals_normalized=srn,
                size_residuals=srn * torch.from_numpy(ms.astype(np.float32)).cuda()[None, None], sem_cls_scores=nt[:, :, s0 + 4 * NS:])
    gs = {k: torch.randn(want[k].shape, device="cuda") for k in H.DECODE}
    for k in H.DECODE:
        assert torch.equal(ep[k], want[k]), k
    sum((ep[k] * gs[k]).sum() for k in H.DECODE if k != "heading_scores").backward()         # one gradient absent
    sum((want[k] * gs[k]).sum() for k in H.DECODE if k != "heading_scores").backward()
    assert torch.allclose(net.grad, net2.grad, rtol=1e-6, atol=1e-6) and torch.equal(agg.grad, agg2.grad)


def test_in_place_weight_update_between_calls(M):
    """An optimiser steps the weights and biases in place: the next forward uses them (the tiles follow both version counters)."""
    torch.manual_seed(0)
    mod = M.VotingModule(1, 256).cuda().eval()
    xyz = torch.rand(4, 256, 3, device="cuda")
    f = point_major(4, 256, 256, 10)
    with torch.no_grad():
        _, before = mod(xyz, f)
        opt = torch.optim.Adam(mod.parameters(), lr=0.05)
        for q in mod.parameters():
            q.grad = torch.randn_like(q)
        opt.step()
        _, after = mod(xyz, f)
    assert not torch.equal(before, after)
    _, of = H.voting(xyz.double().cpu(), f.double().cpu(), H.head_params(mod.state_dict()), 1, False)
    assert max_rel(after, of) < 1e-4


def test_eval_mode_is_forward_only(M):
    mod = M.VotingModule(1, 64).cuda().eval()
    with pytest.raises(NotImplementedError, match="no_grad"):
        mod(torch.rand(1, 32, 3, device="cuda"), point_major(1, 64, 32, 11))


# ------------------------------------------------------------------------------------------------ drop-in VoteNet
def _votenet(ours):
    """The staged, unmodified models/votenet.py on this library's `me`, PointNet++ operators and modules and det_loss, with (ours) or
    without det_heads.install()."""
    import importlib
    import sys
    import types
    from oracle import detection_ref, det_loss_ref, stage_ref
    if not (detection_ref.available() and det_loss_ref.available()):
        pytest.skip("oracle/_ref/votenet/models not staged (the original repository is absent)")
    try:                  # the original's plotting helpers import cv2 and never call it here: a cv2 that fails to import is stubbed
        importlib.import_module("cv2")
    except Exception:
        sys.modules["cv2"] = types.ModuleType("cv2")
    from oracle import det_eval_ref
    det_eval_ref.load()
    from pointcontrast_b200 import det_heads, det_loss, me, pointnet2, pointnet2_modules
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k in (
            "pointnet2_utils", "pointnet2_modules", "pytorch_utils", "backbone_module", "proposal_module", "voting_module", "loss_helper",
            "dump_helper")]:
        del sys.modules[k]
    me.install()
    pointnet2.install()
    # the original's pointnet2_utils imports pytorch_utils from its own directory, which the original pointnet2_modules puts on sys.path
    # when it is imported; here the library's pointnet2_modules stands in for it in both routes
    for p in (detection_ref.ROOT, stage_ref.path("votenet", "models", "backbone", "pointnet2")):
        if p not in sys.path:
            sys.path.insert(0, p)
    pointnet2_modules.install()
    if ours:
        det_heads.install()
    det_loss.install()
    votenet = importlib.import_module("models.votenet")
    assert (votenet.VotingModule is det_heads.VotingModule) == ours
    assert (votenet.ProposalModule is det_heads.ProposalModule) == ours
    return votenet


@pytest.mark.parametrize("backbone", ["pointnet2", "sparseconv"])
def test_votenet_heads_drop_in(backbone):
    """One Adam step of the unmodified VoteNet after det_heads.install(), against the same model on its torch heads (TF32 off), same
    weights: loss and every gradient, checkpoints loading both ways, the next loss after a step written in place, and
    BNMomentumScheduler's momentum on the heads' BatchNorms."""
    import importlib
    import sys
    from pointcontrast_b200 import det_heads, det_loss, detection, synth
    from tests.helpers import det_init
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    saved = dict(sys.modules)
    try:
        NH, NS, C = 12, 10, 10
        ms = np.random.default_rng(6).uniform(0.3, 2.0, (NS, 3))
        cfg = type("Cfg", (), dict(num_heading_bin=NH, num_size_cluster=NS, num_class=C, mean_size_arr=ms))()
        ep = synth.synth_votenet_loss_batch(41, 8, 20000, 1024, 256, 1, NH, ms, C)
        pts = torch.from_numpy(ep["point_clouds"]).cuda()
        inputs = {"point_clouds": pts}
        if backbone == "sparseconv":
            b = detection.voxelize_batch({"point_clouds": pts}, 0.025)
            inputs = {k: b[k] for k in ("point_clouds", "voxel_coords", "voxel_inds", "voxel_feats")}
        labels = ("center_label", "heading_class_label", "heading_residual_label", "size_class_label", "size_residual_label",
                  "sem_cls_label", "box_label_mask", "vote_label", "vote_label_mask")
        nets = []
        for ours in (False, True):
            votenet = _votenet(ours)
            torch.manual_seed(0)
            net = votenet.VoteNet(C, NH, NS, ms, input_feature_dim=0, num_proposal=256, vote_factor=1, sampling="seed_fps",
                                  backbone=backbone)
            if backbone == "sparseconv":
                det_init(net.backbone_net.net, 2)
            nets.append(net)
        ref, our = nets
        assert [(k, v.shape) for k, v in ref.state_dict().items()] == [(k, v.shape) for k, v in our.state_dict().items()]
        for k, v in ref.state_dict().items():
            assert torch.equal(v, our.state_dict()[k]), k                   # the same seeded construction
        our.load_state_dict(ref.state_dict())
        ref.load_state_dict(our.state_dict())
        assert isinstance(our.vgen, det_heads.VotingModule) and isinstance(our.pnet, det_heads.ProposalModule)
        ref, our = ref.cuda().train(), our.cuda().train()

        def step(net):
            net.zero_grad()
            end_points = net(dict(inputs))
            for k in labels:
                end_points[k] = torch.from_numpy(ep[k]).cuda()
            loss, _ = det_loss.get_loss(end_points, cfg)
            loss.backward()
            return float(loss.detach()), {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

        la, ga = step(ref)
        lb, gb = step(our)
        assert abs(la - lb) <= 1e-4 * abs(la), (la, lb)
        assert ga.keys() == gb.keys()
        # a convolution bias in front of a BatchNorm has a zero gradient in exact arithmetic: both routes give rounding noise there, so
        # every gradient is measured against at least 1e-4 of the largest one; ReLU and pool decisions within rounding may differ.
        floor = 1e-4 * max(float(g.norm()) for g in ga.values())
        errs = {k: float((ga[k] - gb[k]).norm()) / max(float(ga[k].norm()), floor) for k in ga}
        print(backbone, "loss", la, lb, "worst gradients", sorted(errs.items(), key=lambda kv: -kv[1])[:3])
        assert max(errs.values()) <= 3e-2, max(errs.items(), key=lambda kv: kv[1])
        for net in (ref, our):
            torch.optim.Adam(net.parameters(), lr=1e-3).step()
        # Adam's first step is lr sign(g): where a gradient is at rounding level the routes step differently, so the original's stepped
        # weights are written into ours in place, and the next losses must agree: the tiles follow in-place updates of weights and biases.
        with torch.no_grad():
            for pa, pb in zip(ref.parameters(), our.parameters()):
                pb.copy_(pa)
        la2, _ = step(ref)
        lb2, _ = step(our)
        assert la2 != la and abs(la2 - lb2) <= 1e-3 * abs(la2), (la2, lb2)
        pu = importlib.import_module("models.backbone.pointnet2.pytorch_utils")
        for net in (ref, our):
            pu.BNMomentumScheduler(net, bn_lambda=lambda e: 0.5)
        assert our.vgen.bn1.momentum == 0.5 and our.pnet.bn2.momentum == 0.5
        before = our.vgen.bn1.running_mean.clone()
        step(ref)
        step(our)
        rb = ref.vgen.bn1
        assert not torch.equal(before, our.vgen.bn1.running_mean)
        assert (our.vgen.bn1.running_mean - rb.running_mean).abs().max() <= 1e-4 * rb.running_mean.abs().max() + 1e-6
        assert int(our.vgen.bn1.num_batches_tracked) == int(rb.num_batches_tracked) == 3
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        # torch's and cv2's own modules imported on the way stay: neither extension survives a second import in one process (torch
        # registers its operator libraries twice, cv2's bindings come back incomplete)
        for k in [k for k in sys.modules if k not in saved and k.partition(".")[0] not in ("torch", "cv2")]:
            del sys.modules[k]
        sys.modules.update(saved)
