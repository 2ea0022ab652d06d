"""PointnetSAModuleVotes / PointnetFPModule on the library (pointcontrast_b200/pointnet2_modules.py, csrc/pointnet2_mlp.cu, DESIGN.md 8f-16)
against the fp64 oracle (oracle/pointnet2_mlp_cpu.py) at the configurations VoteNet runs, in training and eval mode:
  * outputs within 1e-4 of fp64 relative to their largest magnitude; the pooled slots agree with fp64's choice except within rounding;
  * gradients of features, xyz and every parameter within the DESIGN.md section 5 bound (norm-relative, with the library's own pooled
    slots replayed in the oracle: a choice within rounding distance is a coin flip in any precision), running statistics and
    num_batches_tracked;
  * two calls give the same bits;
  * the new kernels bit-exact on exactly representable operands; the selection rule; weights updated in place between two calls.
SA1 runs at B = 2 (the fp64 oracle of 1 M grouped rows per scene batch of 8 does not fit the check's host memory); the others at B = 8."""
import copy

import numpy as np
import pytest
import torch

from oracle import pointnet2_mlp_cpu as PM

pytestmark = pytest.mark.gpu
D = torch.float64

# name: (B, N, C, npoint, nsample, radius, mlp, given inds)
SA = {
    "sa1_sunrgbd": (2, 20000, 1, 2048, 64, 0.2, [1, 64, 64, 128], False),
    "sa1_scannet": (2, 40000, 1, 2048, 64, 0.2, [1, 64, 64, 128], False),
    "sa1_no_height": (2, 20000, 0, 2048, 64, 0.2, [0, 64, 64, 128], False),
    "sa2": (8, 2048, 128, 1024, 32, 0.4, [128, 128, 128, 256], False),
    "sa3": (8, 1024, 256, 512, 16, 0.8, [256, 128, 128, 256], False),
    "sa4": (8, 512, 256, 256, 16, 1.2, [256, 128, 128, 256], False),
    "vote_fps": (8, 1024, 256, 256, 16, 0.3, [256, 128, 128, 128], False),
    "vote_inds": (8, 1024, 256, 256, 16, 0.3, [256, 128, 128, 128], True),
}
# DESIGN.md section 5: norm-relative bound of every gradient.  The operand formats alone give ~1e-5 (measured on an H100); the rest of
# the margin is for ReLU decisions within rounding distance of zero, which the oracle does not replay: each one moves every upstream
# gradient by about 1 / sqrt(rows x channels) of its norm (3e-4 at SA3's 65 536 x 128).
GRAD_TOL = 5e-3


def room(seed, B, N):
    rng = np.random.default_rng(seed)
    p = rng.random((B, N, 3)) * np.array([6.0, 6.0, 2.5]) - np.array([3.0, 3.0, 0.5])
    return torch.from_numpy(p.astype(np.float32))


def feats(seed, *shape):
    return torch.from_numpy(np.abs(np.random.default_rng(seed).standard_normal(shape)).astype(np.float32))


def perturb_bn(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(torch.randn(m.num_features, generator=g))          # about half the channels pool minima
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)


def max_rel(a, b):
    return float((a.double().cpu() - b.detach()).abs().max() / b.detach().abs().max())


def norm_rel(a, b):
    return float((a.double().cpu() - b.detach()).norm() / b.detach().norm())


@pytest.fixture(scope="module")
def M():
    from pointcontrast_b200 import pointnet2_modules
    return pointnet2_modules


class _I32:
    def __init__(self, p, n, C):
        self.__cuda_array_interface__ = {"shape": (n, C), "strides": (4 * C, 4), "typestr": "<i4", "data": (p, False), "version": 2}


class _CaptureSel:
    """Stands in for the module's `lib` and copies the slots [B npoint, C] each pcb_sa_pool call selects (the oracle replays them)."""

    def __init__(self, lib):
        self.lib, self.sel = lib, None

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if name != "pcb_sa_pool":
            return f

        def pool(*a):
            rc = f(*a)
            self.sel = torch.as_tensor(_I32(a[9], a[2], a[4]), device="cuda").clone()
            return rc
        return pool


def _sa_run(M, mod, xyz, f, inds, train, gw, gx, monkeypatch):
    cap = _CaptureSel(M.lib)
    monkeypatch.setattr(M, "lib", cap)
    mod.train(train)
    x = xyz.cuda().requires_grad_(train)
    ff = f.cuda().requires_grad_(train) if f is not None else None
    with torch.set_grad_enabled(train):
        new_xyz, nf, out_inds = mod(x, ff, inds)
        if train:
            ((nf * gw.cuda()).sum() + (new_xyz * gx.cuda()).sum()).backward()
    monkeypatch.setattr(M, "lib", cap.lib)
    grads = [x.grad, ff.grad if ff is not None else None] + [p.grad for p in mod.parameters()] if train else []
    return new_xyz.detach(), nf.detach(), out_inds, grads, cap.sel


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("name", list(SA))
def test_sa_matches_oracle(M, name, train, monkeypatch):
    from pointcontrast_b200 import pointnet2
    B, N, C, npoint, S, radius, mlp, given = SA[name]
    torch.manual_seed(0)
    mod = M.PointnetSAModuleVotes(npoint=npoint, radius=radius, nsample=S, mlp=list(mlp), use_xyz=True, normalize_xyz=True)
    perturb_bn(mod, 1)
    mod = mod.cuda()
    twin = copy.deepcopy(mod)
    layers = PM.layer_params(mod.mlp_module, "")
    xyz, f = room(N, B, N), (feats(N + 1, B, C, N) if C else None)
    inds = torch.randint(0, N, (B, npoint), generator=torch.Generator().manual_seed(2), dtype=torch.int32).cuda() if given else None
    CL = mlp[-1]
    gw = torch.randn(B, CL, npoint, generator=torch.Generator().manual_seed(3))
    gx = torch.randn(B, npoint, 3, generator=torch.Generator().manual_seed(4))
    stats0 = {k: v.clone() for k, v in mod.state_dict().items()}
    new_xyz, nf, out_inds, grads, sel = _sa_run(M, mod, xyz, f, inds, train, gw, gx, monkeypatch)
    if not train:                                                                        # eval: the running statistics are left alone
        assert all(torch.equal(v, stats0[k]) for k, v in mod.state_dict().items())
    again = _sa_run(M, twin, xyz, f, inds, train, gw, gx, monkeypatch)                                  # two calls: the same bits
    assert torch.equal(nf, again[1]) and torch.equal(sel, again[4])
    assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(grads, again[3]))
    if given:
        assert out_inds is inds
    else:
        assert torch.equal(out_inds, pointnet2.ext.furthest_point_sampling(xyz.cuda(), npoint))
    idx = pointnet2.ext.ball_query(new_xyz, xyz.cuda(), radius, S).cpu()
    xo = xyz.double().requires_grad_()
    fo = f.double().requires_grad_() if C else None
    sel = sel.view(B, npoint, CL).cpu()
    nx, pooled, _, zs = PM.sa_forward(xo, fo, out_inds.cpu(), idx, layers, radius, True, train, sel=sel)
    own = torch.argmax(torch.where(layers[-1]["weight"].detach() >= 0, zs[-1].detach(), -zs[-1].detach()), dim=2)
    differ = float((own != sel).double().mean())
    assert differ < 1e-3, differ                                                          # only near-ties choose differently
    assert torch.equal(new_xyz.cpu().double(), nx.detach())
    err = max_rel(nf.transpose(1, 2), pooled)
    assert err < 1e-4, err
    if not train:
        return
    ((pooled.transpose(1, 2) * gw.double()).sum() + (nx * gx.double()).sum()).backward()
    want = [xo.grad, fo.grad if C else None] + [p[k].grad for p in layers for k in ("W", "weight", "bias")]
    errs = {}
    for i, (a, b) in enumerate(zip(grads, want)):
        if b is not None:
            errs[i] = norm_rel(a.reshape(b.shape), b)
    print(name, "feature err", err, "slots differing", differ, "grad errs", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < GRAD_TOL, errs
    for (conv, bn), p in zip(M._layers(mod.mlp_module), layers):
        assert max_rel(bn.running_mean, p["running_mean"]) < 1e-4 and max_rel(bn.running_var, p["running_var"]) < 1e-4
        assert int(bn.num_batches_tracked) == 1


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("B,n,m", [(8, 512, 256), (8, 1024, 512)])
def test_fp_matches_oracle(M, B, n, m, train):
    from pointcontrast_b200 import pointnet2
    torch.manual_seed(0)
    mod = M.PointnetFPModule(mlp=[512, 256, 256])
    perturb_bn(mod, 5)
    mod = mod.cuda().train(train)
    layers = PM.layer_params(mod.mlp, "")
    unknown, known = room(n, B, n).cuda(), room(m + 1, B, m).cuda()
    uf, kf = feats(6, B, 256, n).cuda().requires_grad_(train), feats(7, B, 256, m).cuda().requires_grad_(train)
    gw = torch.randn(B, 256, n, generator=torch.Generator().manual_seed(8))
    with torch.set_grad_enabled(train):
        out = mod(unknown, known, uf, kf)
        if train:
            (out * gw.cuda()).sum().backward()
    dist2, idx = pointnet2.ext.three_nn(unknown, known)
    recip = 1.0 / (torch.sqrt(dist2) + 1e-8)
    w = (recip / recip.sum(2, keepdim=True)).cpu()
    kfo, ufo = kf.detach().double().cpu().requires_grad_(), uf.detach().double().cpu().requires_grad_()
    o = PM.fp_forward(kfo, ufo, idx.cpu(), w, layers, train)
    err = max_rel(out.detach().transpose(1, 2), o)
    assert err < 1e-4, err
    if train:
        (o.transpose(1, 2) * gw.double()).sum().backward()
        errs = [norm_rel(kf.grad, kfo.grad), norm_rel(uf.grad, ufo.grad)] + \
            [norm_rel(t.grad.reshape(p[k].shape), p[k].grad) for t, (p, k) in zip(mod.parameters(), [(p, k) for p in layers
                                                                                                     for k in ("W", "weight", "bias")])]
        print("fp", n, m, "err", err, "grad errs", [f"{e:.2e}" for e in errs])
        assert max(errs) < GRAD_TOL, errs


def test_kernels_exact_on_representable_operands():
    """pcb_sa_layer0 and pcb_sa_pool on small integers and power-of-two weights and radius: every value exact in fp32 -> bit-exact."""
    from pointcontrast_b200 import _lib
    from pointcontrast_b200._lib import check, lib, ptr, stream
    rng = np.random.default_rng(9)
    B, N, npoint, S, C0 = 2, 50, 6, 8, 64
    xyz = torch.from_numpy(rng.integers(-8, 8, (B, N, 3)).astype(np.float32)).cuda()
    inds = torch.from_numpy(rng.integers(0, N, (B, npoint)).astype(np.int32))
    new_xyz = xyz[torch.arange(B)[:, None], inds.long().cuda()].contiguous()
    idx = torch.from_numpy(rng.integers(0, N, (B, npoint, S)).astype(np.int32))
    idx[:, :, S // 2:] = idx[:, :, :1]                                              # padded duplicates
    idx = idx.cuda()
    P = torch.from_numpy(rng.integers(-16, 16, (B * N, C0)).astype(np.float32)).cuda()
    wx = torch.from_numpy((2.0 ** rng.integers(-3, 3, (3, C0)) * rng.choice([-1, 1], (3, C0))).astype(np.float32)).cuda()
    R = B * npoint * S
    rel, gidx, z = torch.empty(R, 3, device="cuda"), torch.empty(R, dtype=torch.int32, device="cuda"), torch.empty(R, C0, device="cuda")
    check(lib.pcb_sa_layer0(ptr(xyz), ptr(new_xyz), ptr(idx), B, N, npoint, S, 0.5, ptr(P), C0, ptr(wx), C0, ptr(rel), ptr(gidx), ptr(z), C0,
                            stream()))
    j = idx.long().view(B, -1).cpu()
    x64 = xyz.double().cpu()
    want_rel = ((x64[torch.arange(B)[:, None], j].view(B, npoint, S, 3) - new_xyz.double().cpu()[:, :, None]) / 0.5).view(R, 3)
    gj = (j + torch.arange(B)[:, None] * N).view(-1)
    want_z = P.double().cpu()[gj] + want_rel @ wx.double().cpu()
    assert torch.equal(rel.double().cpu(), want_rel) and torch.equal(z.double().cpu(), want_z) and torch.equal(gidx.long().cpu(), gj)
    check(lib.pcb_sa_layer0(ptr(xyz), ptr(new_xyz), ptr(idx), B, N, npoint, S, 0.5, None, 0, ptr(wx), C0, ptr(rel), ptr(gidx), ptr(z), C0,
                            stream()))                                                  # no features: P == NULL
    assert torch.equal(z.double().cpu(), want_rel @ wx.double().cpu())
    # the xyz rows: grel / radius per row, then each centre's given gradient minus its rows' sum in ascending slot order
    grel = torch.from_numpy(rng.integers(-8, 8, (R, 3)).astype(np.float32)).cuda()
    dn = torch.from_numpy(rng.integers(-8, 8, (B * npoint, 3)).astype(np.float32)).cuda()
    rows = torch.empty(R + B * npoint, 3, device="cuda")
    check(lib.pcb_sa_xyz_rows(ptr(grel), ptr(dn), B * npoint, S, 0.5, ptr(rows), stream()))
    g64 = grel.double().cpu() / 0.5
    assert torch.equal(rows[:R].double().cpu(), g64)
    assert torch.equal(rows[R:].double().cpu(), dn.double().cpu() - g64.view(B * npoint, S, 3).sum(1))
    # the pool: integer z with ties, gamma of both signs, power-of-two invstd
    Mc, C = B * npoint, 64
    zz = torch.from_numpy(rng.integers(-4, 4, (Mc * S, C)).astype(np.float32)).cuda()
    gamma = torch.from_numpy(rng.choice([-2.0, -0.5, 0.0, 0.5, 1.0], C).astype(np.float32)).cuda()
    beta = torch.from_numpy(rng.integers(-2, 3, C).astype(np.float32)).cuda()
    mean = torch.from_numpy(rng.integers(-2, 2, C).astype(np.float32)).cuda()
    invstd = torch.full((C,), 0.25, device="cuda")
    sel, out = torch.empty(Mc, C, dtype=torch.int32, device="cuda"), torch.empty(Mc, C, device="cuda")
    check(lib.pcb_sa_pool(ptr(zz), C, Mc, S, C, ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(sel), ptr(out), C, stream()))
    z3 = zz.double().cpu().view(Mc, S, C)
    y = torch.relu((z3 - mean.double().cpu()) * 0.25 * gamma.double().cpu() + beta.double().cpu())
    assert torch.equal(out.double().cpu(), y.max(1).values)
    key = torch.where(gamma.cpu() >= 0, z3, -z3)
    assert torch.equal(sel.long().cpu(), torch.argmax(key, 1))                           # first extreme: the smallest slot
    assert (gamma < 0).any() and (gamma == 0).any()
    # its gradient: the selected slot only, where the pooled value is positive
    g = torch.from_numpy(rng.integers(-3, 4, (Mc, C)).astype(np.float32)).cuda()
    dY = torch.empty(Mc * S, C, device="cuda")
    check(lib.pcb_sa_pool_grad(ptr(g), C, ptr(sel), ptr(out), C, Mc, S, C, ptr(dY), stream()))
    want = torch.zeros(Mc, S, C)
    want.scatter_(1, sel.long().cpu()[:, None], (g * (out > 0)).cpu()[:, None])
    assert torch.equal(dY.cpu().view(Mc, S, C), want)
    assert _lib.ERR_ARG == lib.pcb_sa_pool(ptr(zz), C, Mc, 0, C, ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(sel), ptr(out), C,
                                           stream())


def test_in_place_weight_update_between_calls(M):
    """An optimiser steps the weights in place: the next forward uses the new weights (the weight tiles follow the version counter)."""
    from pointcontrast_b200 import pointnet2
    B, N, C, npoint, S, radius, mlp, _ = SA["sa3"]
    torch.manual_seed(0)
    mod = M.PointnetSAModuleVotes(npoint=npoint, radius=radius, nsample=S, mlp=list(mlp), normalize_xyz=True).cuda().eval()
    xyz, f = room(1, B, N), feats(2, B, C, N)
    with torch.no_grad():
        _, before, inds = mod(xyz.cuda(), f.cuda())
        opt = torch.optim.Adam(mod.parameters(), lr=0.05)
        for p in mod.parameters():
            p.grad = torch.randn_like(p)
        opt.step()
        new_xyz, after, _ = mod(xyz.cuda(), f.cuda())
    assert not torch.equal(before, after)
    idx = pointnet2.ext.ball_query(new_xyz, xyz.cuda(), radius, S).cpu()
    _, pooled, _, _ = PM.sa_forward(xyz.double(), f.double(), inds.cpu(), idx, PM.layer_params(mod.mlp_module, ""), radius, True, False)
    assert max_rel(after.transpose(1, 2), pooled) < 1e-4


def test_eval_mode_is_forward_only(M):
    mod = M.PointnetSAModuleVotes(npoint=16, radius=0.3, nsample=8, mlp=[0, 32, 32, 32]).cuda().eval()
    with pytest.raises(NotImplementedError, match="no_grad"):
        mod(room(0, 1, 100).cuda())


# ------------------------------------------------------------------------------------------------ drop-in VoteNet
def _votenet(ours):
    """The staged, unmodified models/votenet.py on this library's `me` and `pointnet2`, with (ours) or without pointnet2_modules.install(),
    and det_loss.install()."""
    import importlib
    import sys
    from oracle import detection_ref, det_loss_ref
    if not (detection_ref.available() and det_loss_ref.available()):
        pytest.skip("oracle/_ref/votenet/models not staged (the original repository is absent)")
    from oracle import det_eval_ref
    det_eval_ref.load()                          # stand-ins for the original's plotting and PLY imports (dump_helper, pc_util)
    from pointcontrast_b200 import det_loss, me, pointnet2, pointnet2_modules
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k in (
            "pointnet2_utils", "pointnet2_modules", "pytorch_utils", "backbone_module", "proposal_module", "voting_module", "loss_helper",
            "dump_helper")]:
        del sys.modules[k]
    me.install()
    pointnet2.install()
    if detection_ref.ROOT not in sys.path:
        sys.path.insert(0, detection_ref.ROOT)
    if ours:
        pointnet2_modules.install()
        assert sys.modules["pointnet2_modules"] is pointnet2_modules
    det_loss.install()
    votenet = importlib.import_module("models.votenet")
    bm = importlib.import_module("models.backbone_module")
    assert (bm.PointnetSAModuleVotes is pointnet2_modules.PointnetSAModuleVotes) == ours
    return votenet


@pytest.mark.parametrize("backbone", ["pointnet2"])
def test_votenet_drop_in(backbone):
    """One Adam step of the unmodified VoteNet (backbone='pointnet2') after
    pointnet2_modules.install(), against the same model on pointnet2.install() alone (torch's modules, TF32 off), same weights: loss and
    every gradient, checkpoints loading both ways, the step's effect on the next loss, and BNMomentumScheduler's momentum."""
    import sys
    from pointcontrast_b200 import det_loss, detection, pointnet2_modules, synth
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
        our.load_state_dict(ref.state_dict())                                   # an original checkpoint loads into ours ...
        ref.load_state_dict(our.state_dict())                                   # ... and back
        n_ours = sum(isinstance(m, pointnet2_modules.PointnetSAModuleVotes) for m in our.modules())
        assert n_ours == (5 if backbone == "pointnet2" else 1)
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
        # every gradient is measured against at least 1e-4 of the largest one.  The original route's fp32 cuDNN BatchNorm backward is
        # itself ~1e-3 from fp64 at SA1's size (tests/test_gpu_pointnet2.py), and ReLU / pool decisions within rounding may differ.
        floor = 1e-4 * max(float(g.norm()) for g in ga.values())
        errs = {k: float((ga[k] - gb[k]).norm()) / max(float(ga[k].norm()), floor) for k in ga}
        print(backbone, "loss", la, lb, "worst gradients", sorted(errs.items(), key=lambda kv: -kv[1])[:3])
        assert max(errs.values()) <= 3e-2, max(errs.items(), key=lambda kv: kv[1])
        for net in (ref, our):
            torch.optim.Adam(net.parameters(), lr=1e-3).step()
        # Adam's first step is lr sign(g): wherever a gradient is at rounding level (a bias in front of a BatchNorm) the two routes step
        # differently.  So the original's stepped weights are written into ours in place as well, and the next losses must agree: the
        # weight tiles follow the in-place updates.
        with torch.no_grad():
            for pa, pb in zip(ref.parameters(), our.parameters()):
                pb.copy_(pa)
        la2, _ = step(ref)
        lb2, _ = step(our)
        assert la2 != la and abs(la2 - lb2) <= 1e-3 * abs(la2), (la2, lb2)
        # BNMomentumScheduler (the original's, an isinstance walk over nn.BatchNorm{1,2,3}d) reaches our BatchNorm2d modules
        import importlib
        pu = importlib.import_module("models.backbone.pointnet2.pytorch_utils")
        for net in (ref, our):
            pu.BNMomentumScheduler(net, bn_lambda=lambda e: 0.5)
        sa = [m for m in our.modules() if isinstance(m, pointnet2_modules.PointnetSAModuleVotes)][0]
        bn = sa.mlp_module.layer0.bn.bn
        assert bn.momentum == 0.5
        before = bn.running_mean.clone()
        step(ref)
        step(our)
        rb = [m for m in ref.modules() if type(m).__name__ == "PointnetSAModuleVotes"][0].mlp_module.layer0.bn.bn
        assert not torch.equal(before, bn.running_mean)
        assert (bn.running_mean - rb.running_mean).abs().max() <= 1e-4 * rb.running_mean.abs().max() + 1e-6
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        for k in [k for k in sys.modules if k not in saved]:
            del sys.modules[k]
        sys.modules.update(saved)
