"""The fp64 shared-MLP oracle (oracle/pointnet2_mlp_cpu.py) against the staged, unmodified original PointnetSAModuleVotes /
PointnetFPModule run in fp64 on oracle.pointnet2_cpu: forward, the gradients of features, xyz and every parameter, the running statistics
and num_batches_tracked, in training and eval mode (skipped where the original is absent).  The xyz gradient is autograd's of the
oracle's explicit formula: the original cannot take one on the oracle `_ext`.  Also the selection rule on its own."""
import numpy as np
import pytest
import torch

from oracle import pointnet2_cpu as O
from oracle import pointnet2_mlp_cpu as PM
from tests.test_oracle_pointnet2 import reference_modules

D = torch.float64


def _scene(seed, B, N, C):
    rng = np.random.default_rng(seed)
    xyz = torch.from_numpy((rng.random((B, N, 3)) * 2 - 1).astype(np.float32))
    f = torch.from_numpy(rng.standard_normal((B, C, N))) if C else None
    return xyz, f


def _perturb_bn(mod, seed):
    """Non-trivial gamma (some negative), beta and running statistics, so every branch of the selection and eval mode is exercised."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(torch.randn(m.num_features, generator=g))
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("C,normalize", [(1, True), (5, False)])
def test_sa_oracle_matches_the_original(train, C, normalize):
    _, ref = reference_modules(O.install)
    torch.manual_seed(0)
    sa = ref.PointnetSAModuleVotes(npoint=24, radius=0.5, nsample=8, mlp=[C, 16, 16, 32], use_xyz=True, normalize_xyz=normalize).double()
    _perturb_bn(sa, 1)
    sa.train(train)
    layers = PM.layer_params(sa.mlp_module, "")
    xyz, f = _scene(2, 2, 300, C)
    x = xyz.clone()          # the original's in-place grouped_xyz update forbids an xyz gradient on the oracle `_ext` (a view)
    ff = f.clone().requires_grad_() if C else None
    new_xyz, new_f, inds = sa(x, ff)
    xo = xyz.double().requires_grad_()
    fo = f.clone().requires_grad_() if C else None
    idx = O.ball_query(new_xyz.detach().float(), xyz, 0.5, 8)
    nx, pooled, sel, _ = PM.sa_forward(xo, fo, inds, idx, layers, 0.5, normalize, train)
    assert torch.allclose(nx, new_xyz.double(), rtol=0, atol=0)
    assert torch.allclose(pooled.transpose(1, 2), new_f, rtol=1e-12, atol=1e-12)
    gw = torch.randn(new_f.shape, dtype=D, generator=torch.Generator().manual_seed(4))
    gx = torch.randn(new_xyz.shape, dtype=torch.float32, generator=torch.Generator().manual_seed(5))
    (new_f * gw).sum().backward()
    (pooled.transpose(1, 2) * gw).sum().backward()
    if C:
        assert torch.allclose(fo.grad, ff.grad, rtol=1e-10, atol=1e-12)
    for i, p in enumerate(layers):
        conv, bn = getattr(sa.mlp_module, f"layer{i}").conv, getattr(sa.mlp_module, f"layer{i}").bn.bn
        assert torch.allclose(p["W"].grad, conv.weight.grad.flatten(1), rtol=1e-9, atol=1e-10)
        assert torch.allclose(p["weight"].grad, bn.weight.grad, rtol=1e-9, atol=1e-10)
        assert torch.allclose(p["bias"].grad, bn.bias.grad, rtol=1e-9, atol=1e-10)
        assert torch.allclose(p["running_mean"], bn.running_mean, rtol=1e-12, atol=1e-14)
        assert torch.allclose(p["running_var"], bn.running_var, rtol=1e-12, atol=1e-14)
        assert int(bn.num_batches_tracked) == (1 if train else 0)


@pytest.mark.parametrize("train", [True, False])
def test_fp_oracle_matches_the_original(train):
    _, ref = reference_modules(O.install)
    torch.manual_seed(0)
    fp = ref.PointnetFPModule(mlp=[24 + 8, 16, 16]).double()
    _perturb_bn(fp, 2)
    fp.train(train)
    layers = PM.layer_params(fp.mlp, "")
    unknown, u_f = _scene(3, 2, 100, 8)
    known, k_f = _scene(4, 2, 30, 24)
    kf, uf = k_f.clone().requires_grad_(), u_f.clone().requires_grad_()
    out = fp(unknown, known, uf, kf)
    dist2, idx = O.three_nn(unknown, known)
    recip = 1.0 / (torch.sqrt(dist2) + 1e-8)
    w = recip / recip.sum(2, keepdim=True)
    kfo, ufo = k_f.clone().requires_grad_(), u_f.clone().requires_grad_()
    o = PM.fp_forward(kfo, ufo, idx, w, layers, train)
    assert torch.allclose(o.transpose(1, 2), out, rtol=1e-6, atol=1e-7)              # the original's weights are fp32
    gw = torch.randn(out.shape, dtype=D, generator=torch.Generator().manual_seed(6))
    (out * gw).sum().backward()
    (o.transpose(1, 2) * gw).sum().backward()
    assert torch.allclose(kfo.grad, kf.grad, rtol=1e-5, atol=1e-6)
    assert torch.allclose(ufo.grad, uf.grad, rtol=1e-5, atol=1e-6)


def test_selection_takes_minima_under_negative_gamma_and_the_first_of_equals():
    layers = [dict(W=torch.eye(3, dtype=D).requires_grad_(), weight=torch.tensor([1.0, -1.0, 0.0], dtype=D), bias=torch.zeros(3, dtype=D),
                   running_mean=torch.zeros(3, dtype=D), running_var=torch.ones(3, dtype=D))]
    xyz = torch.tensor([[[0.0, 0, 0], [1, -2, 5], [3, 1, 5], [1, -2, 5]]], dtype=D)
    idx = torch.tensor([[[1, 2, 3, 1]]])                                          # padded duplicate of sample 0 in slot 3
    _, pooled, sel, _ = PM.sa_forward(xyz, None, torch.tensor([[0]]), idx, layers, 1.0, False, False)
    assert sel.tolist() == [[[1, 0, 0]]]                    # max x; min y (gamma < 0); gamma == 0: every slot equal, the first
    assert torch.allclose(pooled.detach(), torch.tensor([[[3.0, 2.0, 0.0]]], dtype=D) / (1 + 1e-5) ** 0.5)
