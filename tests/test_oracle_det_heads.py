"""The fp64 heads oracle (oracle/det_heads_cpu.py) against the staged, unmodified original VotingModule and ProposalModule (its layers
and decode_scores after the vote aggregation) run in fp64 on the CPU: outputs, the gradients of the inputs and of every parameter, the
running statistics and num_batches_tracked, in training and eval mode (skipped where the original is absent)."""
import importlib

import numpy as np
import pytest
import torch

from oracle import det_heads_cpu as H
from oracle import pointnet2_cpu as O
from oracle import stage_ref
from tests.test_oracle_pointnet2 import reference_modules

D = torch.float64
DATASETS = {"scannet": (1, 18, 18), "sunrgbd": (12, 10, 10)}        # NH, NS, C


def _original(name):
    """A fresh import of the staged models/<name>.py, with the original's PointNet++ Python layer on the CPU oracle."""
    reference_modules(O.install)
    with stage_ref.installed({name: None}, path=[stage_ref.path("votenet", "models"), stage_ref.path("votenet", "pointnet2")]):
        return importlib.import_module(name)


def perturb_bn(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.copy_(torch.randn(m.num_features, generator=g, dtype=m.weight.dtype))
                m.bias.copy_(torch.randn(m.num_features, generator=g, dtype=m.weight.dtype) * 0.1)
                m.running_mean.copy_(torch.randn(m.num_features, generator=g, dtype=m.weight.dtype) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g, dtype=m.weight.dtype) + 0.5)


def _params(mod):
    return [mod.conv1.weight, mod.conv1.bias, mod.conv2.weight, mod.conv2.bias, mod.conv3.weight, mod.conv3.bias, mod.bn1.weight,
            mod.bn1.bias, mod.bn2.weight, mod.bn2.bias]


def _check_state(mod, p, train):
    for c in ("bn1", "bn2"):
        bn = getattr(mod, c)
        assert torch.allclose(p[c]["running_mean"], bn.running_mean, rtol=1e-12, atol=1e-14)
        assert torch.allclose(p[c]["running_var"], bn.running_var, rtol=1e-12, atol=1e-14)
        assert int(bn.num_batches_tracked) == (1 if train else 0)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("V", [1, 2])
def test_voting_oracle_matches_the_original(V, train):
    vm = _original("voting_module")
    torch.manual_seed(0)
    mod = vm.VotingModule(V, 64).double().train(train)
    perturb_bn(mod, 1)
    p = H.head_params(mod.state_dict())
    rng = np.random.default_rng(2)
    xyz = torch.from_numpy(rng.standard_normal((2, 40, 3)))
    f = torch.from_numpy(rng.standard_normal((2, 64, 40)))
    xa, fa, xo, fo = (t.clone().requires_grad_() for t in (xyz, f, xyz, f))
    vx, vf = mod(xa, fa)
    ox, of = H.voting(xo, fo, p, V, train)
    assert torch.allclose(vx, ox, rtol=1e-12, atol=1e-12) and torch.allclose(vf, of, rtol=1e-12, atol=1e-12)
    gx, gf = torch.randn(vx.shape, dtype=D), torch.randn(vf.shape, dtype=D)
    ((vx * gx).sum() + (vf * gf).sum()).backward()
    ((ox * gx).sum() + (of * gf).sum()).backward()
    assert torch.allclose(xa.grad, xo.grad, rtol=1e-10, atol=1e-12) and torch.allclose(fa.grad, fo.grad, rtol=1e-10, atol=1e-12)
    for a, b in zip(_params(mod), H.grads(p)):
        assert torch.allclose(a.grad.reshape(b.shape), b, rtol=1e-9, atol=1e-10)
    _check_state(mod, p, train)


class _Aggregation(torch.nn.Module):
    """Stands in for the vote aggregation: returns the given aggregated xyz, features and indices."""

    def __init__(self, xyz, features):
        super().__init__()
        self.out = (xyz, features, torch.zeros(xyz.shape[:2], dtype=torch.int32))

    def forward(self, *args):
        return self.out


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("dataset", list(DATASETS))
def test_proposal_oracle_matches_the_original(dataset, train, monkeypatch):
    pm = _original("proposal_module")
    NH, NS, C = DATASETS[dataset]
    ms = np.random.default_rng(3).uniform(0.3, 2.0, (NS, 3))
    torch.manual_seed(0)
    mod = pm.ProposalModule(C, NH, NS, ms, 24, "vote_fps").double().train(train)
    perturb_bn(mod, 4)
    p = H.head_params(mod.state_dict())
    rng = np.random.default_rng(5)
    agg = torch.from_numpy(rng.standard_normal((2, 24, 3)))
    f = torch.from_numpy(rng.standard_normal((2, 128, 24)))
    aa, fa, ao, fo = (t.clone().requires_grad_() for t in (agg, f, agg, f))
    mod.vote_aggregation = _Aggregation(aa, fa)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)       # decode_scores moves mean_size with .cuda()
    ep = mod(None, None, {})
    want = H.proposal(ao, fo, p, NH, NS, ms, train)
    loss_a, loss_o = 0, 0
    for i, k in enumerate(H.DECODE):
        assert ep[k].shape == want[k].shape, k
        assert torch.allclose(ep[k], want[k], rtol=1e-12, atol=1e-12), k
        g = torch.randn(want[k].shape, dtype=D, generator=torch.Generator().manual_seed(10 + i))
        loss_a = loss_a + (ep[k] * g).sum()
        loss_o = loss_o + (want[k] * g).sum()
    loss_a.backward()
    loss_o.backward()
    assert torch.allclose(aa.grad, ao.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(fa.grad, fo.grad, rtol=1e-10, atol=1e-12)
    for a, b in zip(_params(mod), H.grads(p)):
        assert torch.allclose(a.grad.reshape(b.shape), b, rtol=1e-9, atol=1e-10)
    _check_state(mod, p, train)
