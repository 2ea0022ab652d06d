"""Host checks of the PointNet++ oracle (oracle/pointnet2_cpu.py) against independent computations, and of the argument checks of the
pcb_* PointNet++ entry points, which reject bad input before touching a device."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import pointnet2_cpu as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOTENET = os.path.join(ROOT, "oracle", "_ref", "votenet", "pointnet2")


def reference_modules(install):
    """Fresh imports of the staged, unmodified pointnet2_utils / pointnet2_modules bound to the `_ext` that `install()` registers
    (pointnet2_utils binds `pointnet2._ext` at import time, so each backend needs its own import)."""
    if not os.path.isfile(os.path.join(VOTENET, "pointnet2_modules.py")):
        pytest.skip("oracle/_ref/votenet not staged (the original repository is absent)")
    for m in ("pointnet2_utils", "pointnet2_modules", "pytorch_utils"):
        sys.modules.pop(m, None)
    install()
    if VOTENET not in sys.path:
        sys.path.insert(0, VOTENET)
    return importlib.import_module("pointnet2_utils"), importlib.import_module("pointnet2_modules")


def scene(rng, B, N, scale=3.0):
    return torch.from_numpy((rng.random((B, N, 3)) * scale - scale / 2).astype(np.float32))


def test_ball_query_matches_kdtree():
    rng = np.random.default_rng(0)
    xyz = scene(rng, 2, 3000)
    new = xyz[:, rng.choice(3000, 200, replace=False)].contiguous()
    for radius, S in ((0.2, 16), (0.4, 64)):
        idx = O.ball_query(new, xyz, radius, S).numpy()
        r2 = np.float32(radius) * np.float32(radius)
        for b in range(2):
            p, q = xyz[b].numpy(), new[b].numpy()
            for m, nb in enumerate(cKDTree(p.astype(np.float64)).query_ball_point(q.astype(np.float64), radius * 1.001)):
                d = q[m] - p[sorted(nb)]
                hits = [k for k, e in zip(sorted(nb), d) if (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2] < r2]   # the same fp32 predicate
                want = hits[:S] + [hits[0] if hits else 0] * (S - min(S, len(hits)))
                assert idx[b, m].tolist() == want


def test_three_nn_matches_kdtree():
    rng = np.random.default_rng(1)
    known, unknown = scene(rng, 2, 400), scene(rng, 2, 900)
    dist2, idx = O.three_nn(unknown, known)
    for b in range(2):
        d, i = cKDTree(known[b].numpy().astype(np.float64)).query(unknown[b].numpy().astype(np.float64), k=3)
        assert (idx[b].numpy() == i).all()
        np.testing.assert_allclose(dist2[b].numpy(), d ** 2, rtol=1e-5, atol=1e-7)
    d2, i2 = O.three_nn(unknown[:, :10].contiguous(), known[:, :2].contiguous())      # m < 3: inf / 0 in the missing slots
    assert torch.isinf(d2[..., 2]).all() and (i2[..., 2] == 0).all() and torch.isfinite(d2[..., :2]).all()


def test_fps_picks_the_furthest_point_every_step():
    rng = np.random.default_rng(2)
    xyz = scene(rng, 2, 1500)
    xyz[0, 7] = 0.0                     # inside the origin skip radius: never chosen
    xyz[0, 8] = 0.01
    idx = O.furthest_point_sampling(xyz, 100).numpy()
    for b in range(2):
        p = xyz[b].numpy().astype(np.float64)
        cand = (p ** 2).sum(1) > 1e-3
        chosen = [0]
        mind = np.full(len(p), np.inf)
        for j in range(1, 100):
            mind = np.minimum(mind, ((p - p[chosen[-1]]) ** 2).sum(1))
            k = int(idx[b, j])
            assert cand[k] and k not in chosen
            assert mind[k] >= mind[cand].max() * (1 - 1e-5)      # maximises the min-distance (fp64 recomputation, fp32 rounding)
            chosen.append(k)
        assert idx[b, 0] == 0
    assert 7 not in idx[0] and 8 not in idx[0]


def test_fps_ties_smallest_index_and_no_candidates():
    xyz = torch.tensor([[[1., 0, 0], [2., 0, 0], [0., 0, 0], [3., 0, 0], [-1., 0, 0]]])      # after 0, points 3 and 4 tie at d = 4
    assert O.furthest_point_sampling(xyz, 3).tolist() == [[0, 3, 4]]
    dup = torch.tensor([[[1., 0, 0], [5., 0, 0], [5., 0, 0], [5., 0, 0]]])                     # then every running distance is 0
    assert O.furthest_point_sampling(dup, 4).tolist() == [[0, 1, 0, 0]]
    assert O.furthest_point_sampling(torch.zeros(1, 4, 3), 3).tolist() == [[0, 0, 0]]         # no candidate at all: index 0


def test_backward_passes_match_autograd():
    rng = np.random.default_rng(3)
    B, C, N, M, S = 2, 5, 60, 17, 6
    f = torch.from_numpy(rng.standard_normal((B, C, N))).requires_grad_()
    idx2 = torch.from_numpy(rng.integers(0, N, (B, M)).astype(np.int32))
    idx3 = torch.from_numpy(rng.integers(0, N, (B, M, S)).astype(np.int32))
    w = torch.from_numpy(rng.random((B, M, 3)))
    i3 = torch.from_numpy(rng.integers(0, N, (B, M, 3)).astype(np.int32))
    g2, g3, gi = (torch.from_numpy(rng.standard_normal(s)) for s in ((B, C, M), (B, C, M, S), (B, C, M)))
    ix = lambda i: i.long().reshape(B, 1, -1).expand(B, C, -1)                                       # noqa: E731
    (a,) = torch.autograd.grad((torch.gather(f, 2, ix(idx2)) * g2).sum(), f)
    assert torch.allclose(O.gather_points_grad(g2, idx2, N), a, rtol=1e-12, atol=1e-12)
    (a,) = torch.autograd.grad((torch.gather(f, 2, ix(idx3)).reshape(B, C, M, S) * g3).sum(), f)
    assert torch.allclose(O.group_points_grad(g3, idx3, N), a, rtol=1e-12, atol=1e-12)
    interp = (torch.gather(f, 2, ix(i3)).reshape(B, C, M, 3) * w[:, None]).sum(-1)
    (a,) = torch.autograd.grad((interp * gi).sum(), f)
    assert torch.allclose(O.three_interpolate_grad(gi, i3, w, N), a, rtol=1e-12, atol=1e-12)
    fo = O.three_interpolate(f.detach().float(), i3, w.float())
    assert torch.allclose(fo.double(), interp.detach(), rtol=1e-5, atol=1e-6)


def test_pointnet2_argument_errors_do_not_need_a_gpu():
    from pointcontrast_b200 import _lib, pointnet2
    L = _lib.lib
    big = 1 << 31
    for rc in (L.pcb_furthest_point_sampling(None, 1, 10, 0, None, None, 0, None),            # npoint < 1
               L.pcb_furthest_point_sampling(None, 1, big, 4, None, None, 0, None),            # N >= 2^31
               L.pcb_ball_query(None, None, 1, 4, 5, 0.1, 0, None, None),                      # nsample < 1
               L.pcb_ball_query(None, None, 1, 4, 5, 0.0, 4, None, None),                      # radius <= 0
               L.pcb_ball_query(None, None, 1, 4, 5, -1.0, 4, None, None),
               L.pcb_three_nn(None, None, 1, big, 3, None, None, None),
               L.pcb_gather_points(None, None, 1, 2, big, 4, None, None),
               L.pcb_three_interpolate(None, None, None, big, 2, 3, 4, None, None),
               L.pcb_gather_points_grad(None, None, 1, 2, 3, big, None, None, 0, None),
               L.pcb_three_interpolate_grad(None, None, None, 1, 2, 3, 4, None, None, 0, None)):    # no workspace
        assert rc == 2 and b"bad argument" in L.pcb_last_error()
    assert L.pcb_points_grad_ws_bytes(8, 20000, 2048 * 64) > 4 * 8 * 2048 * 64 * 4
    assert L.pcb_furthest_point_sampling_ws_bytes(8, 40000) == 0           # held on chip
    assert L.pcb_furthest_point_sampling_ws_bytes(1, 200000) == 200000 * 4
    with pytest.raises(_lib.PcbError):
        pointnet2.ext.furthest_point_sampling(torch.zeros(1, 8, 3), 2)
    with pytest.raises(_lib.PcbError):
        pointnet2.ext.ball_query(torch.zeros(1, 2, 3), torch.zeros(1, 8, 3), 0.1, 4)


def test_install_registers_the_ext_module():
    from pointcontrast_b200 import pointnet2
    saved = {k: sys.modules.get(k) for k in ("pointnet2", "pointnet2._ext")}
    try:
        ext = pointnet2.install()
        import pointnet2._ext as e  # noqa: F401
        assert sys.modules["pointnet2._ext"] is ext and all(hasattr(ext, f) for f in pointnet2.EXT_FUNCTIONS)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_reference_modules_run_on_the_oracle():
    """The original's unmodified PointnetSAModuleVotes and PointnetFPModule, forward and backward, on the oracle `_ext` (CPU)."""
    saved = {k: sys.modules.get(k) for k in ("pointnet2", "pointnet2._ext")}
    try:
        utils, mods = reference_modules(O.install)
        torch.manual_seed(0)
        rng = np.random.default_rng(4)
        xyz = scene(rng, 2, 600).double()
        feats = torch.from_numpy(rng.standard_normal((2, 3, 600))).requires_grad_()
        sa = mods.PointnetSAModuleVotes(npoint=64, radius=0.4, nsample=16, mlp=[3, 16, 32], use_xyz=True, normalize_xyz=True).double()
        new_xyz, new_f, inds = sa(xyz, feats)
        assert new_xyz.shape == (2, 64, 3) and new_f.shape == (2, 32, 64) and inds.shape == (2, 64)
        assert torch.equal(new_xyz[0], xyz[0, inds[0].long()])
        fp = mods.PointnetFPModule(mlp=[32 + 3, 16]).double()
        up = fp(xyz, new_xyz, feats, new_f)
        assert up.shape == (2, 16, 600)
        (up.sum() + new_f.sum()).backward()
        assert feats.grad is not None and torch.isfinite(feats.grad).all() and feats.grad.abs().sum() > 0
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
