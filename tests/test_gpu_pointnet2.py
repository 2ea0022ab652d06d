"""PointNet++ operators on the GPU (pointcontrast_b200/pointnet2.py, csrc/pointnet2.cu, DESIGN.md 8f-5):
  * every op against the CPU oracle (oracle/pointnet2_cpu.py) at VoteNet shapes and at edge cases: indices and forward values bit-exact,
    backward passes within 1e-6 of the fp64 oracle relative to the sum of |terms|, and bit-identical across two calls;
  * against the reference's own kernels, compiled for sm_90a by __graft_entry__.build() (oracle/_ref/pointnet2_ext; skipped where the
    original repository was absent at build time);
  * the original's unmodified PointnetSAModuleVotes / PointnetFPModule on this library after `pointnet2.install()`."""
import sys

import numpy as np
import pytest
import torch

from oracle import pointnet2_cpu as O
from oracle import pointnet2_ref
from tests.test_oracle_pointnet2 import reference_modules

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P():
    from pointcontrast_b200 import pointnet2
    return pointnet2.ext


@pytest.fixture(scope="module")
def REF():
    ref = pointnet2_ref.load()
    if ref is None:
        pytest.skip("oracle/_ref/pointnet2_ext not built (the original repository was absent at build time)")
    return ref


def room(seed, B, N):
    """Seeded continuous VoteNet-like input: points of a 6 m x 6 m x 2.5 m room around the camera (fp32, no exact duplicates)."""
    rng = np.random.default_rng(seed)
    p = rng.random((B, N, 3)) * np.array([6.0, 6.0, 2.5]) - np.array([3.0, 3.0, 0.5])
    return torch.from_numpy(p.astype(np.float32))


def feats(seed, *shape):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal(shape).astype(np.float32))


def check_grad(ours, oracle_fn, oracle_abs_fn, tol=1e-6):
    """|ours - fp64 oracle| <= tol * (sum of |terms| + tiny), elementwise."""
    want, scale = oracle_fn(), oracle_abs_fn()
    err = (ours.double().cpu() - want).abs()
    bad = err > tol * scale + 1e-30
    assert not bad.any(), f"{int(bad.sum())} elements off; worst {float((err / (scale + 1e-30)).max()):.3e}"


# ------------------------------------------------------------------------------------------------ against the oracle
FPS_CASES = [(8, 20000, 2048), (8, 40000, 2048), (8, 2048, 1024), (8, 1024, 512), (8, 512, 256)]


@pytest.mark.parametrize("B,N,npoint", FPS_CASES)
def test_fps_matches_oracle(P, B, N, npoint):
    xyz = room(N, B, N)
    got = P.furthest_point_sampling(xyz.cuda(), npoint).cpu()
    assert got.dtype == torch.int32 and torch.equal(got, O.furthest_point_sampling(xyz, npoint))


BQ_CASES = [(8, 20000, 2048, 0.2, 64), (8, 40000, 2048, 0.2, 64), (8, 2048, 1024, 0.4, 32), (8, 1024, 512, 0.8, 16), (8, 512, 256, 1.2, 16),
            (8, 1024, 256, 0.3, 16)]


@pytest.mark.parametrize("B,N,M,radius,S", BQ_CASES)
def test_ball_query_and_grouping_match_oracle(P, B, N, M, radius, S):
    xyz = room(N + 1, B, N)
    new = xyz[:, torch.from_numpy(np.random.default_rng(M).choice(N, M, replace=False))].contiguous()
    idx = P.ball_query(new.cuda(), xyz.cuda(), radius, S)
    want = O.ball_query(new, xyz, radius, S)
    assert idx.dtype == torch.int32 and torch.equal(idx.cpu(), want)
    C = 64 if N > 2048 else 128
    f = feats(1, B, C, N)
    g = P.group_points(f.cuda(), idx)
    assert torch.equal(g.cpu(), O.group_points(f, want))
    go = feats(2, B, C, M, S).cuda()
    d1, d2 = P.group_points_grad(go, idx, N), P.group_points_grad(go, idx, N)
    assert torch.equal(d1, d2)
    check_grad(d1, lambda: O.group_points_grad(go.cpu(), want, N), lambda: O.group_points_grad(go.cpu(), want, N, absolute=True))


@pytest.mark.parametrize("B,N,M,C", [(8, 20000, 2048, 3), (8, 40000, 2048, 3), (8, 2048, 1024, 128), (8, 20000, 256, 256)])
def test_gather_points_matches_oracle(P, B, N, M, C):
    f = feats(3, B, C, N)
    idx = torch.from_numpy(np.random.default_rng(4).integers(0, N, (B, M)).astype(np.int32))
    out = P.gather_points(f.cuda(), idx.cuda())
    assert torch.equal(out.cpu(), O.gather_points(f, idx))
    go = feats(5, B, C, M).cuda()
    d1, d2 = P.gather_points_grad(go, idx.cuda(), N), P.gather_points_grad(go, idx.cuda(), N)
    assert torch.equal(d1, d2)
    check_grad(d1, lambda: O.gather_points_grad(go.cpu(), idx, N), lambda: O.gather_points_grad(go.cpu(), idx, N, absolute=True))


@pytest.mark.parametrize("B,n,m,C", [(8, 512, 256, 256), (8, 1024, 512, 256), (2, 20000, 2048, 128)])
def test_three_nn_and_interpolate_match_oracle(P, B, n, m, C):
    unknown, known = room(n, B, n), room(m + 7, B, m)
    dist2, idx = P.three_nn(unknown.cuda(), known.cuda())
    wd, wi = O.three_nn(unknown, known)
    assert torch.equal(idx.cpu(), wi) and torch.equal(dist2.cpu(), wd)
    recip = 1.0 / (torch.sqrt(wd) + 1e-8)
    w = (recip / recip.sum(2, keepdim=True)).contiguous()
    f = feats(6, B, C, m)
    out = P.three_interpolate(f.cuda(), idx, w.cuda())
    assert torch.equal(out.cpu(), O.three_interpolate(f, wi, w))
    go = feats(7, B, C, n).cuda()
    d1, d2 = P.three_interpolate_grad(go, idx, w.cuda(), m), P.three_interpolate_grad(go, idx, w.cuda(), m)
    assert torch.equal(d1, d2)
    check_grad(d1, lambda: O.three_interpolate_grad(go.cpu(), wi, w, m), lambda: O.three_interpolate_grad(go.cpu(), wi, w, m, absolute=True))


def test_fps_edge_cases(P):
    cases = {
        "N=1": room(1, 2, 1),
        "npoint=1": room(2, 2, 300),
        "npoint>N": room(3, 2, 40),
        "all within the origin skip radius": room(4, 2, 500) * 0.01,
        "duplicated points (ties)": room(5, 2, 64).repeat(1, 8, 1),
        "mixed skip and duplicates": torch.cat([torch.zeros(2, 100, 3), room(6, 2, 50).repeat(1, 3, 1)], 1),
    }
    npoints = {"N=1": 4, "npoint=1": 1, "npoint>N": 100, "all within the origin skip radius": 16, "duplicated points (ties)": 200,
               "mixed skip and duplicates": 120}
    for name, xyz in cases.items():
        xyz = xyz.contiguous()
        got = P.furthest_point_sampling(xyz.cuda(), npoints[name]).cpu()
        assert torch.equal(got, O.furthest_point_sampling(xyz, npoints[name])), name


def test_fps_above_on_chip_capacity(P):
    from pointcontrast_b200 import _lib
    N = 110000
    assert _lib.lib.pcb_furthest_point_sampling_ws_bytes(2, N) > 0        # this size spills its running distances to the workspace
    xyz = room(8, 2, N)
    got = P.furthest_point_sampling(xyz.cuda(), 96).cpu()
    assert torch.equal(got, O.furthest_point_sampling(xyz, 96))


def test_query_edge_cases(P):
    xyz = room(9, 2, 700)
    new = room(10, 2, 50)
    for radius, S in ((1e-4, 8), (0.3, 1), (5.0, 4)):                   # empty balls (zero rows), nsample = 1, every point a hit
        idx = P.ball_query(new.cuda(), xyz.cuda(), radius, S).cpu()
        assert torch.equal(idx, O.ball_query(new, xyz, radius, S)), (radius, S)
    one = room(11, 2, 1)
    assert torch.equal(P.ball_query(new.cuda(), one.cuda(), 5.0, 3).cpu(), O.ball_query(new, one, 5.0, 3))
    for m in (1, 2):                                                      # m < 3: inf / 0 in the missing slots
        known = room(12, 2, m)
        d, i = P.three_nn(new.cuda(), known.cuda())
        wd, wi = O.three_nn(new, known)
        assert torch.equal(d.cpu(), wd) and torch.equal(i.cpu(), wi)
    dup = room(13, 2, 30).repeat(1, 4, 1).contiguous()                    # exact distance ties: the earlier k
    d, i = P.three_nn(new.cuda(), dup.cuda())
    wd, wi = O.three_nn(new, dup)
    assert torch.equal(d.cpu(), wd) and torch.equal(i.cpu(), wi)
    assert torch.equal(P.ball_query(new.cuda(), dup.cuda(), 0.8, 16).cpu(), O.ball_query(new, dup, 0.8, 16))


def test_inputs_are_checked(P):
    from pointcontrast_b200._lib import PcbError
    xyz = room(14, 2, 100).cuda()
    with pytest.raises(PcbError):
        P.furthest_point_sampling(xyz.cpu(), 4)
    with pytest.raises(PcbError):
        P.furthest_point_sampling(xyz.double(), 4)
    with pytest.raises(PcbError):
        P.furthest_point_sampling(xyz.transpose(0, 1), 4)
    with pytest.raises(PcbError):
        P.ball_query(xyz[:, :10], xyz, 0.2, 8)                          # non-contiguous slice
    with pytest.raises(PcbError):
        P.gather_points(feats(0, 2, 4, 100).cuda(), torch.zeros(2, 5, dtype=torch.int64, device="cuda"))
    with pytest.raises(PcbError):
        P.group_points(feats(0, 2, 4, 100).cuda(), torch.zeros(2, 5, 3, dtype=torch.int32))
    with pytest.raises(PcbError):
        P.three_interpolate(feats(0, 2, 4, 10).cuda(), torch.zeros(2, 5, 3, dtype=torch.int32, device="cuda"),
                            torch.zeros(2, 5, 3, dtype=torch.float64, device="cuda"))
    with pytest.raises(PcbError):
        P.ball_query(xyz, xyz, 0.0, 8)


# ------------------------------------------------------------------------------------------------ against the reference kernels
def first_fps_difference_is_a_tie(xyz, ours, ref):
    """At the first iteration where the two index lists differ, both picks must have exactly the same running fp32 distance."""
    p = xyz.numpy()
    cand = ~(((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]).astype(np.float64) <= 1e-3)
    temp = np.full(len(p), 1e10, dtype=np.float32)
    for j in range(1, len(ours)):
        temp = np.where(cand, np.minimum(O._d2(p, p[ours[j - 1]]), temp), temp)
        if ours[j] != ref[j]:
            return bool(cand[ours[j]] and cand[ref[j]] and temp[ours[j]] == temp[ref[j]] == temp[cand].max())
    return True


@pytest.mark.parametrize("B,N,npoint", [(8, 20000, 2048), (8, 40000, 2048), (8, 2048, 1024)])
def test_fps_matches_reference_kernel(P, REF, B, N, npoint):
    xyz = room(N + 2, B, N)
    ours = P.furthest_point_sampling(xyz.cuda(), npoint).cpu().numpy()
    ref = REF.furthest_point_sampling(xyz.cuda(), npoint).cpu().numpy()
    for b in range(B):
        if not np.array_equal(ours[b], ref[b]):
            assert first_fps_difference_is_a_tie(xyz[b], ours[b], ref[b]), f"scene {b}: differs without an exact fp32 tie"


@pytest.mark.parametrize("B,N,M,radius,S", BQ_CASES[:3])
def test_ball_query_and_gathers_match_reference_kernels(P, REF, B, N, M, radius, S):
    xyz = room(N + 3, B, N).cuda()
    new = xyz[:, torch.randperm(N, generator=torch.Generator().manual_seed(0))[:M].cuda()].contiguous()
    idx = P.ball_query(new, xyz, radius, S)
    assert torch.equal(idx, REF.ball_query(new, xyz, radius, S))
    f = feats(8, B, 32, N).cuda()
    assert torch.equal(P.group_points(f, idx), REF.group_points(f, idx))
    go = feats(9, B, 32, M, S).cuda()
    scale = O.group_points_grad(go.cpu(), idx.cpu(), N, absolute=True)
    err = (P.group_points_grad(go, idx, N).double() - REF.group_points_grad(go, idx, N).double()).abs().cpu()
    assert (err <= 2e-6 * scale + 1e-30).all()                  # both within 1e-6 of the exact sum (the reference's order varies)
    fidx = idx[:, :, 0].contiguous()
    assert torch.equal(P.gather_points(f, fidx), REF.gather_points(f, fidx))
    go2 = feats(10, B, 32, M).cuda()
    scale = O.gather_points_grad(go2.cpu(), fidx.cpu(), N, absolute=True)
    err = (P.gather_points_grad(go2, fidx, N).double() - REF.gather_points_grad(go2, fidx, N).double()).abs().cpu()
    assert (err <= 2e-6 * scale + 1e-30).all()


@pytest.mark.parametrize("B,n,m", [(8, 512, 256), (8, 1024, 512)])
def test_three_nn_and_interpolate_match_reference_kernels(P, REF, B, n, m):
    unknown, known = room(n + 5, B, n).cuda(), room(m + 9, B, m).cuda()
    d, i = P.three_nn(unknown, known)
    rd, ri = REF.three_nn(unknown, known)
    assert torch.equal(d, rd) and torch.equal(i, ri)
    recip = 1.0 / (torch.sqrt(d) + 1e-8)
    w = (recip / recip.sum(2, keepdim=True)).contiguous()
    f = feats(11, B, 128, m).cuda()
    assert torch.equal(P.three_interpolate(f, i, w), REF.three_interpolate(f, i, w))
    go = feats(12, B, 128, n).cuda()
    scale = O.three_interpolate_grad(go.cpu(), i.cpu(), w.cpu(), m, absolute=True)
    err = (P.three_interpolate_grad(go, i, w, m).double() - REF.three_interpolate_grad(go, i, w, m).double()).abs().cpu()
    assert (err <= 2e-6 * scale + 1e-30).all()


# ------------------------------------------------------------------------------------------------ drop-in
def test_reference_modules_run_on_this_library():
    """The original's unmodified PointnetSAModuleVotes (VoteNet SA1) and a PointnetFPModule, forward and backward on CUDA after
    pointnet2.install(), against the same modules with the same weights on the oracle `_ext` in fp64 (TF32 off).
    Training mode: indices and outputs.  Eval mode: outputs and the input gradient -- in training mode the fp32 BatchNorm backward
    (cuDNN) alone puts ~1e-3 between the GPU and the fp64 input gradient at this size, which says nothing about the ops under test."""
    from pointcontrast_b200 import pointnet2
    saved = {k: sys.modules.get(k) for k in ("pointnet2", "pointnet2._ext")}
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        B, N = 2, 20000
        xyz = room(15, B, N)
        f0 = feats(16, B, 3, N)

        def run(install, device, dtype, train):
            _, mods = reference_modules(install)
            torch.manual_seed(0)
            sa = mods.PointnetSAModuleVotes(npoint=2048, radius=0.2, nsample=64, mlp=[3, 64, 64, 128], use_xyz=True, normalize_xyz=True)
            fp = mods.PointnetFPModule(mlp=[128 + 3, 64])
            sa, fp = sa.to(device, dtype).train(train), fp.to(device, dtype).train(train)
            x = xyz.to(device)                                           # xyz stays fp32: the index ops take fp32 coordinates
            f = f0.to(device, dtype).requires_grad_()
            new_xyz, new_f, inds = sa(x, f)
            up = fp(x, new_xyz, f, new_f)
            (new_f.square().mean() + up.square().mean()).backward()
            return [t.detach().cpu() for t in (inds, new_f, up, f.grad)]

        for train in (True, False):
            ours = run(pointnet2.install, "cuda", torch.float32, train)
            want = run(O.install, "cpu", torch.float64, train)
            assert torch.equal(ours[0].long(), want[0].long())
            checked = zip(("features", "interpolated", "input gradient"), ours[1:], want[1:])
            for name, a, b in list(checked)[:2 if train else 3]:
                rel = float((a.double() - b).abs().max() / b.abs().max())
                assert rel < 1e-4, (name, train, rel)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
