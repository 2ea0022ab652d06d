"""VoteNet's PointNet++ modules on the library (pointnet2_modules, DESIGN.md 8f-16) against the original's torch modules on
pointnet2.install(), forward + backward, timed as the other profiles time (CUDA events, warmed, windows >= 1 s, the routes alternating):
  * every module VoteNet runs at B = 8, SA1 at SUN RGB-D (N = 20 000) and ScanNet (N = 40 000) shapes, the vote aggregation also at the
    sparse-conv scripts' B = 32 and 64; the original once at torch's defaults (TF32 on, what users get) and once with TF32 off;
  * the whole Pointnet2Backbone + vote aggregation chain (SA1-SA4, FP1, FP2, vote aggregation), with each route's peak device memory;
  * the achieved bytes/s of each new kernel at SA1's shape, from byte counts computed here;
  * the chain's outputs of both routes (same weights, TF32 off) within the tests' 1e-4.
(The chain's agreement is the largest difference of each stage over its largest value.)  The original modules are the ones __graft_entry__.build() staged under oracle/_ref/votenet/pointnet2.  Prints one JSON line with the GPU
name and power limit read in the same call.

    python profiles/bench_pointnet2_modules.py
"""
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from pointcontrast_b200 import pointnet2, pointnet2_modules  # noqa: E402
from pointcontrast_b200._lib import check, lib, ptr, stream  # noqa: E402
from oracle import stage_ref  # noqa: E402
from profiles.bench_pointnet2 import gpu_info, time_ms  # noqa: E402

# name: (B, N, C_in, npoint, nsample, radius, mlp) -- backbone_module.py / proposal_module.py
SA = {"sa1_sunrgbd": (8, 20000, 0, 2048, 64, 0.2, [0, 64, 64, 128]), "sa1_scannet": (8, 40000, 0, 2048, 64, 0.2, [0, 64, 64, 128]),
      "sa2": (8, 2048, 128, 1024, 32, 0.4, [128, 128, 128, 256]), "sa3": (8, 1024, 256, 512, 16, 0.8, [256, 128, 128, 256]),
      "sa4": (8, 512, 256, 256, 16, 1.2, [256, 128, 128, 256]), "vote_b8": (8, 1024, 256, 256, 16, 0.3, [256, 128, 128, 128]),
      "vote_b32": (32, 1024, 256, 256, 16, 0.3, [256, 128, 128, 128]), "vote_b64": (64, 1024, 256, 256, 16, 0.3, [256, 128, 128, 128])}
FP = {"fp1": (8, 512, 256), "fp2": (8, 1024, 512)}       # (B, n unknown, m known); mlp [512, 256, 256]


def original():
    if not stage_ref.available("votenet"):
        raise SystemExit("the original modules are not staged under oracle/_ref/votenet/pointnet2 (run __graft_entry__.build())")
    for m in ("pointnet2_utils", "pointnet2_modules", "pytorch_utils"):
        sys.modules.pop(m, None)
    pointnet2.install()
    sys.path.insert(0, stage_ref.path("votenet", "pointnet2"))
    return importlib.import_module("pointnet2_modules")


def pair(ref, cls, **kw):
    """(original, ours) with the same weights."""
    a = getattr(ref, cls)(**{k: list(v) if isinstance(v, list) else v for k, v in kw.items()}).cuda().train()
    b = getattr(pointnet2_modules, cls)(**{k: list(v) if isinstance(v, list) else v for k, v in kw.items()}).cuda().train()
    b.load_state_dict(a.state_dict())
    return a, b


def room(B, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(B, N, 3, device="cuda", generator=g) * torch.tensor([6.0, 6.0, 2.5], device="cuda")
            - torch.tensor([3.0, 3.0, 0.5], device="cuda"))


def routes(fn_ours, fn_ref):
    """Mean ms of ours, the original with TF32 on and with TF32 off, alternating over two rounds (the smaller of each)."""
    res = {"ours": [], "original_tf32": [], "original_fp32": []}
    for _ in range(2):
        res["ours"].append(time_ms(fn_ours))
        for name, on in (("original_tf32", True), ("original_fp32", False)):
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
            res[name].append(time_ms(fn_ref))
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, True          # torch's defaults
    return {k: round(min(v), 3) for k, v in res.items()}


def sa_step(mod, xyz, f):
    def run():
        mod.zero_grad(set_to_none=True)
        _, nf, _ = mod(xyz, f)
        nf.sum().backward()
    return run


def bench_modules(ref):
    out = {}
    for name, (B, N, C, npoint, S, radius, mlp) in SA.items():
        a, b = pair(ref, "PointnetSAModuleVotes", npoint=npoint, radius=radius, nsample=S, mlp=mlp, normalize_xyz=True)
        xyz = room(B, N, 1)
        f = torch.rand(B, C, N, device="cuda", requires_grad=True) if C else None
        out[name] = routes(sa_step(b, xyz, f), sa_step(a, xyz, f))
    for name, (B, n, m) in FP.items():
        a, b = pair(ref, "PointnetFPModule", mlp=[512, 256, 256])
        unknown, known = room(B, n, 2), room(B, m, 3)
        uf = torch.rand(B, 256, n, device="cuda", requires_grad=True)
        kf = torch.rand(B, 256, m, device="cuda", requires_grad=True)

        def step(mod):
            def run():
                mod.zero_grad(set_to_none=True)
                mod(unknown, known, uf, kf).sum().backward()
            return run
        out[name] = routes(step(b), step(a))
    return out


def chain(mods, xyz):
    """Pointnet2Backbone (backbone_module.py) + the vote aggregation on the seeds, forward + backward; returns the outputs."""
    sa1, sa2, sa3, sa4, fp1, fp2, va = mods
    x1, f1, _ = sa1(xyz, None)
    x2, f2, _ = sa2(x1, f1)
    x3, f3, _ = sa3(x2, f2)
    x4, f4, _ = sa4(x3, f3)
    g = fp1(x3, x4, f3, f4)
    g = fp2(x2, x3, f2, g)
    inds = pointnet2.furthest_point_sample(x2[:, :1024].contiguous(), 256)
    _, agg, _ = va(x2[:, :1024].contiguous(), g, inds)
    (agg.square().mean() + g.square().mean()).backward()
    return agg.detach(), g.detach()


def bench_chain(ref, N):
    kw = [dict(npoint=2048, radius=0.2, nsample=64, mlp=[0, 64, 64, 128]), dict(npoint=1024, radius=0.4, nsample=32, mlp=[128, 128, 128, 256]),
          dict(npoint=512, radius=0.8, nsample=16, mlp=[256, 128, 128, 256]), dict(npoint=256, radius=1.2, nsample=16, mlp=[256, 128, 128, 256])]
    pairs = [pair(ref, "PointnetSAModuleVotes", normalize_xyz=True, **k) for k in kw]
    pairs += [pair(ref, "PointnetFPModule", mlp=[512, 256, 256]) for _ in range(2)]
    pairs.append(pair(ref, "PointnetSAModuleVotes", npoint=256, radius=0.3, nsample=16, mlp=[256, 128, 128, 128], normalize_xyz=True))
    theirs, ours = [p[0] for p in pairs], [p[1] for p in pairs]
    xyz = room(8, N, 4)
    res = routes(lambda: chain(ours, xyz), lambda: chain(theirs, xyz))
    for name, mods, tf32 in (("ours", ours, False), ("original_fp32", theirs, False)):
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
        for m in mods:
            m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        chain(mods, xyz)
        torch.cuda.synchronize()
        res[f"peak_mib_{name}"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    # agreement: fresh pairs (the same weights and running statistics), one training-mode forward each, TF32 off
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    pairs = [pair(ref, "PointnetSAModuleVotes", normalize_xyz=True, **k) for k in kw]
    pairs += [pair(ref, "PointnetFPModule", mlp=[512, 256, 256]) for _ in range(2)]
    pairs.append(pair(ref, "PointnetSAModuleVotes", npoint=256, radius=0.3, nsample=16, mlp=[256, 128, 128, 128], normalize_xyz=True))
    with torch.no_grad():
        got = _fwd([p[1] for p in pairs], xyz)
        want = _fwd([p[0] for p in pairs], xyz)
    res["max_rel_diff"] = {k: float((got[k] - want[k]).abs().max() / want[k].abs().max()) for k in want}
    torch.backends.cudnn.allow_tf32 = True
    return res


def _fwd(mods, xyz):
    """Every stage's features of the chain (forward only)."""
    sa1, sa2, sa3, sa4, fp1, fp2, va = mods
    x1, f1, _ = sa1(xyz, None)
    x2, f2, _ = sa2(x1, f1)
    x3, f3, _ = sa3(x2, f2)
    x4, f4, _ = sa4(x3, f3)
    g1 = fp1(x3, x4, f3, f4)
    g2 = fp2(x2, x3, f2, g1)
    inds = pointnet2.furthest_point_sample(x2.contiguous(), 256)
    return dict(sa1=f1, sa2=f2, sa3=f3, sa4=f4, fp1=g1, fp2=g2, vote_aggregation=va(x2.contiguous(), g2, inds)[1])


def bench_kernels():
    """Each new kernel at SA1's SUN RGB-D shape (B 8, 2048 x 64 rows, 64 / 128 channels): ms and GB/s of the bytes it must move."""
    B, N, npoint, S, C0, CL = 8, 20000, 2048, 64, 64, 128
    M, R = B * npoint, B * npoint * S
    xyz = room(B, N, 5)
    new_xyz = xyz[:, :npoint].contiguous()
    idx = torch.randint(0, N, (B, npoint, S), dtype=torch.int32, device="cuda")
    P = torch.rand(B * N, C0, device="cuda")
    wx = torch.rand(3, C0, device="cuda")
    rel, gidx, z0 = torch.empty(R, 3, device="cuda"), torch.empty(R, dtype=torch.int32, device="cuda"), torch.empty(R, C0, device="cuda")
    z = torch.randn(R, CL, device="cuda")
    mean, invstd, gamma, beta = torch.zeros(CL, device="cuda"), torch.ones(CL, device="cuda"), torch.randn(CL, device="cuda"), torch.zeros(CL, device="cuda")
    sel, out, g = torch.empty(M, CL, dtype=torch.int32, device="cuda"), torch.empty(M, CL, device="cuda"), torch.randn(M, CL, device="cuda")
    dY = torch.empty(R, CL, device="cuda")
    grel, rows = torch.randn(R, 3, device="cuda"), torch.empty(R + M, 3, device="cuda")
    st = stream()
    kernels = {
        # idx + P rows read, z0 + rel + gidx written (xyz / centres are L2-resident)
        "sa_layer0": (lambda: check(lib.pcb_sa_layer0(ptr(xyz), ptr(new_xyz), ptr(idx), B, N, npoint, S, 0.2, ptr(P), C0, ptr(wx), C0,
                                                      ptr(rel), ptr(gidx), ptr(z0), C0, st)), R * (4 + 4 * C0 + 4 * C0 + 12 + 4)),
        "sa_pool": (lambda: check(lib.pcb_sa_pool(ptr(z), CL, M, S, CL, ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(sel), ptr(out),
                                                  CL, st)), R * CL * 4 + M * CL * 8),
        "sa_pool_grad": (lambda: check(lib.pcb_sa_pool_grad(ptr(g), CL, ptr(sel), ptr(out), CL, M, S, CL, ptr(dY), st)), M * CL * 12 + R * CL * 4),
        "sa_xyz_rows": (lambda: check(lib.pcb_sa_xyz_rows(ptr(grel), None, M, S, 0.2, ptr(rows), st)), R * 24 + M * 12),
    }
    res = {}
    for name, (fn, nbytes) in kernels.items():
        ms = time_ms(fn)
        res[name] = {"ms": round(ms, 4), "GB/s": round(nbytes / ms / 1e6, 1)}
    return res


def main():
    torch.cuda.set_device(0)
    ref = original()
    torch.manual_seed(0)
    result = {"gpu": gpu_info(), "unit": "ms per forward + backward (min of two alternating rounds)",
              "modules": bench_modules(ref),
              "backbone_plus_vote_aggregation": {"sunrgbd_N20000": bench_chain(ref, 20000), "scannet_N40000": bench_chain(ref, 40000)},
              "kernels": bench_kernels()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
