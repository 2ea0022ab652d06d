"""PointNet++ operators (DESIGN.md 8f-5) at VoteNet's shapes, B = 8: SUN RGB-D (N = 20 000) and ScanNet (N = 40 000) point clouds.
Device time of every op (CUDA events, warmed, each timed window >= 1 s), this library and -- where __graft_entry__.build() compiled it
into oracle/_ref/pointnet2_ext -- the reference's own kernels in the same run, alternating; the SA1 module (FPS + ball query + grouping
+ shared MLP, the reference's PointnetSAModuleVotes on pointnet2.install()) forward + backward end to end; achieved bytes/s of the
gather-type ops against the H100 SXM's 3.35 TB/s; the GPU name and power limit read in the same call.  Prints one JSON line.

    python profiles/bench_pointnet2.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointcontrast_b200 import pointnet2  # noqa: E402

HBM = 3.35e12
B = 8


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def load_ref():
    """The compiled reference `_ext` (what build() produced), or None; the original repository itself is never read."""
    import glob
    import importlib.machinery
    import importlib.util
    so = glob.glob(os.path.join(ROOT, "oracle", "_ref", "pointnet2_ext", "_ext*.so"))
    if not so:
        return None
    loader = importlib.machinery.ExtensionFileLoader("_ext", so[0])
    spec = importlib.util.spec_from_file_location("_ext", so[0], loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def time_ms(fn, min_window_s=1.0):
    """Mean device time per call: warm up, size the window to >= min_window_s, time it with CUDA events."""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    n = max(3, int(min_window_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def workloads(N):
    g = torch.Generator(device="cuda").manual_seed(N)
    xyz = (torch.rand(B, N, 3, device="cuda", generator=g) * torch.tensor([6.0, 6.0, 2.5], device="cuda") - torch.tensor([3.0, 3.0, 0.5], device="cuda")).contiguous()
    E = pointnet2.ext
    inds = E.furthest_point_sampling(xyz, 2048)
    new = E.gather_points(xyz.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
    idx = E.ball_query(new, xyz, 0.2, 64)
    f = torch.randn(B, 64, N, device="cuda", generator=g)
    go = torch.randn(B, 64, 2048, 64, device="cuda", generator=g)
    up_u, up_k = new[:, :1024].contiguous(), new[:, :512].contiguous()
    d, i3 = E.three_nn(up_u, up_k)
    w = (1.0 / (d + 1e-8)); w = (w / w.sum(2, keepdim=True)).contiguous()
    fk = torch.randn(B, 256, 512, device="cuda", generator=g)
    gi = torch.randn(B, 256, 1024, device="cuda", generator=g)
    xyz_t = xyz.transpose(1, 2).contiguous()
    gg = torch.randn(B, 3, 2048, device="cuda", generator=g)
    # (name, call(ext), bytes moved by the algorithm or None)
    return [
        ("fps_2048", lambda e: e.furthest_point_sampling(xyz, 2048), None),
        ("ball_query_r0.2_s64", lambda e: e.ball_query(new, xyz, 0.2, 64), None),
        ("group_points_c64_2048x64", lambda e: e.group_points(f, idx), (B * 64 * 2048 * 64) * 4 * 2 + idx.numel() * 4),
        ("group_points_grad", lambda e: e.group_points_grad(go, idx, N), go.numel() * 4 + idx.numel() * 4 + B * 64 * N * 4),
        ("gather_points_xyz_2048", lambda e: e.gather_points(xyz_t, inds), B * 3 * 2048 * 4 * 2 + inds.numel() * 4),
        ("gather_points_grad", lambda e: e.gather_points_grad(gg, inds, N), gg.numel() * 4 + inds.numel() * 4 + B * 3 * N * 4),
        ("three_nn_1024_from_512", lambda e: e.three_nn(up_u, up_k), None),
        ("three_interpolate_c256_1024", lambda e: e.three_interpolate(fk, i3, w), gi.numel() * 4 + i3.numel() * 8 + fk.numel() * 4),
        ("three_interpolate_grad", lambda e: e.three_interpolate_grad(gi, i3, w, 512), gi.numel() * 4 + i3.numel() * 8 + fk.numel() * 4),
    ]


def sa1_ms(N):
    """The reference's PointnetSAModuleVotes(2048, 0.2, 64, [3, 64, 64, 128]) forward + backward on this library, when staged."""
    mods_dir = os.path.join(ROOT, "oracle", "_ref", "votenet", "pointnet2")
    if not os.path.isfile(os.path.join(mods_dir, "pointnet2_modules.py")):
        return None
    pointnet2.install()
    sys.path.insert(0, mods_dir)
    import pointnet2_modules
    sa = pointnet2_modules.PointnetSAModuleVotes(npoint=2048, radius=0.2, nsample=64, mlp=[3, 64, 64, 128], use_xyz=True,
                                                 normalize_xyz=True).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(1)
    xyz = (torch.rand(B, N, 3, device="cuda", generator=g) * 6 - 3).contiguous()
    f = torch.randn(B, 3, N, device="cuda", generator=g, requires_grad=True)

    def step():
        _, nf, _ = sa(xyz, f)
        nf.sum().backward()
    return time_ms(step)


def main():
    torch.backends.cudnn.benchmark = True
    ref = load_ref()
    out = {"gpu": gpu_info(), "B": B, "reference_kernels": ref is not None, "ops": {}}
    for N in (20000, 40000):
        tag = "sunrgbd_N20000" if N == 20000 else "scannet_N40000"
        rows = {}
        for name, call, nbytes in workloads(N):
            ours, theirs = [], []
            for _ in range(2):                                       # alternate ours / reference twice, keep the best of each
                ours.append(time_ms(lambda: call(pointnet2.ext)))
                if ref is not None:
                    theirs.append(time_ms(lambda: call(ref)))
            r = {"ours_ms": min(ours)}
            if ref is not None:
                r["reference_ms"] = min(theirs)
                r["speedup"] = r["reference_ms"] / r["ours_ms"]
            if nbytes:
                r["ours_GBps"] = nbytes / (r["ours_ms"] * 1e-3) / 1e9
                r["ours_frac_of_3.35TBps"] = nbytes / (r["ours_ms"] * 1e-3) / HBM
            rows[name] = r
        rows["sa1_fwd_bwd_ms"] = sa1_ms(N)
        out["ops"][tag] = rows
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
