"""Sparse-conv detection backbone (DESIGN.md 8f-7) at the two detection scripts' shapes, 2.5 cm voxels, synthetic rooms
(synth.synth_votenet_batch): ScanNet B = 32, N = 40 000 and SUN RGB-D B = 64, N = 20 000.  Reports voxel counts; `voxelize_batch`
time; seed sampling as one ragged launch against the per-scene loop the original module runs on this library (boolean-mask gathers +
one `furthest_point_sample` per scene), timed alternately in the same call with identical seeds asserted; backbone forward + backward
per step, ours and -- where build() staged it into oracle/_ref/votenet -- the original module on this library, alternately; peak device
memory.  Device time by CUDA events over warmed shapes, windows >= 1 s; the GPU name and power limit read in the same call.  A
workload that does not fit is reported as such.  Prints one JSON line.

    python profiles/bench_detection.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointcontrast_b200 import detection, pointnet2, synth  # noqa: E402

VOXEL = 0.025
WORKLOADS = (("scannet", 32, 40000), ("sunrgbd", 64, 20000))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def time_ms(fn, min_window_s=1.0):
    """Mean device time per call: warm up, size the window to >= min_window_s, time it with CUDA events."""
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    n = max(3, int(min_window_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, rounds=2):
    """{name: [ms per round]}, the candidates timed in turn."""
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            out[k].append(round(time_ms(f), 3))
    return out


def original_module():
    """The original `models/backbone_module.py` staged by build(), on this library; None where it was not staged."""
    staged = os.path.join(ROOT, "oracle", "_ref", "votenet")
    if not os.path.isfile(os.path.join(staged, "models", "backbone_module.py")):
        return None
    from pointcontrast_b200 import me
    me.install()
    pointnet2.install()
    sys.path.insert(0, staged)
    import importlib
    return importlib.import_module("models.backbone_module")


def per_scene_loop(points, coords, inds, num_seed):
    """`models/backbone_module.py:163-171`: one furthest_point_sample per scene on its boolean-mask gather."""
    B, N, _ = points.shape
    flat = points.view(-1, 3)
    batch_ids = coords[:, 0]
    voxel_ids = inds + batch_ids * N
    return torch.stack([pointnet2.furthest_point_sample(flat[voxel_ids[batch_ids == b]].unsqueeze(0), num_seed).squeeze(0)
                        for b in range(B)])


def ragged(points, coords, inds, num_seed):
    B, N, _ = points.shape
    offsets = detection.scene_offsets(coords[:, 0], B)
    vxyz = points.reshape(-1, 3)[inds.long() + coords[:, 0].long() * N].contiguous()
    return pointnet2.furthest_point_sampling_ragged(vxyz, offsets, N, num_seed)


def workload(name, B, N, bm):
    res = {"B": B, "N": N}
    xyz = torch.from_numpy(synth.synth_votenet_batch(0, B, N)).cuda()
    batch = detection.voxelize_batch({"point_clouds": xyz}, VOXEL)
    counts = torch.bincount(batch["voxel_coords"][:, 0].long(), minlength=B).tolist()
    res["voxels_total"], res["voxels_per_scene_min_mean_max"] = sum(counts), [min(counts), round(sum(counts) / B), max(counts)]
    res["voxelize_batch_ms"] = round(time_ms(lambda: detection.voxelize_batch({"point_clouds": xyz}, VOXEL)), 3)
    c, i = batch["voxel_coords"], batch["voxel_inds"]
    assert torch.equal(ragged(xyz, c, i, 1024), per_scene_loop(xyz, c, i, 1024))
    seeds = alternate({"ragged_one_launch": lambda: ragged(xyz, c, i, 1024), "per_scene_loop": lambda: per_scene_loop(xyz, c, i, 1024)})
    res["seed_sampling_ms"] = seeds
    res["seed_sampling_speedup"] = round(min(seeds["per_scene_loop"]) / min(seeds["ragged_one_launch"]), 2)
    torch.manual_seed(0)
    ours = detection.SparseConvBackbone().cuda().train()
    w = torch.randn(B, 256, 1024, device="cuda")
    models = {"ours": ours}
    if bm is not None:
        ref = bm.SparseConvBackbone()
        ref.load_state_dict(ours.state_dict())
        models["original_module"] = ref.cuda().train()

    def step(m):
        def f():
            m.zero_grad(set_to_none=True)
            ep = m(xyz, c, batch["voxel_feats"], i, {})
            (ep["fp2_features"] * w).sum().backward()
        return f
    torch.cuda.reset_peak_memory_stats()
    try:
        res["fwd_bwd_step_ms"] = alternate({k: step(m) for k, m in models.items()})
        res["peak_memory_GiB"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
    except torch.cuda.OutOfMemoryError as e:
        res["fwd_bwd_step_ms"] = f"out of memory: {str(e).splitlines()[0]}"
    del models, ours
    torch.cuda.empty_cache()
    return res


def main():
    torch.cuda.set_device(0)
    out = {"gpu": gpu_info(), "voxel_size": VOXEL, "num_seed": 1024}
    bm = original_module()
    out["original_module_staged"] = bm is not None
    for name, B, N in WORKLOADS:
        out[name] = workload(name, B, N, bm)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
