"""The pair-list oracle (oracle/pair_list_cpu.py) against literal restatements of the reference's per-point loops, and the reference's
unmodified scripts (staged by oracle/pair_list_ref.py, run on stub open3d / SensorData modules) against the oracle's writers."""
import math
import os
import shutil

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import pair_list_cpu as O
from oracle import pair_list_ref
from pointcontrast_b200 import synth


def down_sample_literal(xyz, voxel_size):
    """open3d `VoxelDownSample` point by point: a dict voxel -> (running fp64 sum, count), then sum / count, in voxel order."""
    lo = [min(p[k] for p in xyz) - voxel_size * 0.5 for k in range(3)]
    acc = {}
    for p in xyz:
        key = tuple(int(math.floor((float(p[k]) - lo[k]) / voxel_size)) for k in range(3))
        s, c = acc.get(key, ([0.0, 0.0, 0.0], 0))
        acc[key] = ([s[k] + float(p[k]) for k in range(3)], c + 1)
    return np.array([[s[k] / c for k in range(3)] for s, c in (acc[key] for key in sorted(acc))])


def counts_literal(frames, radius):
    F = len(frames)
    out = np.zeros((F, F), np.int64)
    for i in range(F):
        for j in range(F):
            if i == j:
                continue
            for q in frames[j]:
                for p in frames[i]:
                    dx, dy, dz = float(p[0] - q[0]), float(p[1] - q[1]), float(p[2] - q[2])
                    if (dx * dx + dy * dy) + dz * dz < radius * radius:
                        out[i, j] += 1
                        break
    return out


def boundary_frames():
    """[(frame, voxel_size)] with points ON voxel boundaries.  Each frame holds its per-axis minimum m as a point, so lo = m - v / 2.
    Dyadic v: a point m + (k + 1/2) v has (p - lo) / v = k + 1 exactly (mixed per axis with voxel centres m + k v).  v = 0.05: points
    lo + k v (rounded) and both their fp64 neighbours, whose quotients lie within a few ulp of an integer on either side."""
    rng = np.random.default_rng(11)
    out = []
    for v, m in ((0.25, np.array([1.0, -2.0, 3.5])), (0.125, np.array([1024.0, -512.25, 7.0]))):
        k = rng.integers(0, 40, (3000, 3))
        out.append((np.concatenate([m[None], m + np.where(rng.random((3000, 3)) < 0.7, k + 0.5, k) * v]), v))
    v, m = 0.05, np.array([0.3, -1.7, 2.9])
    p = (m - v * 0.5) + rng.integers(1, 200, (2000, 3)) * v
    out.append((np.concatenate([m[None], p, np.nextafter(p, np.inf), np.nextafter(p, -np.inf)]), v))
    return out


def test_boundary_frames_lie_on_boundaries():
    """The boundary set is what it claims: exact integer quotients, and at v = 0.05 a kernel multiplying by 1 / v instead of dividing
    would put some of its points in other voxels."""
    for xyz, v in boundary_frames():
        q = (xyz - (xyz.min(0) - v * 0.5)) / v
        exact = q == np.floor(q)
        assert exact.mean() > (0.5 if v != 0.05 else 0.05), (v, exact.mean())
        if v == 0.05:
            recip = np.floor((xyz - (xyz.min(0) - v * 0.5)) * (1.0 / v))
            assert (recip != np.floor(q)).any()


@pytest.mark.parametrize("case", range(3))
def test_down_sample_on_voxel_boundaries_is_the_literal_loop(case):
    xyz, v = boundary_frames()[case]
    got, want = O.voxel_down_sample(xyz, v), down_sample_literal(xyz, v)
    assert got.shape == want.shape and np.array_equal(got.view(np.uint64), want.view(np.uint64))


def small_frames(seed, F, n):
    return [f[:n] for f in synth.synth_scan_frames(seed, F, points_per_frame=n, scale=0.5)]


@pytest.mark.parametrize("voxel", [0.05, 0.013])
def test_down_sample_is_the_literal_loop(voxel):
    rng = np.random.default_rng(1)
    xyz = np.concatenate([rng.normal(0, 0.2, (600, 3)), np.full((50, 3), 0.1), rng.integers(-8, 8, (100, 3)) * voxel])
    got = O.voxel_down_sample(xyz, voxel)
    want = down_sample_literal(xyz, voxel)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))


def test_counts_are_the_brute_force_loop():
    frames = small_frames(3, 4, 150)
    assert np.array_equal(O.frame_overlap_counts(frames, 0.075), counts_literal(frames, 0.075))
    assert np.array_equal(O.frame_overlap_counts([frames[0]], 0.075), np.zeros((1, 1), np.int64))


def test_counts_agree_with_ckdtree_away_from_the_boundary():
    frames = [O.voxel_down_sample(f, 0.05) for f in synth.synth_scan_frames(5, 5, points_per_frame=40_000)]
    r = 0.075
    got = O.frame_overlap_counts(frames, r)
    for i in range(len(frames)):
        tree = cKDTree(frames[i])
        for j in range(len(frames)):
            if i == j:
                continue
            inner = tree.query_ball_point(frames[j], r * (1 - 1e-6), return_length=True) > 0
            outer = tree.query_ball_point(frames[j], r * (1 + 1e-6), return_length=True) > 0
            assert inner.sum() <= got[i, j] <= outer.sum()
            if np.array_equal(inner, outer):
                assert got[i, j] == inner.sum()


def test_reference_scripts_write_the_oracles_files(tmp_path):
    if not pair_list_ref.available():
        pytest.skip("the reference's pair-list scripts are not staged")
    voxel = 0.05
    scene = tmp_path / "scene0000_00" / "pcd"
    scene.mkdir(parents=True)
    frames = synth.synth_scan_frames(7, 5, points_per_frame=20_000, scale=0.8)
    for k, f in enumerate(frames):
        np.savez(scene / f"{k * 25}.npz", pcd=f)
    pair_list_ref.run("compute_full_overlapping.py", ["--input_path", str(scene), "--voxel_size", str(voxel)])
    ref_overlap = (scene / "overlap.txt").read_text()
    pair_list_ref.run("generate_list.py", ["--target_dir", str(tmp_path)])
    ref_list = (tmp_path / "overlap-30-full.txt").read_text()

    names = sorted(os.path.join(str(scene), f) for f in os.listdir(scene) if f.endswith(".npz"))
    down = [O.voxel_down_sample(np.load(n)["pcd"], voxel) for n in names]
    mine = tmp_path / "mine"
    (mine / "scene0000_00" / "pcd").mkdir(parents=True)
    O.write_overlap(str(mine / "scene0000_00" / "pcd" / "overlap.txt"), names, O.frame_overlap_counts(down, 1.5 * voxel),
                    [len(d) for d in down])
    O.write_list(str(mine), [str(mine / "scene0000_00" / "pcd" / "overlap.txt")])

    def pairs(text):
        return {frozenset(line.split()[:2]): line.split()[2] for line in text.splitlines()}
    mine_overlap = (mine / "scene0000_00" / "pcd" / "overlap.txt").read_text()
    assert len(ref_overlap.splitlines()) == 10
    assert pairs(ref_overlap) == pairs(mine_overlap)                       # bit-identical values as printed
    assert 0 < len(ref_list.splitlines()) < 10
    assert sorted(pairs(ref_list).items(), key=str) == sorted(pairs((mine / "overlap-30-full.txt").read_text()).items(), key=str)
