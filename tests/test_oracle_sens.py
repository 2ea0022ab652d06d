"""The `.sens` oracle (oracle/sens_cpu.py) and `pair_list.read_sens` against the reference's unmodified `SensorData.py`, `reader.py`
and `point_cloud_extractor.py` (staged by oracle/sens_ref.py, with its lossless array codec in place of PNG), and against the golden
they wrote (tests/golden/sens_extract.npz).  No GPU; the tests that run the original skip where it is not staged."""
import io
import os

import numpy as np
import pytest

from oracle import sens_cpu, sens_ref
from pointcontrast_b200 import pair_list, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sens_extract.npz")
staged = pytest.mark.skipif(not sens_ref.available(), reason="the reference's .sens scripts are not staged")


def small_scan(tmp_path, n=6):
    depth, poses, K = synth.synth_sens_scan(5, n, width=80, height=60, holes=0.05, far=0.01, bad_poses=(2,))
    depth[4] = 0
    path = str(tmp_path / "scene0001_00.sens")
    synth.write_sens(path, depth, poses, K, color_bytes=(3000, 6000))
    return path


@staged
def test_original_sensor_data_reads_what_read_sens_reads(tmp_path):
    path = small_scan(tmp_path)
    sd = sens_ref.sensor_data(path)
    s = pair_list.read_sens(path, 1)
    assert sd.sensor_name == s.sensor_name
    for k in ("intrinsic_color", "extrinsic_color", "intrinsic_depth", "extrinsic_depth"):
        assert np.array_equal(getattr(sd, k), getattr(s, k)), k
    for k in ("color_compression_type", "depth_compression_type", "color_width", "color_height", "depth_width", "depth_height",
              "depth_shift"):
        assert getattr(sd, k) == getattr(s, k), k
    assert len(sd.frames) == s.num_frames == len(s.frames)
    for k, fr in enumerate(sd.frames):
        assert np.array_equal(fr.camera_to_world, s.camera_to_world[k], equal_nan=True)
        assert fr.decompress_depth(sd.depth_compression_type) == s.depth[k].astype("<u2").tobytes()


@staged
def test_original_text_files_are_the_round_trip(tmp_path):
    path = small_scan(tmp_path)
    scene = str(tmp_path / "scene")
    sens_ref.run("reader.py", ["--filename", path, "--output_path", scene, "--frame_skip", "2", "--export_poses", "--export_intrinsics"])
    s = pair_list.read_sens(path, 2)
    for k, f in enumerate(s.frames):
        text = open(os.path.join(scene, "pose", f"{f}.txt")).read()
        assert np.array_equal(np.loadtxt(io.StringIO(text)), s.poses[k], equal_nan=True)
        assert np.array_equal(sens_cpu.text_round_trip(s.camera_to_world[k]), s.poses[k], equal_nan=True)
    assert np.array_equal(np.loadtxt(os.path.join(scene, "intrinsic", "intrinsic_depth.txt")), s.intrinsic)
    assert sorted(os.listdir(os.path.join(scene, "pose"))) == sorted(f"{f}.txt" for f in s.frames)


def check_against_original(frames_pcd, scan):
    """Each original npz frame against the restatement: same rows in the same order, within the derived bound (NaN equal to NaN)."""
    assert len(frames_pcd) == len(scan.frames)
    exact = 0
    for k, ref in enumerate(frames_pcd):
        mine = sens_cpu.depth_to_points(scan.depth[k], scan.intrinsic, scan.poses[k])
        assert mine.shape == ref.shape == (int((scan.depth[k] != 0).sum()), 3)
        assert sens_cpu.within_bound(mine, ref, sens_cpu.dot_bound(scan.depth[k], scan.intrinsic, scan.poses[k])), k
        exact += int(np.array_equal(mine, ref, equal_nan=True))
    return exact


@staged
def test_original_extractor_agrees_with_the_restatement(tmp_path):
    path = small_scan(tmp_path)
    scene = str(tmp_path / "scene")
    sens_ref.extract(path, scene, 1)
    s = pair_list.read_sens(path, 1)
    pcd = [np.load(os.path.join(scene, "pcd", f"{f}.npz"))["pcd"] for f in s.frames]
    check_against_original(pcd, s)
    assert pcd[4].shape == (0, 3) and np.isnan(pcd[2]).any()


def golden():
    z = np.load(GOLDEN)
    off = z["offsets"]
    return z, [z["pcd"][off[k]:off[k + 1]] for k in range(len(off) - 1)]


def test_golden_agrees_with_the_restatement(tmp_path):
    z, pcd = golden()
    path = str(tmp_path / "scene0000_00.sens")
    open(path, "wb").write(z["sens"].tobytes())
    s = pair_list.read_sens(path, int(z["frame_skip"]))
    assert np.array_equal(s.frames, z["frames"])
    for k in range(len(s.frames)):
        assert np.array_equal(np.loadtxt(io.StringIO(str(z["pose_text"][k]))), s.poses[k], equal_nan=True)
    assert np.array_equal(np.loadtxt(io.StringIO(str(z["intrinsic_text"]))), s.intrinsic)
    check_against_original(pcd, s)
    assert pcd[1].shape == (0, 3) and np.isnan(pcd[2]).any() and (s.depth == 65535).any()
