"""`pair_list.read_sens` on synthetic `.sens` files (`synth.write_sens`): the header, the kept frames, the poses and intrinsics after
the reference's text round trip, and every error it raises.  No GPU."""
import os
import struct

import numpy as np
import pytest

from oracle import sens_cpu
from pointcontrast_b200 import pair_list, synth


def write(tmp_path, n=7, name="s.sens", **kw):
    depth, poses, K = synth.synth_sens_scan(3, n, width=32, height=24, bad_poses=(3,) if n > 3 else ())
    path = str(tmp_path / name)
    synth.write_sens(path, depth, poses, K, color_bytes=(500, 900), **kw)
    return path, depth, poses, K


def header_offset():
    """The byte offset of the depth width in `write_sens`'s header (version, name length, "StructureSensor", 4 matrices, 2 types,
    the colour size)."""
    return 4 + 8 + len(b"StructureSensor") + 256 + 8 + 8


@pytest.mark.parametrize("skip", [1, 2, 3, 7])
def test_header_frames_poses_and_depth(tmp_path, skip):
    path, depth, poses, K = write(tmp_path)
    s = pair_list.read_sens(path, skip)
    assert s.sensor_name == b"StructureSensor" and s.num_frames == 7
    assert (s.color_compression_type, s.depth_compression_type) == ("jpeg", "zlib_ushort")
    assert (s.color_width, s.color_height, s.depth_width, s.depth_height, s.depth_shift) == (1296, 968, 32, 24, 1000.0)
    assert np.array_equal(s.intrinsic_depth, K.astype(np.float32)) and np.array_equal(s.extrinsic_depth, np.eye(4, dtype=np.float32))
    kept = np.arange(0, 7, skip)
    assert np.array_equal(s.frames, kept)
    assert np.array_equal(s.depth, depth[kept])
    assert np.array_equal(s.camera_to_world, poses[kept].astype(np.float32))
    assert np.array_equal(s.poses, sens_cpu.text_round_trip(poses[kept].astype(np.float32)), equal_nan=True)
    assert np.array_equal(s.intrinsic, sens_cpu.text_round_trip(K.astype(np.float32)))
    if 3 in kept:
        assert np.isneginf(s.poses[list(kept).index(3)]).all()


def test_text_round_trip_is_savetxt_loadtxt():
    rng = np.random.default_rng(0)
    a = np.concatenate([rng.normal(0, 3, 40), rng.normal(0, 1e-7, 12), [1e7, -2.5e-7, 0.0, -0.0, 5e-7, -5e-7, np.inf, -np.inf, np.nan,
                                                                       0.1234565, 1.0000005, -3.9999995]]).astype(np.float32)
    a = a.reshape(4, 4, 4)
    got, want = pair_list.text_round_trip(a), sens_cpu.text_round_trip(a)
    assert np.array_equal(got, want, equal_nan=True)
    assert got[3, 1, 0] == 1e7 and got[3, 1, 2] == 0.0 and np.isneginf(got[3, 2, 3]) and np.isnan(got[3, 3, 0])


def test_frame_skip_beyond_the_frame_count(tmp_path):
    path, depth, _, _ = write(tmp_path, n=3)
    s = pair_list.read_sens(path, 100)
    assert np.array_equal(s.frames, [0]) and np.array_equal(s.depth, depth[:1])
    with pytest.raises(ValueError, match="frame_skip"):
        pair_list.read_sens(path, 0)


def test_no_frames(tmp_path):
    path = str(tmp_path / "e.sens")
    synth.write_sens(path, np.zeros((0, 24, 32), np.uint16), np.zeros((0, 4, 4)), np.eye(4))
    s = pair_list.read_sens(path, 25)
    assert s.num_frames == 0 and s.depth.shape == (0, 24, 32) and s.poses.shape == (0, 4, 4)


def test_version_other_than_4(tmp_path):
    path, *_ = write(tmp_path, version=3)
    with pytest.raises(ValueError, match="version 3"):
        pair_list.read_sens(path)


@pytest.mark.parametrize("code", [0, 2, -1])
def test_depth_compression_other_than_zlib(tmp_path, code):
    path, *_ = write(tmp_path, depth_compression=code)
    with pytest.raises(ValueError, match="only 'zlib_ushort'"):
        pair_list.read_sens(path)


def test_unknown_compression_type(tmp_path):
    path, *_ = write(tmp_path, depth_compression=7)
    with pytest.raises(ValueError, match="unknown compression"):
        pair_list.read_sens(path)


@pytest.mark.parametrize("cut", [3, 100, 340, -1, -3000])
@pytest.mark.parametrize("skip", [1, 2])
def test_truncated_file(tmp_path, cut, skip):
    """Cut in the header, in the middle of the frames, and one byte short of the end (the last frame's depth: read at skip 1,
    seeked past at skip 2 when it is dropped)."""
    path, *_ = write(tmp_path)
    data = open(path, "rb").read()
    open(path, "wb").write(data[:cut] if cut > 0 else data[:len(data) + cut])
    with pytest.raises(ValueError, match="truncated"):
        pair_list.read_sens(path, skip)


def test_truncated_dropped_last_frame(tmp_path):
    path, *_ = write(tmp_path, n=8)              # frame 7 is dropped at skip 2: its bytes are only seeked past
    data = open(path, "rb").read()
    open(path, "wb").write(data[:-1])
    with pytest.raises(ValueError, match="truncated"):
        pair_list.read_sens(path, 2)


def test_depth_of_the_wrong_size(tmp_path):
    path, *_ = write(tmp_path)
    data = bytearray(open(path, "rb").read())
    o = header_offset()
    assert struct.unpack("<II", data[o:o + 8]) == (32, 24)
    data[o:o + 4] = struct.pack("<I", 31)
    open(path, "wb").write(bytes(data))
    with pytest.raises(ValueError, match="inflates to 1536 bytes, not 2 \\* 31 \\* 24"):
        pair_list.read_sens(path)


def test_depth_that_does_not_inflate(tmp_path):
    path = str(tmp_path / "z.sens")
    depth, poses, K = synth.synth_sens_scan(4, 2, width=16, height=12)
    synth.write_sens(path, depth, poses, K, color_bytes=(10, 20))
    data = bytearray(open(path, "rb").read())
    data[-8:] = b"\x00" * 8                      # the last frame's zlib stream loses its end and checksum
    open(path, "wb").write(bytes(data))
    with pytest.raises(ValueError, match="frame 1's depth does not inflate"):
        pair_list.read_sens(path)


def test_extract_refuses_too_many_frames_before_writing(tmp_path, monkeypatch):
    path, *_ = write(tmp_path)
    monkeypatch.setattr(pair_list, "MAX_FRAMES", 3)
    out = tmp_path / "scene"
    with pytest.raises(pair_list._lib.PcbError, match="at most 3"):
        pair_list.extract_scene(path, str(out), 2)
    assert not os.path.exists(out)
