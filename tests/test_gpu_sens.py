"""pcb_depth_to_points and `pair_list.extract_scene` / `extract_scenes` against the restatement (oracle/sens_cpu.py): points bit-exact,
offsets and NaN flags equal; against the reference's own output (tests/golden/sens_extract.npz) within the derived bound; the
overlap.txt byte-identical to what `compute_full_overlapping` writes from the npz files."""
import ctypes
import os
import threading

import numpy as np
import pytest
import torch

from oracle import sens_cpu
from pointcontrast_b200 import _lib, pair_list, synth
from tests.test_oracle_sens import check_against_original, golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def edge_batch():
    """640 x 480 frames: two rendered frames with holes and depth 65535, an all-zero frame, a full-valid frame, a one-pixel frame
    (at the last pixel), a frame with a -inf pose, one with a NaN in its pose, and one whose valid pixels end each 1024-pixel tile."""
    depth, poses, K = synth.synth_sens_scan(2, 8, holes=0.05, far=0.002, bad_poses=(5,))
    depth[2] = 0
    depth[3] = np.random.default_rng(1).integers(1, 65536, (480, 640))
    depth[4] = 0
    depth[4, -1, -1] = 7
    poses[6, 1, 2] = np.nan
    depth[7] = 0
    depth[7].reshape(-1)[1023::1024] = 1234
    depth[7].reshape(-1)[:3] = 65535
    return depth, poses, K


def run_gpu(depth, poses, K):
    pts, off, host, nan = pair_list.depth_to_points(torch.from_numpy(depth.view(np.int16)).to(DEV), K, torch.from_numpy(poses).to(DEV))
    assert off.cpu().tolist() == host
    return pts.cpu().numpy(), host, nan


def test_depth_to_points_is_the_restatement_bit_for_bit():
    depth, poses, K = edge_batch()
    K = pair_list.text_round_trip(K)
    got, host, nan = run_gpu(depth, poses, K)
    want = [sens_cpu.depth_to_points(depth[f], K, poses[f]) for f in range(len(depth))]
    assert host == np.concatenate([[0], np.cumsum([len(w) for w in want])]).tolist()
    assert nan == [bool(np.isnan(w).any()) for w in want] == [False] * 5 + [True, True, False]
    assert [len(w) for w in want][2:5] == [0, 480 * 640, 1]
    w = np.concatenate(want)
    assert got.shape == w.shape and np.array_equal(got.view(np.uint64), w.view(np.uint64))


@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 7, 5), (2, 33, 31), (5, 48, 64)])
def test_depth_to_points_small_shapes(shape):
    rng = np.random.default_rng(sum(shape))
    depth = np.where(rng.random(shape) < 0.3, 0, rng.integers(1, 65536, shape)).astype(np.uint16)
    poses = np.tile(np.eye(4), (shape[0], 1, 1))
    poses[:, :3] += rng.normal(0, 1, (shape[0], 3, 4))
    K = np.array([[50.3, 0, shape[2] / 2 + 0.37, 0.01], [0, 51.7, shape[1] / 2 - 0.21, -0.02], [0, 0, 1, 0], [0, 0, 0, 1]])
    got, host, nan = run_gpu(depth, poses, K)
    want = np.concatenate([sens_cpu.depth_to_points(depth[f], K, poses[f]) for f in range(shape[0])])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)) and not any(nan)


def test_gpu_agrees_with_the_original_golden(tmp_path):
    z, pcd = golden()
    path = str(tmp_path / "scene0000_00.sens")
    open(path, "wb").write(z["sens"].tobytes())
    s = pair_list.read_sens(path, int(z["frame_skip"]))
    got, host, nan = run_gpu(s.depth, s.poses, s.intrinsic)
    check_against_original([got[host[k]:host[k + 1]] for k in range(len(s.frames))], s)
    assert host == z["offsets"].tolist() and nan == [False, False, True, False, False]


def write_scan(path, n=12, bad=(10,), seed=3, zero=(8,)):
    depth, poses, K = synth.synth_sens_scan(seed, n, width=320, height=240, frames_per_view=2, bad_poses=bad)
    for f in zero:
        depth[f] = 0
    synth.write_sens(path, depth, poses, K, seed=seed)


def read_dir(d):
    """{file: bytes}, an npz file as the bytes of its `pcd` array (the zip container holds the time it was written)."""
    return {f: np.load(os.path.join(d, f))["pcd"].tobytes() if f.endswith(".npz") else open(os.path.join(d, f), "rb").read()
            for f in sorted(os.listdir(d))}


def test_extract_scene_writes_the_restatement_and_the_overlap(tmp_path):
    sens = str(tmp_path / "scene0002_00.sens")
    write_scan(sens)
    out = str(tmp_path / "out" / "scene0002_00")
    M, names, secs = pair_list.extract_scene(sens, out, 2, 0.05)
    pcd = os.path.join(out, "pcd")
    s = pair_list.read_sens(sens, 2)
    assert sorted(os.listdir(pcd)) == sorted([f"{f}.npz" for f in s.frames] + ["overlap.txt"])
    for k, f in enumerate(s.frames):
        got = np.load(os.path.join(pcd, f"{f}.npz"))["pcd"]
        want = sens_cpu.depth_to_points(s.depth[k], s.intrinsic, s.poses[k])
        assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got.view(np.uint64), want.view(np.uint64))
    # of the kept frames 0, 2, ..., 10, frame 8 (no point) and frame 10 (NaN from its -inf pose) are left out of the overlap
    assert names == sorted(os.path.join(pcd, f"{f}.npz") for f in (0, 2, 4, 6)) and set(secs) == {"gpu", "write", "overlap"}
    ours = open(os.path.join(pcd, "overlap.txt"), "rb").read()
    M2, names2 = pair_list.compute_full_overlapping(pcd, 0.05)
    assert names2 == names and np.array_equal(M, M2) and open(os.path.join(pcd, "overlap.txt"), "rb").read() == ours and ours


def test_chunk_size_does_not_change_the_outputs(tmp_path, monkeypatch):
    sens = str(tmp_path / "scene0003_00.sens")
    write_scan(sens, n=15, bad=(4,), zero=(6, 7))
    outs = []
    for chunk in (1, 7, 15):
        monkeypatch.setattr(pair_list, "EXTRACT_CHUNK", chunk)
        out = str(tmp_path / f"c{chunk}")
        pair_list.extract_scene(sens, out, 1, 0.05)
        files = read_dir(os.path.join(out, "pcd"))
        files["overlap.txt"] = files["overlap.txt"].replace(out.encode(), b"")
        outs.append(files)
    assert outs[0] == outs[1] == outs[2] and len(outs[0]) == 16


def test_extract_ignores_stale_frames(tmp_path):
    sens = str(tmp_path / "scene0004_00.sens")
    write_scan(sens, n=4, bad=(), zero=())
    out = str(tmp_path / "scene0004_00")
    os.makedirs(os.path.join(out, "pcd"))
    np.savez(os.path.join(out, "pcd", "999.npz"), pcd=np.zeros((5, 3)))
    M, names, _ = pair_list.extract_scene(sens, out, 1, 0.05)
    assert len(names) == 4 and "999.npz" not in open(os.path.join(out, "pcd", "overlap.txt")).read()


def test_extract_scenes_stops_at_a_truncated_scene(tmp_path):
    paths = []
    for k in range(3):
        p = str(tmp_path / "scans" / f"scene000{k}_00" / f"scene000{k}_00.sens")
        os.makedirs(os.path.dirname(p))
        write_scan(p, n=6, bad=(), zero=(), seed=10 + k)
        paths.append(p)
    data = open(paths[1], "rb").read()
    open(paths[1], "wb").write(data[:len(data) // 2])
    target = str(tmp_path / "target")
    before = threading.active_count()
    with pytest.raises(ValueError, match="scene0001_00.sens: truncated"):
        pair_list.extract_scenes(paths, target, 2, 0.05, log=None)
    assert threading.active_count() == before
    assert sorted(os.listdir(os.path.join(target, "scene0000_00", "pcd"))) == ["0.npz", "2.npz", "4.npz", "overlap.txt"]
    assert len(open(os.path.join(target, "scene0000_00", "pcd", "overlap.txt")).read().splitlines()) == 3
    assert not os.path.exists(os.path.join(target, "scene0001_00")) and not os.path.exists(os.path.join(target, "scene0002_00"))


def test_cli_extract_then_list_is_overlap_then_list(tmp_path):
    paths = []
    for k in range(2):
        p = str(tmp_path / "scans" / f"scene001{k}_00.sens")
        os.makedirs(os.path.dirname(p), exist_ok=True)
        write_scan(p, n=10, bad=(), zero=(), seed=20 + k)
        paths.append(p)
    target = str(tmp_path / "target")
    pair_list.main(["extract", "--target_dir", target, "--frame_skip", "2"] + paths)
    listed = pair_list.generate_list(target)
    ours = open(listed, "rb").read()
    scenes = [os.path.join(target, f"scene001{k}_00", "pcd") for k in range(2)]
    extracted = [open(os.path.join(d, "overlap.txt"), "rb").read() for d in scenes]
    pair_list.main(["overlap", "--input_path"] + scenes)
    pair_list.main(["list", "--target_dir", target])
    assert [open(os.path.join(d, "overlap.txt"), "rb").read() for d in scenes] == extracted
    assert open(listed, "rb").read() == ours and ours


def test_depth_to_points_argument_errors():
    lib = _lib.lib
    F, H, W = 3, 48, 64
    depth = torch.ones(F, H, W, dtype=torch.int16, device=DEV)
    poses = torch.eye(4, dtype=torch.float64, device=DEV).repeat(F, 1, 1).contiguous()
    out = torch.empty(F * H * W, 3, dtype=torch.float64, device=DEV)
    off = torch.empty(F + 1, dtype=torch.int64, device=DEV)
    host, nan = (ctypes.c_int64 * (F + 1))(), (ctypes.c_int32 * F)()
    st = torch.cuda.current_stream().cuda_stream
    _lib.stream()
    wsb = lib.pcb_depth_to_points_ws_bytes(F, H, W)
    ws = torch.full((wsb + (1 << 20),), 0xA5, dtype=torch.uint8, device=DEV)

    def call(d=depth.data_ptr(), f=F, h=H, w=W, p=poses.data_ptr(), o=out.data_ptr(), b=wsb):
        return lib.pcb_depth_to_points(d, f, h, w, 1.0, 1.0, 0.5, 0.5, 0.0, 0.0, p, o, off.data_ptr(), host, nan, ws.data_ptr(), b, st)
    assert call(b=wsb - 1) == 2
    assert call() == 0
    torch.cuda.synchronize()
    assert bool((ws[wsb:] == 0xA5).all()), "bytes at or beyond the query were written"
    assert list(host) == [0, H * W, 2 * H * W, 3 * H * W] and list(nan) == [0, 0, 0]
    for bad in (dict(f=0), dict(f=4097), dict(h=0), dict(w=1 << 15 | 1), dict(d=None), dict(p=None), dict(o=None)):
        assert call(**bad) == 2, bad
    assert lib.pcb_depth_to_points_ws_bytes(0, H, W) == 0 and lib.pcb_depth_to_points_ws_bytes(F, 0, W) == 0
    with pytest.raises(_lib.PcbError, match="uint16"):
        pair_list.depth_to_points(depth.float(), np.eye(4), poses)
    with pytest.raises(_lib.PcbError, match="poses"):
        pair_list.depth_to_points(depth, np.eye(4), poses[:2])
