"""pcb_voxel_down_sample / pcb_frame_overlap and pointcontrast_b200.pair_list against the fp64 oracle (oracle/pair_list_cpu.py): points,
offsets and counts bit-exact, the written files byte-identical."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import pair_list_cpu as O
from pointcontrast_b200 import _lib, pair_list, synth
from pointcontrast_b200.config import Config
from tests.test_oracle_pair_list import boundary_frames

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def ragged(frames):
    off = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.int64)
    xyz = np.concatenate([np.asarray(f, np.float64).reshape(-1, 3) for f in frames]) if off[-1] else np.zeros((0, 3))
    return torch.from_numpy(xyz).to(DEV), torch.from_numpy(off).to(DEV)


def check_down(frames, voxel):
    xyz, off = ragged(frames)
    pts, doff, host = pair_list.voxel_down_sample(xyz, off, voxel)
    want = [O.voxel_down_sample(f, voxel) for f in frames]
    want_off = np.concatenate([[0], np.cumsum([len(w) for w in want])])
    assert host == want_off.tolist()
    assert np.array_equal(doff.cpu().numpy(), want_off)
    got = pts.cpu().numpy()
    want = np.concatenate(want) if want_off[-1] else np.zeros((0, 3))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    return pts, doff


def check_counts(frames, radius):
    pts, off = ragged(frames)
    got = pair_list.overlap_counts(pts, off, radius).cpu().numpy()
    want = O.frame_overlap_counts(frames, radius)
    assert np.array_equal(got, want)
    return got


def test_down_sample_synthetic_scans():
    frames = synth.synth_scan_frames(1, 8)
    check_down(frames, 0.05)


def test_down_sample_edge_cases():
    rng = np.random.default_rng(2)
    v = 0.05
    dup = np.repeat(rng.normal(0, 0.3, (200, 3)), 50, axis=0)
    rng.shuffle(dup)
    one_voxel = 0.31 + rng.random((5000, 3)) * 0.004
    single = [rng.normal(0, 1, (1, 3)) for _ in range(5)]
    far = rng.normal(0, 1, (3000, 3)) * 50 - 1.0e4
    check_down([dup, one_voxel] + single + [np.zeros((0, 3)), far, np.zeros((0, 3))], v)
    check_down([np.zeros((0, 3))], v)
    check_down([one_voxel], 0.013)


def test_down_sample_on_voxel_boundaries():
    """Points whose (p - lo) / v is an exact integer, or within a few ulp of one (tests/test_oracle_pair_list.py::boundary_frames,
    whose own test shows that multiplying by 1 / v would misplace some of them)."""
    frames = boundary_frames()
    for xyz, v in frames:
        check_down([xyz], v)
    rng = np.random.default_rng(3)
    check_down([rng.normal(0, 1, (500, 3)), frames[2][0], np.zeros((0, 3)), frames[2][0][::-1].copy()], 0.05)


def test_counts_consecutive_frames():
    frames = [O.voxel_down_sample(f, 0.05) for f in synth.synth_scan_frames(4, 10, points_per_frame=60_000)]
    c = check_counts(frames, 0.075)
    assert (np.diag(c) == 0).all() and (np.diag(c, 1) > 0).any()


def test_counts_across_cell_boundaries():
    """Pairs at r (1 +- 2^-40) apart straddling a cell boundary on each axis (cells of r (1 + 2^-20) from x = 0)."""
    r = 0.075
    cell = r * (1 + 2.0 ** -20)
    p, q = [], []
    for k in range(3):
        for m in range(-3, 4):
            for si, s in enumerate((1 - 2.0 ** -40, 1 + 2.0 ** -40, 1.0)):
                a = np.array([0.013, -0.021, 0.034])
                a[(k + 1) % 3] = 0.5 * (3 * si + k + 1)            # pairs at least a metre apart from each other
                a[k] = 3 * m * cell - 0.5 * r * s
                b = a.copy()
                b[k] = a[k] + r * s
                p.append(a); q.append(b)
    # pairs r (1 - 2^-40) apart that start just below (or above) the cell boundary at 0: neighbours in cells of r (1 + 2^-20), two
    # cells apart (so missed) in cells of r (1 - 2^-20) -- this pins the margin of the cell size
    small = r * (1 - 2.0 ** -20)
    for k in range(3):
        for sign in (1.0, -1.0):
            a = np.array([0.013, -0.021, 0.034])
            a[(k + 1) % 3] = -0.5 * (2 * k + (sign > 0) + 1)
            a[k] = -sign * r * 2.0 ** -22
            b = a.copy()
            b[k] = a[k] + sign * r * (1 - 2.0 ** -40)
            assert abs(np.floor(b[k] / small) - np.floor(a[k] / small)) == 2
            assert abs(np.floor(b[k] / cell) - np.floor(a[k] / cell)) == 1
            p.append(a); q.append(b)
    check_counts([np.array(p), np.array(q)], r)
    check_counts([np.array(p), np.array(q), np.array(p) + 1e-12], r)


def test_counts_small_shapes():
    rng = np.random.default_rng(5)
    one = [rng.normal(0, 0.1, (100, 3))]
    assert not check_counts(one, 0.075).any()
    check_counts([rng.normal(0, 0.1, (300, 3)), rng.normal(0.05, 0.1, (200, 3))], 0.075)
    tiny = [rng.normal(0, 0.3, (int(rng.integers(1, 6)), 3)) for _ in range(300)]
    check_counts(tiny, 0.075)
    dense = [0.01 + rng.random((int(rng.integers(20, 60)), 3)) * 0.05 for _ in range(100)]       # one cell, thousands of points
    c = check_counts(dense + [rng.normal(0, 0.1, (50, 3)) + 10.0], 0.075)                       # and a frame with no neighbour
    assert not c[-1].any() and not c[:, -1].any()


def write_scene(root, frames, scene="scene0000_00"):
    d = os.path.join(root, scene, "pcd")
    os.makedirs(d, exist_ok=True)
    for k, f in enumerate(frames):
        np.savez(os.path.join(d, f"{k * 25}.npz"), pcd=f)
    return d


def test_end_to_end_files_match_the_oracle(tmp_path):
    frames = synth.synth_scan_frames(6, 7, points_per_frame=80_000)
    bad = frames[3].copy(); bad[10, 1] = np.nan
    frames = frames[:3] + [bad, np.zeros((0, 3))] + frames[4:]
    d = write_scene(str(tmp_path), frames)
    M, names = pair_list.compute_full_overlapping(d, 0.05)
    assert len(names) == 6 and os.path.join(d, "75.npz") not in names
    gpu_overlap = open(os.path.join(d, "overlap.txt"), "rb").read()
    listed = pair_list.generate_list(str(tmp_path))
    gpu_list = open(listed, "rb").read()
    down = [O.voxel_down_sample(np.load(n)["pcd"], 0.05) for n in names]
    O.write_overlap(os.path.join(d, "overlap.txt"), names, O.frame_overlap_counts(down, 0.075), [len(x) for x in down])
    assert open(os.path.join(d, "overlap.txt"), "rb").read() == gpu_overlap
    O.write_list(str(tmp_path), [os.path.join(d, "overlap.txt")])
    assert open(listed, "rb").read() == gpu_list and gpu_list
    M2, _ = pair_list.compute_full_overlapping(d, 0.05)
    assert np.array_equal(M, M2) and open(os.path.join(d, "overlap.txt"), "rb").read() == gpu_overlap
    # the list feeds the pretraining loader
    from pointcontrast_b200.scannet_pairs import ScanNetMatchPairDataset
    cfg = Config({"data": {"voxel_size": 0.025, "dataset_root_dir": str(tmp_path), "scannet_match_dir": "overlap-30-full.txt"},
                  "trainer": {"positive_pair_search_voxel_size_multiplier": 1.5, "min_scale": 0.8, "max_scale": 1.2, "rotation_range": 360}})
    ds = ScanNetMatchPairDataset("train", config=cfg, device=DEV, manual_seed=True)
    assert len(ds) == len(gpu_list.splitlines())
    xyz0, xyz1, c0, c1, f0, f1, matches, trans = ds[0]
    assert len(xyz0) and len(xyz1) and len(matches) and trans.shape == (4, 4)


def test_cli_processes_several_scenes(tmp_path):
    a = write_scene(str(tmp_path), synth.synth_scan_frames(8, 3, points_per_frame=20_000), "sceneA")
    b = write_scene(str(tmp_path), synth.synth_scan_frames(9, 4, points_per_frame=20_000), "sceneB")
    pair_list.main(["overlap", "--input_path", a, b, "--voxel_size", "0.05"])
    pair_list.main(["list", "--target_dir", str(tmp_path)])
    assert len(open(os.path.join(a, "overlap.txt")).read().splitlines()) == 3
    assert len(open(os.path.join(b, "overlap.txt")).read().splitlines()) == 6
    assert os.path.isfile(os.path.join(str(tmp_path), "overlap-30-full.txt"))


def test_several_scenes_leave_no_reader_thread_when_one_fails(tmp_path):
    import threading
    a = write_scene(str(tmp_path), synth.synth_scan_frames(10, 3, points_per_frame=20_000), "sceneA")
    b = write_scene(str(tmp_path), synth.synth_scan_frames(11, 3, points_per_frame=20_000), "sceneB")
    before = threading.active_count()
    with pytest.raises(OSError):                     # no directory to write the missing scene's overlap.txt into
        pair_list.compute_scenes([a, str(tmp_path / "missing" / "pcd"), b], 0.05, log=None)
    assert threading.active_count() == before
    assert os.path.isfile(os.path.join(a, "overlap.txt")) and not os.path.isfile(os.path.join(b, "overlap.txt"))


def test_workspace_and_argument_errors():
    lib = _lib.lib
    frames = [O.voxel_down_sample(f, 0.05) for f in synth.synth_scan_frames(3, 4, points_per_frame=30_000)]
    xyz, off = ragged(frames)
    n, F = xyz.shape[0], len(frames)
    st = torch.cuda.current_stream().cuda_stream
    _lib.stream()
    out = torch.empty(n, 3, dtype=torch.float64, device=DEV)
    doff = torch.empty(F + 1, dtype=torch.int64, device=DEV)
    host = (ctypes.c_int64 * (F + 1))()
    counts = torch.empty(F, F, dtype=torch.int64, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    for wsf, call in ((lib.pcb_voxel_down_sample_ws_bytes,
                       lambda ws, b: lib.pcb_voxel_down_sample(xyz.data_ptr(), n, off.data_ptr(), F, 0.05, out.data_ptr(), doff.data_ptr(), host,
                                                               ws.data_ptr(), b, st)),
                      (lib.pcb_frame_overlap_ws_bytes,
                       lambda ws, b: lib.pcb_frame_overlap(xyz.data_ptr(), n, off.data_ptr(), F, 0.075, counts.data_ptr(), status.data_ptr(),
                                                           ws.data_ptr(), b, st))):
        wsb = wsf(n, F)
        ws = torch.empty(wsb + (1 << 20), dtype=torch.uint8, device=DEV)
        assert call(ws, wsb - 1) == 2
        ws.fill_(0xA5)
        assert call(ws, wsb) == 0
        torch.cuda.synchronize()
        assert bool((ws[wsb:] == 0xA5).all()), "bytes at or beyond the query were written"
        first = (out.clone(), counts.clone())
        ws.fill_(0x5A)
        assert call(ws, wsb + (1 << 20)) == 0
        torch.cuda.synchronize()
        assert torch.equal(first[0], out) and torch.equal(first[1], counts)
    assert int(status.item()) == 0
    p = xyz.data_ptr()
    ws = torch.empty(lib.pcb_voxel_down_sample_ws_bytes(n, F), dtype=torch.uint8, device=DEV)
    ws_ov = torch.empty(lib.pcb_frame_overlap_ws_bytes(n, F), dtype=torch.uint8, device=DEV)     # each call a workspace that suffices
    for args in ((p, n, off.data_ptr(), 0, 0.05), (p, n, off.data_ptr(), 4097, 0.05), (p, -1, off.data_ptr(), F, 0.05),
                 (p, n, off.data_ptr(), F, 0.0), (p, n, off.data_ptr(), F, -1.0), (None, n, off.data_ptr(), F, 0.05), (p, n, None, F, 0.05)):
        assert lib.pcb_voxel_down_sample(*args, out.data_ptr(), doff.data_ptr(), host, ws.data_ptr(), ws.numel(), st) == 2
        assert lib.pcb_frame_overlap(*args[:4], args[4] * 1.5, counts.data_ptr(), status.data_ptr(), ws_ov.data_ptr(), ws_ov.numel(), st) == 2
    assert lib.pcb_frame_overlap(p, n, off.data_ptr(), F, 0.075, None, status.data_ptr(), ws_ov.data_ptr(), ws_ov.numel(), st) == 2
    assert lib.pcb_frame_overlap(p, n, off.data_ptr(), F, 0.075, counts.data_ptr(), None, ws_ov.data_ptr(), ws_ov.numel(), st) == 2
    assert lib.pcb_frame_overlap(p, n, off.data_ptr(), F, 0.075, counts.data_ptr(), status.data_ptr(), ws_ov.data_ptr(), ws_ov.numel(), st) == 0
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert lib.pcb_voxel_down_sample_ws_bytes(n, 0) == 0 and lib.pcb_frame_overlap_ws_bytes(-1, F) == 0
    # offsets that do not cover the rows are found on the device
    bad_off = off.clone(); bad_off[-1] -= 1
    for bad in (bad_off, torch.flip(off, [0]).contiguous()):
        with pytest.raises(_lib.PcbError, match="offsets must run"):
            pair_list.voxel_down_sample(xyz, bad, 0.05)
        with pytest.raises(_lib.PcbError, match="offsets must run"):
            pair_list.overlap_counts(xyz, bad, 0.075)


@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_coordinates_are_range_errors(value):
    rng = np.random.default_rng(7)
    frames = [rng.normal(0, 1, (500, 3)), rng.normal(0, 1, (400, 3))]
    frames[1][17, 2] = value
    xyz, off = ragged(frames)
    with pytest.raises(_lib.PcbError, match="not finite"):
        pair_list.voxel_down_sample(xyz, off, 0.05)
    with pytest.raises(_lib.PcbError, match="not finite"):
        pair_list.overlap_counts(xyz, off, 0.075)
