"""Host checks of the semseg data-path oracle (oracle/semseg_data_cpu.py): it replays the reference's own augmentation
(tests/golden/semseg_augment.npz, written by tests/golden/make_semseg_golden.py) from the recorded draws, its blur and interpolation
equal scipy's bit for bit; plus the PLY reader and the argument checks of the new pcb_* entry points, which need no GPU."""
import ctypes
import os

import numpy as np
import pytest
import scipy.interpolate
import scipy.ndimage

from oracle import semseg_data_cpu as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "semseg_augment.npz")
PARAMS = {"scannet2cm": O.SCANNET_2CM, "stanford": O.STANFORD}


@pytest.mark.parametrize("s", [0, 1])
def test_oracle_replays_the_reference_augmentation(s):
    z = np.load(GOLDEN)
    pre = f"s{s}_"
    p = PARAMS[str(z[pre + "name"])]
    out = O.run_scene(z[pre + "xyz"], z[pre + "rgb"].astype(np.float32), z[pre + "label"].astype(np.int32), p,
                      O.Replay(O.read_draws(z, pre)))
    for k in ("vox_coords", "vox_labels", "coords", "labels"):
        assert out[k].shape == z[pre + k].shape and (out[k] == z[pre + k]).all(), k
    for k in ("elastic", "vox_feats", "feats", "transformation"):
        assert out[k].shape == z[pre + k].shape
        assert np.abs(out[k].astype(np.float64) - z[pre + k]).max() <= 1e-12 * max(1.0, np.abs(z[pre + k]).max()), k


def test_golden_covers_the_branches():
    z = np.load(GOLDEN)
    k0 = list(z["s0_kinds"])
    assert k0[:3] == ["random", "randn", "randn"] and "choice" in k0          # elastic distortion (2 rounds), dropout
    assert len(z["s0_coords"]) < len(z["s0_vox_coords"])
    assert str(z["s1_name"]) == "stanford" and len(z["s1_xyz"]) > len(z["s1_vox_coords"])
    for s in (0, 1):
        lab = z[f"s{s}_vox_labels"]
        assert (lab == 255).any() and (lab != 255).any()                      # mixed-label voxels became ignore_label


def test_blur_and_interpolation_equal_scipy():
    rng = np.random.default_rng(3)
    coords = (rng.random((5000, 3)) * np.array([4.0, 3.0, 2.0])).astype(np.float32)
    for g in (0.2, 0.8):
        noise_dim, cmin = O.noise_shape(coords, g)
        noise = rng.standard_normal((*noise_dim, 3)).astype(np.float32)
        ref = noise
        for _ in range(2):
            for shape in ((3, 1, 1, 1), (1, 3, 1, 1), (1, 1, 3, 1)):
                ref = scipy.ndimage.convolve(ref, np.ones(shape).astype("float32") / 3, mode="constant", cval=0)
        blurred = O.smooth_noise(noise)
        assert blurred.dtype == np.float32 and np.array_equal(blurred, ref)
        axes = O.grid_axes(cmin, g, noise_dim)
        q = np.concatenate([coords, coords[:50] + 10, coords[:50] - 10])                  # includes points outside the grid
        ip = scipy.interpolate.RegularGridInterpolator(axes, ref, bounds_error=0, fill_value=0)
        assert np.array_equal(O.interpolate(axes, blurred, q), ip(q))


def test_sparse_quantize_label_semantics():
    c = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [1, 0, 0], [2, 0, 0], [2, 0, 0], [3, 0, 0], [3, 0, 0], [-1, 5, 0]], np.int32)
    lab = np.array([4, 7, 4, 8, 255, 255, 255, 6, 2])
    coords, feats, labels = O.sparse_quantize(c, np.arange(9)[:, None], labels=lab, ignore_label=255)
    assert coords.tolist() == [[-1, 5, 0], [0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]]
    assert feats[:, 0].tolist() == [8, 0, 1, 4, 6]
    assert labels.tolist() == [2, 4, 255, 255, 255]            # agree / mixed / all ignore / ignore + one real label


def _write_ply(path, v):
    types = {"<f4": "float", "|u1": "uchar"}
    head = ["ply", "format binary_little_endian 1.0", "comment written by the test", f"element vertex {len(v)}"]
    head += [f"property {types[v.dtype[n].str]} {n}" for n in v.dtype.names]
    with open(path, "wb") as f:
        f.write(("\n".join(head + ["end_header"]) + "\n").encode("ascii"))
        f.write(v.tobytes())


@pytest.mark.parametrize("with_label", [True, False])
def test_read_ply_round_trip(tmp_path, with_label):
    from pointcontrast_b200.semseg_data import read_ply
    rng = np.random.default_rng(1)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")] + ([("label", "u1")] if with_label else [])
    v = np.empty(777, dtype=fields)
    for n, t in fields:
        v[n] = rng.normal(size=777).astype(np.float32) if t == "<f4" else rng.integers(0, 256, 777)
    _write_ply(tmp_path / "a.ply", v)
    got = read_ply(tmp_path / "a.ply")
    assert got.dtype.names == v.dtype.names and np.array_equal(got, v)
    (tmp_path / "b.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nend_header\n1\n")
    with pytest.raises(ValueError):
        read_ply(tmp_path / "b.ply")


def test_semseg_entry_points_reject_bad_arguments_without_a_gpu():
    from pointcontrast_b200 import _lib
    L = _lib.lib
    m = ctypes.c_int64(0)
    lo, hi = (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    T = (ctypes.c_double * 16)()
    mn = (ctypes.c_int32 * 3)()
    bad = [
        L.pcb_voxelize_labels(None, None, -1, 255, None, None, None, ctypes.byref(m), None, 0, None),          # n < 0
        L.pcb_voxelize_labels(None, None, 10, 255, None, None, None, ctypes.byref(m), None, 0, None),          # null pointers
        L.pcb_point_bounds(None, 0, lo, hi, None, 0, None),                                                     # n == 0
        L.pcb_elastic_distort(None, 10, None, 1, 5, 5, None, 1.0, None, 0, None),                               # grid dim < 2
        L.pcb_elastic_distort(None, 10, None, 5, 5, 5, None, 1.0, None, 0, None),                               # null pointers
        L.pcb_affine_floor(None, 10, T, None, mn, None, 0, None),
        L.pcb_semseg_input_transform(None, None, 10, 1, 0, 0.0, None, None, 0.0, 0, None, 0, None),             # flip needs coords
        L.pcb_semseg_input_transform(None, None, 10, 8, 0, 0.0, None, None, 0.0, 0, None, 0, None),             # flip bit 3
    ]
    assert bad == [2] * len(bad) and b"bad argument" in L.pcb_last_error()
    assert L.pcb_voxelize_labels(None, None, 0, 255, None, None, None, ctypes.byref(m), None, 0, None) == 0 and m.value == 0
    assert L.pcb_voxelize_labels_ws_bytes(1000) >= 1000 * 24
    assert L.pcb_elastic_distort_ws_bytes(50, 50, 20) >= 50 * 50 * 20 * 3 * 4
