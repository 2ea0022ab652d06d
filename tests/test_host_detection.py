"""Sparse-conv detection backbone, host side (pointcontrast_b200/detection.py, DESIGN.md 8f-7): the new C entry points are exported and
reject bad arguments before touching the device, the numpy oracle's batched voxelisation against an independent first-occurrence
restatement, the three names `me` adds for the original model package, and our backbone network against the original's, module by
module."""
import importlib
import sys

import numpy as np
import pytest

from oracle import detection_cpu, detection_ref

NEW = ("pcb_voxelize_scenes_ws_bytes", "pcb_voxelize_scenes", "pcb_furthest_point_sampling_ragged_ws_bytes",
       "pcb_furthest_point_sampling_ragged", "pcb_gather_rows_grad")


def original_backbone_module():
    """The staged, unmodified `models/backbone_module.py` imported against this library's `me` and `pointnet2`."""
    if not detection_ref.available():
        pytest.skip("oracle/_ref/votenet/models not staged (the original repository is absent)")
    from pointcontrast_b200 import me, pointnet2
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k in ("pointnet2_utils", "pointnet2_modules",
                                                                                         "pytorch_utils")]:
        del sys.modules[k]
    me.install()
    pointnet2.install()
    if detection_ref.ROOT not in sys.path:
        sys.path.insert(0, detection_ref.ROOT)
    return importlib.import_module("models.backbone_module")


def test_new_symbols_are_exported():
    from pointcontrast_b200 import _lib
    for name in NEW:
        assert name in _lib.EXPORTS
        getattr(_lib.lib, name)


def test_bad_arguments_return_status_2():
    import ctypes
    from pointcontrast_b200._lib import lib
    fake = 256                                   # never dereferenced: every check below fails before the device is touched
    host = (ctypes.c_int64 * 9)()
    ws = lib.pcb_voxelize_scenes_ws_bytes(8, 1000)
    assert ws > 0 and lib.pcb_voxelize_scenes_ws_bytes(0, 1000) == 0
    vox = lambda xyz, B, N, size, c, i, o, h, w, wb: lib.pcb_voxelize_scenes(xyz, B, N, size, c, i, o, h, w, wb, None)
    assert vox(fake, 0, 1000, 0.025, fake, fake, fake, host, fake, ws) == 2            # B <= 0
    assert vox(fake, -1, 1000, 0.025, fake, fake, fake, host, fake, ws) == 2
    assert vox(fake, 8, 0, 0.025, fake, fake, fake, host, fake, ws) == 2               # N <= 0
    assert vox(fake, 8, 1000, 0.0, fake, fake, fake, host, fake, ws) == 2              # voxel_size <= 0
    assert vox(fake, 8, 1000, -0.025, fake, fake, fake, host, fake, ws) == 2
    assert vox(None, 8, 1000, 0.025, fake, fake, fake, host, fake, ws) == 2            # null pointers
    assert vox(fake, 8, 1000, 0.025, None, fake, fake, host, fake, ws) == 2
    assert vox(fake, 8, 1000, 0.025, fake, None, fake, host, fake, ws) == 2
    assert vox(fake, 8, 1000, 0.025, fake, fake, None, host, fake, ws) == 2
    assert vox(fake, 8, 1000, 0.025, fake, fake, fake, None, fake, ws) == 2
    assert vox(fake, 8, 1000, 0.025, fake, fake, fake, host, None, ws) == 2
    assert vox(fake, 8, 1000, 0.025, fake, fake, fake, host, fake, ws - 1) == 2       # workspace too small
    assert vox(fake, 1 << 16, 1 << 16, 0.025, fake, fake, fake, host, fake, ws) == 2  # B * N >= 2^31

    fps = lambda xyz, off, B, M, max_n, npoint, idx, w, wb: lib.pcb_furthest_point_sampling_ragged(xyz, off, B, M, max_n, npoint, idx, w,
                                                                                                    wb, None)
    big = lib.pcb_furthest_point_sampling_ragged_ws_bytes(4, 300000, 110000)
    assert big == 300000 * 4 and lib.pcb_furthest_point_sampling_ragged_ws_bytes(4, 5000, 2000) == 0
    assert lib.pcb_furthest_point_sampling_ragged_ws_bytes(1, 50000, 110000) == 0       # a bound above M counts as M: on chip
    assert fps(fake, fake, 0, 100, 50, 16, fake, None, 0) == 2                          # B <= 0
    assert fps(fake, fake, 8, 4, 4, 16, fake, None, 0) == 2                             # fewer rows than scenes
    assert fps(fake, fake, 4, 100, 0, 16, fake, None, 0) == 2                           # max_n < 1
    assert fps(fake, fake, 4, 100, 50, 0, fake, None, 0) == 2                           # npoint < 1
    assert fps(None, fake, 4, 100, 50, 16, fake, None, 0) == 2
    assert fps(fake, None, 4, 100, 50, 16, fake, None, 0) == 2
    assert fps(fake, fake, 4, 100, 50, 16, None, None, 0) == 2
    assert fps(fake, fake, 4, 300000, 110000, 16, fake, None, 0) == 2                   # spills, no workspace
    assert fps(fake, fake, 4, 300000, 110000, 16, fake, fake, big - 1) == 2             # workspace too small

    gws = lib.pcb_points_grad_ws_bytes(1, 1000, 64)
    assert lib.pcb_gather_rows_grad(fake, fake, 64, 32, 1000, None, fake, gws, None) == 2
    assert lib.pcb_gather_rows_grad(fake, fake, 64, 32, 1000, fake, fake, gws - 1, None) == 2
    assert lib.pcb_gather_rows_grad(None, fake, 64, 32, 1000, fake, fake, gws, None) == 2
    assert lib.pcb_gather_rows_grad(fake, fake, -1, 32, 1000, fake, fake, gws, None) == 2


def first_occurrence_voxels(xyz, voxel_size):
    """Independent restatement: walk each scene's points in order, keep the first point of every new cell."""
    coords, inds, offsets = [], [], [0]
    for b, scene in enumerate(np.asarray(xyz, np.float32)):
        seen = set()
        cells = np.floor(scene / np.float32(voxel_size))
        for i, c in enumerate(cells):
            key = tuple(int(v) for v in c)
            if key not in seen:
                seen.add(key)
                coords.append((b,) + key)
                inds.append(i)
        offsets.append(len(inds))
    return np.asarray(coords, np.int32).reshape(-1, 4), np.asarray(inds, np.int32), np.asarray(offsets, np.int64)


def test_oracle_voxelisation_matches_first_occurrence_restatement():
    rng = np.random.default_rng(3)
    size = 0.025
    xyz = (rng.random((4, 3000, 3)) * np.array([1.0, 0.8, 0.5]) - 0.3).astype(np.float32)
    xyz[1] = xyz[1, rng.integers(0, 100, 3000)]                                    # heavy duplicates
    xyz[2] = np.float32(0.011)                                                     # one voxel
    xyz[3, ::2] = (rng.integers(-20, 20, (1500, 3)) * size).astype(np.float32)     # on (rounded) cell boundaries
    got = detection_cpu.voxelize_scenes(xyz, size)
    want = first_occurrence_voxels(xyz, size)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    assert got[2][3] - got[2][2] == 1


def test_me_exposes_the_sparse_conv_package_names():
    from pointcontrast_b200 import me
    assert me.convert_to_int_tensor(2, 3).tolist() == [2, 2, 2]
    assert me.convert_to_int_tensor([1, 2, 3], 3).tolist() == [1, 2, 3]
    assert me.convert_to_int_tensor(np.array([4, 5, 6]), 3).dtype.is_floating_point is False
    with pytest.raises(AssertionError):
        me.convert_to_int_tensor([1, 2], 3)
    with pytest.raises(ValueError):
        me.convert_to_int_tensor(object(), 3)
    with pytest.raises(NotImplementedError, match="CRF"):
        me.convert_region_type(None)
    with pytest.raises(NotImplementedError, match="CRF"):
        me.MinkowskiConvolutionFunction()
    with pytest.raises(NotImplementedError, match="CRF"):
        me.MinkowskiConvolutionFunction.apply()


def test_original_sparse_conv_package_imports():
    bm = original_backbone_module()
    models = importlib.import_module("models.backbone.sparseconv.models")
    assert models.load_model("Res16UNet34C") is not None and bm.SparseConvBackbone is not None


def test_backbone_network_matches_the_original_module_by_module():
    from pointcontrast_b200 import detection, me
    bm = original_backbone_module()
    cfg = importlib.import_module("models.backbone.sparseconv.config")
    models = importlib.import_module("models.backbone.sparseconv.models")
    ref = models.load_model("Res16UNet34C")(3, 256, cfg.get_config(["--conv1_kernel_size", "3"]))
    ours = detection.SparseConvBackbone()
    assert [(k, tuple(v.shape)) for k, v in ours.net.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    assert list(ours.state_dict()) == list(bm.SparseConvBackbone().state_dict())
    a, b = list(ours.net.named_modules()), list(ref.named_modules())
    assert [n for n, _ in a] == [n for n, _ in b]
    for (name, m1), (_, m2) in zip(a, b):
        assert type(m1).__name__ == type(m2).__name__ or not isinstance(m2, (me._ConvolutionBase, me.MinkowskiBatchNorm)), name
        if isinstance(m1, me._ConvolutionBase):
            assert np.asarray(m1.kernel_generator.offsets).tolist() == np.asarray(m2.kernel_generator.offsets).tolist(), name
            assert m1.kernel_generator.region_type == m2.kernel_generator.region_type, name
            assert list(m1.stride) == list(m2.stride) and m1.has_bias == m2.has_bias and m1.is_transpose == m2.is_transpose, name
        elif isinstance(m1, me.MinkowskiBatchNorm):
            assert m1.bn.momentum == m2.bn.momentum and m1.bn.eps == m2.bn.eps, name
    assert ours.net.bn0.bn.momentum == 0.02 and not ours.net.normalize_feature
    assert sum(p.numel() for p in ours.parameters()) == sum(p.numel() for p in ref.parameters())
