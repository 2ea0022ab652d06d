"""pointcontrast_b200.det_data without a device: argument errors, scan-name selection, DetectionLoader batching and the ctypes layout
of `struct pcb_det_batch`."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from pointcontrast_b200 import _lib, build, det_data, synth

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pcb200.h")


class ScannetConfig:
    nyu40ids = np.array(synth.SCANNET_NYU40IDS)
    mean_size_arr = np.ones((18, 3))
    num_heading_bin = 1
    type2class = {str(i): i for i in range(18)}


class SunConfig:
    mean_size_arr = np.ones((10, 3))
    num_heading_bin = 12
    type2class = {str(i): i for i in range(10)}


@pytest.fixture
def scannet_dir(tmp_path):
    for j, name in enumerate(("scene0000_00", "scene0001_00", "scene0003_00")):
        synth.write_scannet_detection_scene(str(tmp_path), name, j, 50, 2)
    split = tmp_path / "scannetv2_train.txt"
    split.write_text("scene0000_00\nscene0001_00\nscene0002_00\nscene0003_00\n")
    return tmp_path, split


def test_scannet_errors(scannet_dir):
    d, split = scannet_dir
    with pytest.raises(ValueError):
        det_data.ScannetDetectionDataset(use_color=True, data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(),
                                         device="cpu")
    with pytest.raises(ValueError):
        det_data.ScannetDetectionDataset("bogus", data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(), device="cpu")
    ds = det_data.ScannetDetectionDataset(num_points=20, data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(),
                                          device="cpu")
    too_many = {"vert": np.zeros((5, 6), np.float32), "sem": np.zeros(5, np.uint32), "ins": np.zeros(5, np.uint32),
                "bbox": np.tile([[0, 0, 0, 1, 1, 1, 3]], (65, 1)).astype(np.float64)}
    with pytest.raises(ValueError, match="MAX_NUM_OBJ"):
        ds._assemble([too_many], [0])
    bad_id = dict(too_many, bbox=np.array([[0, 0, 0, 1, 1, 1, 2.0]]))
    with pytest.raises(ValueError, match="nyu40"):
        ds._assemble([bad_id], [0])


def test_sunrgbd_errors(tmp_path):
    synth.write_sunrgbd_detection_scene(str(tmp_path), "000001", 0, 50, 2)
    with pytest.raises(ValueError):
        det_data.SunrgbdDetectionVotesDataset(num_points=50001, data_path=str(tmp_path), dataset_config=SunConfig(), device="cpu")
    ds = det_data.SunrgbdDetectionVotesDataset(num_points=20, data_path=str(tmp_path), dataset_config=SunConfig(), device="cpu")
    item = ds._read("000001")
    item["bbox"][0, 7] = 10
    with pytest.raises(ValueError, match="class"):
        ds._assemble([item], [0])
    with pytest.raises(ValueError, match="voxel_size"):
        det_data.DetectionLoader(det_data.SunrgbdDetectionVotesDataset(use_height=True, data_path=str(tmp_path),
                                                                       dataset_config=SunConfig(), device="cpu"), 2, False, 0.025)


def test_scan_name_selection(scannet_dir, tmp_path_factory):
    d, split = scannet_dir
    ds = det_data.ScannetDetectionDataset(data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(), device="cpu")
    assert ds.scan_names == ["scene0000_00", "scene0001_00", "scene0003_00"] and len(ds) == 3
    ds = det_data.ScannetDetectionDataset(data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(), data_ratio=0.5,
                                          device="cpu")
    assert ds.scan_names == ["scene0000_00"]
    s = tmp_path_factory.mktemp("sun")
    for name in ("000005", "000002", "000009", "000001"):
        synth.write_sunrgbd_detection_scene(str(s), name, 1, 20, 1)
    ds = det_data.SunrgbdDetectionVotesDataset(data_path=str(s), dataset_config=SunConfig(), device="cpu")
    assert ds.scan_names == ["000001", "000002", "000005", "000009"]
    ds = det_data.SunrgbdDetectionVotesDataset(data_path=str(s), dataset_config=SunConfig(), scan_idx_list=[3, 1, 0], data_ratio=0.7,
                                               device="cpu")
    assert ds.scan_names == ["000009", "000002"]


def test_loader_len_and_short_last_batch(scannet_dir):
    d, split = scannet_dir
    ds = det_data.ScannetDetectionDataset(data_path=str(d), split_file=str(split), dataset_config=ScannetConfig(), device="cpu")
    seen = []
    ds._assemble = lambda items, idxs: seen.append(list(idxs)) or {"n": len(items)}
    loader = det_data.DetectionLoader(ds, 2, shuffle=False)
    assert len(loader) == 2
    assert [b["n"] for b in loader] == [2, 1] and seen == [[0, 1], [2]]
    loader = det_data.DetectionLoader(ds, 2, shuffle=True)
    seen.clear()
    list(loader)
    assert sorted(sum(seen, [])) == [0, 1, 2] and [len(s) for s in seen] == [2, 1]


def test_det_batch_layout_matches_the_c_compiler(tmp_path):
    cls, cname = _lib.PcbDetBatch, "pcb_det_batch"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcb200.h"', "int main(void) {",
             f'  printf("sizeof %zu 0\\n", sizeof(struct {cname}));']
    for field, _ in cls._fields_:
        lines.append(f'  printf("{field} %zu %zu\\n", offsetof(struct {cname}, {field}), sizeof(((struct {cname}*)0)->{field}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines) + "\n")
    cc = shutil.which("cc") or shutil.which(build.NVCC)
    assert cc
    subprocess.run([cc, "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "abi")], check=True, capture_output=True, text=True)
    out = subprocess.run([str(tmp_path / "abi")], check=True, capture_output=True, text=True).stdout
    c = [(f, int(o), int(s)) for f, o, s in (line.split() for line in out.splitlines())]
    py = [("sizeof", ctypes.sizeof(cls), 0)] + [(f, getattr(cls, f).offset, getattr(cls, f).size) for f, _ in cls._fields_]
    assert py == c


def _batch(offsets, box_offsets, **fields):
    """A pcb_det_batch whose device pointers are placeholders: every call below must be refused by the host-side argument checks."""
    a = _lib.PcbDetBatch()
    a.B, a.M, a.num_points, a.dataset = len(offsets) - 1, int(offsets[-1]), 4, _lib.DET_SCANNET
    a.offsets_host, a.box_offsets_host = offsets.ctypes.data, box_offsets.ctypes.data
    dummy = 256
    for name in ("offsets", "box_offsets", "params", "choices", "vert", "sem", "ins", "boxes", "nyu40ids", "mean_size", "point_clouds",
                 "pcl_color", "vote_label", "vote_label_mask", "center_label", "heading_class_label", "heading_residual_label",
                 "size_class_label", "size_residual_label", "sem_cls_label", "box_label_mask"):
        setattr(a, name, dummy)
    a.n_ids, a.n_size, a.num_heading_bin = 18, 18, 1
    for k, v in fields.items():
        setattr(a, k, v)
    return a


def _refused(rc, cause):
    assert rc == _lib.ERR_ARG
    assert cause in _lib.lib.pcb_last_error().decode()


def test_entry_points_refuse_bad_arguments_before_launching():
    good = np.array([0, 5, 10], np.int64)
    backwards = np.array([0, 6, 4, 10], np.int64)
    empty_scene = np.array([0, 5, 5, 10], np.int64)
    boxes = np.array([0, 3, 7], np.int64)
    lib = _lib.lib
    # offsets that are not monotone, or an empty scene
    for off in (backwards, empty_scene):
        _refused(lib.pcb_det_floor_height(256, 6, 0, off.ctypes.data, 256, len(off) - 1, 256, None), "offsets_ok")
        _refused(lib.pcb_det_choices(off.ctypes.data, 256, len(off) - 1, 4, 0, 0, 256, 256, 1 << 30, None), "offsets_ok")
        a = _batch(off, np.zeros(len(off), np.int64))
        _refused(lib.pcb_det_points(ctypes.byref(a), 256, 1 << 30, None), "batch_ok")
        _refused(lib.pcb_det_boxes(ctypes.byref(a), None), "batch_ok")
    # more than 64 boxes in a scene, box offsets that go backwards
    for boff in (np.array([0, 65, 66], np.int64), np.array([0, 3, 2], np.int64)):
        _refused(lib.pcb_det_boxes(ctypes.byref(_batch(good, boff)), None), "box_offsets")
    # NULL pointers and a short workspace
    _refused(lib.pcb_det_points(ctypes.byref(_batch(good, boxes, choices=None)), 256, 1 << 30, None), "choices")
    _refused(lib.pcb_det_points(ctypes.byref(_batch(good, boxes, ins=None)), 256, 1 << 30, None), "ins")
    _refused(lib.pcb_det_points(ctypes.byref(_batch(good, boxes)), 256, 16, None), "ws_bytes")
    _refused(lib.pcb_det_boxes(ctypes.byref(_batch(good, boxes, center_label=None)), None), "center_label")
    _refused(lib.pcb_det_choices(good.ctypes.data, 256, 2, 4, 0, 0, None, 256, 1 << 30, None), "out")
    _refused(lib.pcb_det_choices(good.ctypes.data, 256, 2, 4, 0, 0, 256, 256, 16, None), "ws_bytes")
    _refused(lib.pcb_det_floor_height(None, 6, 0, good.ctypes.data, 256, 2, 256, None), "z")


def test_replayed_choice_sets_must_lie_in_their_scenes():
    from pointcontrast_b200.semseg_data import ReplayDraws
    with pytest.raises(ValueError, match="outside"):
        ReplayDraws([("choices", [np.array([0, 4]), np.array([1, 7])])], device="cpu").choices([5, 7], 2)
    assert ReplayDraws([("choices", [np.array([0, 4]), np.array([1, 6])])], device="cpu").choices([5, 7], 2).shape == (2, 2)
