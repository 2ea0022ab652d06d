"""Host side of the semseg preprocessing: the ScanNet converter (byte-identical to the oracle's restatement, raising where the original
asserts), the split files, the Area-5 dataset tables and the new ABI entries."""
import os
import re

import numpy as np
import pytest

from oracle import semseg_prep_cpu as O
from pointcontrast_b200 import _lib, semseg_data as S, semseg_prep as P, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_scannet_matches_the_restatement_byte_for_byte(tmp_path):
    for k, name in enumerate(("scene0270_00", "scene0270_02", "scene0384_00", "scene0002_01")):
        synth.write_scannet_raw_scene(tmp_path / "raw", "scans", name, k, n=400)
    synth.write_scannet_raw_scene(tmp_path / "raw", "scans_test", "scene0707_00", 9, n=200, labels=False)
    out = P.convert_scannet(tmp_path / "raw", tmp_path / "ours", log=None)
    O.convert_scannet(tmp_path / "raw", tmp_path / "orc")
    assert len(out) == 5
    for p in out:
        rel = os.path.relpath(p, tmp_path / "ours")
        assert p.read_bytes() == (tmp_path / "orc" / rel).read_bytes(), rel
    v = S.read_ply(tmp_path / "ours" / "train" / "scene0384_00.ply")
    assert not (v["label"] == 149).any() and (S.read_ply(tmp_path / "ours" / "train" / "scene0002_01.ply")["label"] == 149).any()
    assert not S.read_ply(tmp_path / "ours" / "test" / "scene0707_00.ply")["label"].any()


def test_scannet_raises_where_the_original_asserts(tmp_path):
    alpha = np.full(50, 255, np.uint8)
    alpha[3] = 7
    d = synth.write_scannet_raw_scene(tmp_path / "a", "scans", "scene0000_00", 0, n=50, alpha=alpha)
    with pytest.raises(ValueError, match="alpha"):
        P.scannet_scene(os.path.join(d, "scene0000_00_vh_clean_2.ply"), tmp_path)
    d = synth.write_scannet_raw_scene(tmp_path / "b", "scans", "scene0000_00", 0, n=50)
    synth.write_scannet_raw_scene(tmp_path / "c", "scans", "scene0000_00", 1, n=50)      # other vertices
    os.replace(os.path.join(tmp_path, "c", "scans", "scene0000_00", "scene0000_00_vh_clean_2.labels.ply"),
               os.path.join(d, "scene0000_00_vh_clean_2.labels.ply"))
    with pytest.raises(ValueError, match="vertices differ"):
        P.scannet_scene(os.path.join(d, "scene0000_00_vh_clean_2.ply"), tmp_path)
    synth.write_scannet_raw_scene(tmp_path / "e", "scans", "scene0000_00", 1, n=49)
    os.replace(os.path.join(tmp_path, "e", "scans", "scene0000_00", "scene0000_00_vh_clean_2.labels.ply"),
               os.path.join(d, "scene0000_00_vh_clean_2.labels.ply"))
    with pytest.raises(ValueError, match="49 vertices"):
        P.scannet_scene(os.path.join(d, "scene0000_00_vh_clean_2.ply"), tmp_path)


def test_generate_splits_lists_each_area_in_glob_order(tmp_path):
    for a, rooms in ((1, ("office_1", "hallway_2")), (5, ("conferenceRoom_1",))):
        (tmp_path / f"Area_{a}").mkdir()
        for r in rooms:
            (tmp_path / f"Area_{a}" / f"{r}.ply").write_bytes(b"")
    P.generate_splits(str(tmp_path))
    O.generate_splits(str(tmp_path), str(tmp_path / "want"))
    for i in range(1, 7):
        got = (tmp_path / "splits" / f"area{i}.txt").read_bytes()
        assert got == (tmp_path / "want" / f"area{i}.txt").read_bytes()
    assert sorted((tmp_path / "splits" / "area1.txt").read_text().split("\n")) == ["Area_1/hallway_2.ply", "Area_1/office_1.ply"]
    assert (tmp_path / "splits" / "area5.txt").read_text() == "Area_5/conferenceRoom_1.ply"
    assert (tmp_path / "splits" / "area2.txt").read_text() == ""


def test_area5_datasets_keep_the_original_tables():
    want = {"Train": ["area1.txt", "area2.txt", "area3.txt", "area4.txt", "area6.txt"], "Val": "area5.txt", "Test": "area5.txt"}
    for cls, voxel, clip in ((S.StanfordArea5Dataset, 0.05, 4), (S.StanfordArea53cmDataset, 0.03, 3.2),
                             (S.StanfordArea57d5cmDataset, 0.075, 4), (S.StanfordArea510cmDataset, 0.1, 4)):
        assert issubclass(cls, S.StanfordDataset) and cls.DATA_PATH_FILE == want
        assert (cls.VOXEL_SIZE, cls.CLIP_BOUND, cls.NUM_LABELS, cls.IGNORE_LABELS) == (voxel, clip, 14, (10,))
    assert S.StanfordDataset.DATA_PATH_FILE["Train"] == "train.txt"


def test_stanford_rooms_skip_existing_and_report_empty(tmp_path):
    synth.write_s3dis_tree(tmp_path / "in", 0, areas=(1,), rooms_per_area=2, points_per_room=60)
    (tmp_path / "out" / "Area_1").mkdir(parents=True)
    (tmp_path / "out" / "Area_1" / "office_2.ply").write_bytes(b"x")
    logs = []
    todo = P.stanford_rooms(str(tmp_path / "in"), str(tmp_path / "out"), logs.append)
    assert [os.path.basename(t[1]) for t in todo] == ["office_1.ply"]
    assert any(m.endswith("exists") for m in logs) and any(m.endswith("has 0 files.") for m in logs)
    with pytest.raises(ValueError, match="unknown S3DIS class"):
        P._class_index("Annotations/wall.txt")


def test_new_abi_entries_are_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "pcb200.h")).read()
    for name in ("pcb_text_lines_ws_bytes", "pcb_text_lines", "pcb_s3dis_parse", "pcb_ply_rows"):
        assert re.search(r"\b%s\(" % name, hdr) and name in _lib.EXPORTS
    assert (_lib.TEXT_NONASCII, _lib.LINE_KEPT, _lib.LINE_SKIPPED, _lib.LINE_HOST, _lib.LINE_ERROR) == (1, 0, 1, 2, 3)


def test_ply_header_is_the_shipped_plyfile_header():
    assert P.ply_header(3) == (b"ply\r\nformat binary_little_endian 1.0\r\nelement vertex 3\r\nproperty float x\r\nproperty float y\r\n"
                               b"property float z\r\nproperty uchar red\r\nproperty uchar green\r\nproperty uchar blue\r\n"
                               b"property uchar label\r\nend_header\r\n")
