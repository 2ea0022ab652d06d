"""The host side of the detection preprocessing (pointcontrast_b200/det_prep.py), no GPU: the restatement of `read_aggregation` and its
write lists, the meta-line and label parsing, the skip rules and the CLI's arguments."""
import json

import numpy as np
import pytest

from oracle import det_prep_cpu as O
from pointcontrast_b200 import det_prep as P, synth


def _agg(tmp_path, groups):
    p = tmp_path / "a.json"
    p.write_text(json.dumps({"segGroups": groups}))
    return str(p)


def test_read_aggregation_keeps_the_originals_aliasing(tmp_path):
    groups = [{"objectId": 0, "label": "chair", "segments": [1, 2]}, {"objectId": 1, "label": "table", "segments": [3]},
              {"objectId": 2, "label": "chair", "segments": [4]}, {"objectId": 1, "label": "bed", "segments": [5, 6]}]
    objs, labels = P.read_aggregation(_agg(tmp_path, groups))
    assert list(objs) == [1, 2, 3] and objs[1] == [1, 2, 4] and objs[2] == [5, 6] and objs[1] is labels["chair"]
    w = P.write_lists(objs, labels, {"chair": 5, "table": 7, "bed": 4})
    assert w["lab_seg"].tolist() == [1, 2, 4, 3, 5, 6] and w["lab_val"].tolist() == [5, 5, 5, 7, 4, 4]
    assert w["ins_seg"].tolist() == [1, 2, 4, 5, 6, 4] and w["ins_obj"].tolist() == [0, 0, 0, 1, 1, 2]
    assert w["obj_id"].tolist() == [1, 2, 3] and w["first_seg"].tolist() == [1, 5, 4] and w["obj_row"].tolist() == [0, 1, 2]


@pytest.mark.parametrize("groups,lmap,match", [
    ([{"objectId": 0, "label": "spaceship", "segments": [1]}], {"chair": 5}, "not in the label map"),
    ([{"objectId": 0, "label": "chair", "segments": []}], {"chair": 5}, "no segments"),
    ([{"objectId": -3, "label": "chair", "segments": [1]}], {"chair": 5}, "uint32"),
    ([{"objectId": 0, "label": "chair", "segments": [1]}], {"chair": -1}, "uint32"),
    ([{"objectId": 0, "label": "chair", "segments": [1.5]}], {"chair": 5}, "non-integer"),
])
def test_write_lists_raise_where_the_original_raises(tmp_path, groups, lmap, match):
    with pytest.raises(P.SceneError, match=match):
        P.write_lists(*P.read_aggregation(_agg(tmp_path, groups)), lmap)


def test_rows_follow_numpy_indexing(tmp_path):
    groups = [{"objectId": k, "label": "chair", "segments": [k + 10]} for k in (4, -1, 1)]
    w = P.write_lists(*P.read_aggregation(_agg(tmp_path, groups)), {"chair": 5})
    assert w["obj_row"].tolist() == [-1, 2, 1] and w["n_rows"] == 3          # id 5 is out of range, id 0 wraps to the last row


def test_meta_line_uses_the_originals_strip(tmp_path):
    p = tmp_path / "m.txt"
    p.write_text("sceneType = Bedroom\naxisAlignment = 1 0 0 2.5 0 1 0 -1 0 0 1 0.25 0 0 0 1 \naxisAlignment = 9\n")
    m = P.read_axis_alignment(str(p))
    assert m.shape == (4, 4) and m[0, 3] == 2.5 and m[1, 3] == -1 and m[3, 3] == 1
    p.write_text("colorHeight = 968\n")
    with pytest.raises(P.SceneError, match="axisAlignment"):
        P.read_axis_alignment(str(p))


def test_label_map_matches_the_oracle(tmp_path):
    lm = synth.write_scannet_label_map(str(tmp_path / "l.tsv"))
    assert P.read_label_map(lm) == O.read_label_mapping(lm) and P.read_label_map(lm)["office chair"] == 5
    (tmp_path / "i.tsv").write_text("raw_category\tnyu40id\n3\t4\n7\t9\n")
    assert P.read_label_map(str(tmp_path / "i.tsv")) == {3: 4, 7: 9} == O.read_label_mapping(str(tmp_path / "i.tsv"))


def test_sunrgbd_labels_and_boxes(tmp_path):
    p = tmp_path / "l.txt"
    p.write_text("chair 1 2 3 4 0.5 1.5 -0.25 0.3 0.4 0.5 0.6 -0.8\nlamp 1 2 3 4 0 0 0 1 1 1 1 0\nbed 1 2 3 4 1 1 1 0 2 3 0 1\n")
    objs = P.read_sunrgbd_label(str(p))
    assert [o[0] for o in objs] == [o[0] for o in O.read_objects(str(p))] == ["chair", "lamp", "bed"]
    cls, c, l, w, h, heading = objs[0]
    assert (l, w, h) == (0.4, 0.3, 0.5) and c.tolist() == [0.5, 1.5, -0.25] and heading == -np.arctan2(-0.8, 0.6)
    obbs, rows = P.sunrgbd_boxes(objs)
    assert obbs.shape == (2, 8) and obbs[:, 7].tolist() == [3, 0] and np.array_equal(obbs, O.boxes(O.read_objects(str(p))))
    assert rows[1, 6] == np.cos(-1 * obbs[1, 6]) and rows[1, 7] == np.sin(-1 * obbs[1, 6])
    assert P.sunrgbd_boxes([])[0].shape == (0, 8)


def test_scene_list_and_skip_causes(tmp_path):
    lm = synth.write_scannet_label_map(str(tmp_path / "l.tsv"))
    for k, fault in enumerate((None, "no_align", "unknown_label", "no_segments", "vertex_count")):
        synth.write_scannet_det_raw_scene(str(tmp_path / "scans"), "scene%04d_00" % k, k, n=400, n_seg=30, fault=fault)
    (tmp_path / "scans" / "notes").mkdir()
    assert P.scannet_scenes(str(tmp_path / "scans")) == ["scene%04d_00" % k for k in range(5)]
    lmap = P.read_label_map(lm)
    assert P.load_scene(str(tmp_path / "scans"), "scene0000_00", lmap)["vert"].shape == (400, 6)
    for k in range(1, 5):
        with pytest.raises(P.SceneError):
            P.load_scene(str(tmp_path / "scans"), "scene%04d_00" % k, lmap)


def test_cli_arguments():
    with pytest.raises(SystemExit):
        P.main(["scannet", "--scans", "x", "--output", "y"])                # --label_map is required
    with pytest.raises(SystemExit):
        P.main(["sunrgbd", "--output", "y"])
    with pytest.raises(SystemExit):
        P.main(["kitti"])
