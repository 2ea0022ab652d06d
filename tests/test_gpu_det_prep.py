"""VoteNet detection preprocessing on the GPU (pcb_scannet_annotate, pcb_sunrgbd_votes through det_prep) against the numpy restatement
(oracle/det_prep_cpu.py) exactly, against the original's outputs (tests/golden/det_prep.npz), and end to end through the CLI into
det_data.DetectionLoader."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import det_prep_cpu as O
from pointcontrast_b200 import det_data, det_prep as P, synth
from tests.golden.make_det_prep_golden import SCENES, SEED, digests
from tests.test_oracle_det_prep import FAULTS, same_files, scannet_tree, sunrgbd_outputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "det_prep.npz")
DEV = torch.device("cuda")


def _annotate(scans, name, lm):
    scene = P.load_scene(scans, name, P.read_label_map(lm))
    vert, sem, ins, bbox = P.annotate(scene, DEV)
    return vert.cpu().numpy(), sem.cpu().numpy().view(np.uint32), ins.cpu().numpy().view(np.uint32), bbox


def _oracle(scans, name, lm):
    d = os.path.join(scans, name)
    return O.export(os.path.join(d, name + "_vh_clean_2.ply"), os.path.join(d, name + ".aggregation.json"),
                    os.path.join(d, name + "_vh_clean_2.0.010000.segs.json"), os.path.join(d, name + ".txt"), O.read_label_mapping(lm))


@pytest.mark.parametrize("n,n_seg,n_obj", [(1, 1, 1), (255, 12, 8), (257, 200, 12), (4097, 700, 40), (150000, 3000, 40)])
def test_scannet_annotate_matches_the_oracle(tmp_path, n, n_seg, n_obj):
    lm = synth.write_scannet_label_map(str(tmp_path / "labels.tsv"))
    if n < 20:                                          # the writer's quirks need a few objects and segments
        _tiny(tmp_path, lm)
        return
    synth.write_scannet_det_raw_scene(str(tmp_path / "scans"), "scene0000_00", n, n=n, n_seg=n_seg, n_obj=n_obj)
    got, want = _annotate(str(tmp_path / "scans"), "scene0000_00", lm), _oracle(str(tmp_path / "scans"), "scene0000_00", lm)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g.view(np.uint8), w.view(np.uint8))


def _tiny(tmp_path, lm):
    """Three vertices: one instance meeting both signed zeros, one with a NaN coordinate."""
    import json
    d = tmp_path / "scans" / "scene0009_00"
    d.mkdir(parents=True)
    xyz = np.array([[0.0, 1.0, 1.0], [-0.0, -1.0, -1.0], [0.5, 0.25, np.nan]], np.float32)
    synth.write_ply(str(d / "scene0009_00_vh_clean_2.ply"), xyz, np.zeros((3, 3), np.uint8))
    (d / "scene0009_00.txt").write_text("axisAlignment = 1 0 0 -0 0 1 0 -0 0 0 1 -0 0 0 0 1\n")
    (d / "scene0009_00_vh_clean_2.0.010000.segs.json").write_text(json.dumps({"segIndices": [5, 5, 9]}))
    (d / "scene0009_00.aggregation.json").write_text(json.dumps({"segGroups": [
        {"objectId": 0, "label": "chair", "segments": [5]}, {"objectId": 1, "label": "bed", "segments": [9]}]}))
    got, want = _annotate(str(tmp_path / "scans"), "scene0009_00", lm), _oracle(str(tmp_path / "scans"), "scene0009_00", lm)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g, w, equal_nan=True)
    b = got[3]
    assert np.signbit(got[0][1, 0]) and np.isfinite(b[0]).all() and np.isnan(b[1, :6]).all()


@pytest.mark.parametrize("fault", [f for f in FAULTS if f])
def test_scannet_skips_where_the_original_raises(tmp_path, fault):
    lm = synth.write_scannet_label_map(str(tmp_path / "labels.tsv"))
    synth.write_scannet_det_raw_scene(str(tmp_path / "scans"), "scene0000_00", 3, fault=fault)
    with pytest.raises(Exception):
        _oracle(str(tmp_path / "scans"), "scene0000_00", lm)
    with pytest.raises(Exception):
        _annotate(str(tmp_path / "scans"), "scene0000_00", lm)


def test_sunrgbd_votes_match_the_oracle_across_batches():
    rng = np.random.default_rng(1)
    pcs, objs_all = [], []
    for b in range(9):
        n = (0, 1, 255, 256, 257, 4097, 20000, 3, 50000)[b]
        c0 = rng.uniform(-1, 1, 3)
        pc = np.concatenate([c0 + rng.uniform(-1.5, 1.5, (n, 3)), rng.random((n, 3))], 1)
        objs = []
        for k in range(int(rng.integers(0, 12)) if b != 0 else 0):
            size = rng.uniform(0.1, 1.2, 3)
            if k == 3:
                size[0] = 0.0                           # skipped (Qhull raises)
            if k == 4:
                size[2] = 1e-9
            objs.append((("chair", "bed", "lamp", "table")[k % 4], c0 + rng.uniform(-0.3, 0.3, 3), *size, rng.uniform(-np.pi, np.pi)))
        if n >= 8:                                      # points exactly on the faces of an axis-aligned dyadic box
            objs.append(("desk", np.array([0.5, 0.25, 0.125]), 0.25, 0.5, 0.125, -0.0))
            pc[:6, :3] = np.array([0.5, 0.25, 0.125]) + np.array([[0.25, 0, 0], [-0.25, 0, 0], [0, 0.5, 0], [0, -0.5, 0], [0, 0, 0.125],
                                                                   [0.25, 0.5, -0.125]])
        pcs.append(pc)
        objs_all.append(objs)
    rows = [P.sunrgbd_boxes(o)[1] for o in objs_all]
    got = P.sunrgbd_votes(pcs, rows, DEV)
    for pc, objs, g in zip(pcs, objs_all, got):
        w = O.votes(pc, objs)
        assert g.shape == w.shape and np.array_equal(g, w)
    assert sum(int((g[:, 0] == 1).sum()) for g in got) > 1000
    assert all(got[8][:6, 0] == 1)


def test_golden_original_output(tmp_path):
    z = np.load(GOLDEN)
    data, off = z["data"].tobytes(), z["off"]
    for k, rel in enumerate(z["paths"].tolist()):
        p = tmp_path / "in" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(data[off[k]:off[k + 1]])
    np.random.seed(SEED)
    secs = P.convert_scannet(str(tmp_path / "in" / "scans"), str(tmp_path / "out" / "scannet"), str(tmp_path / "in" / "labels.tsv"),
                             scan_list=None, log=None)
    assert secs["failed"] == [n for n, f in SCENES if f]
    P.convert_sunrgbd(str(tmp_path / "in" / "sunrgbd_trainval"), str(tmp_path / "out" / "sunrgbd"), v1=True, log=None)
    assert digests(str(tmp_path / "out")) == dict(zip(z["outputs"].tolist(), z["sha"].tolist()))


def test_cli_end_to_end_and_loaders(tmp_path):
    scans, lm, names = scannet_tree(str(tmp_path / "scannet_in"), n=3000, big=60000)
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    cmd = [sys.executable, "-m", "pointcontrast_b200.det_prep", "scannet", "--scans", scans, "--label_map", lm, "--scan_list",
           str(tmp_path / "list.txt"), "--output", str(tmp_path / "ours_sc"), "--seed", "7"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, check=True)
    assert r.stdout.count("Failed export scan") == sum(1 for f in FAULTS if f)
    np.random.seed(7)
    O.convert_scannet(scans, str(tmp_path / "orc_sc"), lm, names)
    files = sorted(os.listdir(tmp_path / "orc_sc"))
    assert sorted(os.listdir(tmp_path / "ours_sc")) == files and len(files) == 8
    same_files(tmp_path / "ours_sc", tmp_path / "orc_sc", files)
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, check=True)
    assert r.stdout.count("already exists") == 2

    synth.write_sunrgbd_export(str(tmp_path / "sun_in"), 9)
    subprocess.run([sys.executable, "-m", "pointcontrast_b200.det_prep", "sunrgbd", "--input", str(tmp_path / "sun_in"), "--output",
                    str(tmp_path / "ours_sun"), "--v2", "--seed", "8"], cwd=ROOT, capture_output=True, text=True, check=True)
    np.random.seed(8)
    O.convert_sunrgbd(str(tmp_path / "sun_in"), str(tmp_path / "orc_sun"), v1=False)
    files = sunrgbd_outputs(tmp_path / "orc_sun")
    assert sunrgbd_outputs(tmp_path / "ours_sun") == files and len(files) == 18
    same_files(tmp_path / "ours_sun", tmp_path / "orc_sun", files)

    # the fields the loader reads of the original ScannetDatasetConfig (18 classes, 1 heading bin) / SunrgbdDatasetConfig (10, 12)
    from types import SimpleNamespace
    dc = SimpleNamespace(nyu40ids=P.OBJ_CLASS_IDS, type2class=dict(enumerate(range(18))), mean_size_arr=np.ones((18, 3)), num_heading_bin=1)
    split = tmp_path / "split.txt"
    split.write_text(f"{names[0]}\n{names[-1]}\n")
    ds = det_data.ScannetDetectionDataset("train", 20000, data_path=str(tmp_path / "ours_sc"), split_file=str(split), dataset_config=dc)
    b = next(iter(det_data.DetectionLoader(ds, 2, shuffle=False)))
    assert b["point_clouds"].shape == (2, 20000, 3) and b["point_clouds"].is_cuda
    dc = SimpleNamespace(type2class=P.TYPE2CLASS, mean_size_arr=np.ones((10, 3)), num_heading_bin=12)
    ds = det_data.SunrgbdDetectionVotesDataset("train", 20000, data_path=str(tmp_path / "ours_sun" / "sunrgbd_pc_bbox_votes_50k_v2_train"),
                                               dataset_config=dc)
    b = next(iter(det_data.DetectionLoader(ds, 2, shuffle=False)))
    assert b["point_clouds"].shape == (2, 20000, 3) and b["vote_label_mask"].any()
