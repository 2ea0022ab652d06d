"""The staged original VoteNet detection preprocessing (oracle/det_prep_ref.py) against the numpy restatement (oracle/det_prep_cpu.py),
file for file under the same np.random seed: ScanNet scenes with the aggregation quirks and every skip cause, SUN RGB-D scenes with
nested, face-touching, zero-size, thin and non-whitelisted boxes, an empty scene and N below and above 50000.  Skipped where the
original is not staged."""
import os

import numpy as np
import pytest

from oracle import det_prep_cpu as O, det_prep_ref as R
from pointcontrast_b200 import synth

pytestmark = pytest.mark.skipif(not R.available(), reason="the original detection preprocessing is not staged (oracle/det_prep_ref.py)")
FAULTS = (None, "no_align", "unknown_seg", "unknown_label", "no_segments", "id_range", "vertex_count", None)


def scannet_tree(root, n=3000, big=52000):
    os.makedirs(root, exist_ok=True)
    lm = synth.write_scannet_label_map(os.path.join(root, "labels.tsv"))
    names = []
    for k, fault in enumerate(FAULTS):
        names.append("scene%04d_00" % k)
        synth.write_scannet_det_raw_scene(os.path.join(root, "scans"), names[-1], k, n=big if k == len(FAULTS) - 1 else n, fault=fault)
    return os.path.join(root, "scans"), lm, names


def same_files(a, b, names):
    for f in names:
        p, q = os.path.join(a, f), os.path.join(b, f)
        if f.endswith(".npy"):
            assert open(p, "rb").read() == open(q, "rb").read(), f
        else:
            x, y = np.load(p), np.load(q)
            assert x.files == y.files, f
            for k in x.files:
                assert x[k].dtype == y[k].dtype and np.array_equal(x[k], y[k]), (f, k)


def test_scannet_restatement_writes_the_original_files(tmp_path):
    scans, lm, names = scannet_tree(str(tmp_path))
    np.random.seed(3)
    R.scannet(scans, lm, names, str(tmp_path / "ref"))
    np.random.seed(3)
    failed = O.convert_scannet(scans, str(tmp_path / "orc"), lm, names)
    assert failed == [names[k] for k, f in enumerate(FAULTS) if f]
    ok = [names[0], names[-1]]
    assert sorted(os.listdir(tmp_path / "ref")) == sorted(os.listdir(tmp_path / "orc")) == sorted(n + s for n in ok for s in (
        "_vert.npy", "_sem_label.npy", "_ins_label.npy", "_bbox.npy"))
    same_files(tmp_path / "ref", tmp_path / "orc", [n + s for n in ok for s in ("_vert.npy", "_sem_label.npy", "_ins_label.npy", "_bbox.npy")])
    assert len(np.load(tmp_path / "orc" / (names[-1] + "_vert.npy"))) == 50000


def sunrgbd_outputs(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


@pytest.mark.parametrize("v1", [True, False])
def test_sunrgbd_restatement_writes_the_original_files(tmp_path, v1):
    synth.write_sunrgbd_export(str(tmp_path / "in"), 4)
    np.random.seed(5)
    R.sunrgbd(str(tmp_path / "in"), str(tmp_path / "ref"), v1=v1)
    np.random.seed(5)
    O.convert_sunrgbd(str(tmp_path / "in"), str(tmp_path / "orc"), v1=v1)
    files = sunrgbd_outputs(tmp_path / "ref")
    assert files == sunrgbd_outputs(tmp_path / "orc") and len(files) == 18
    same_files(tmp_path / "ref", tmp_path / "orc", files)
    votes = np.load(tmp_path / "orc" / f"sunrgbd_pc_bbox_votes_50k_{'v1' if v1 else 'v2'}_train" / "000002_votes.npz")["point_votes"]
    assert votes[:, 0].any() and (votes[:, 4:7] != votes[:, 1:4]).any(axis=1).any()        # points in two or more boxes


def test_analytic_inside_test_matches_delaunay_off_the_faces():
    """The analytic inside test against scipy's Delaunay (the original's in_hull) on random boxes, thin ones included; points within
    1e-9 of a face are left out, and there are few of them."""
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(0)
    excluded = 0
    for k in range(40):
        c = rng.uniform(-2, 2, 3)
        l, w, h = rng.uniform(0.05, 1.5, 3) if k % 8 else (0.5, 0.3, 1e-9)
        heading = rng.uniform(-np.pi, np.pi)
        t = -1 * heading
        R_ = np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1]])
        corners = (R_ @ np.array([[-l, l, l, -l, -l, l, l, -l], [w, w, -w, -w, w, w, -w, -w], [h, h, h, h, -h, -h, -h, -h]])).T + c
        pts = c + rng.uniform(-1.3, 1.3, (20000, 3)) * np.array([l, w, max(h, 1e-3)])
        a = O.inside(pts, c, l, w, h, heading)
        d = Delaunay(corners).find_simplex(pts) >= 0
        u = (pts - c) @ R_
        near = (np.abs(np.abs(u) - np.array([l, w, h])) < 1e-9).any(1)
        excluded += int(near.sum())
        assert np.array_equal(a[~near], d[~near]), k
    assert excluded < 20000 * 40 * 0.01
