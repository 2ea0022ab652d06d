"""The staged original semseg preprocessing (oracle/semseg_prep_ref.py, with the ME stand-in) against the numpy restatement
(oracle/semseg_prep_cpu.py): byte-identical PLYs and split files for S3DIS and ScanNet on synthetic trees.  Skipped where the original
is not staged."""
import glob
import os

import pytest

from oracle import semseg_prep_cpu as O, semseg_prep_ref as R
from pointcontrast_b200 import synth

pytestmark = pytest.mark.skipif(not R.available(), reason="the original semseg preprocessing is not staged (oracle/semseg_prep_ref.py)")


def _same_tree(a, b, pattern):
    fa, fb = sorted(glob.glob(os.path.join(a, pattern))), sorted(glob.glob(os.path.join(b, pattern)))
    assert fa and [os.path.relpath(p, a) for p in fa] == [os.path.relpath(p, b) for p in fb]
    for p, q in zip(fa, fb):
        assert open(p, "rb").read() == open(q, "rb").read(), p


def test_stanford_restatement_writes_the_original_bytes(tmp_path):
    synth.write_s3dis_tree(tmp_path / "in", 3, areas=(1, 2, 5), rooms_per_area=1, points_per_room=3000)
    R.stanford(str(tmp_path / "in"), str(tmp_path / "ref"), str(tmp_path / "cwd"))
    O.convert_stanford(str(tmp_path / "in"), str(tmp_path / "orc"))
    O.generate_splits(str(tmp_path / "orc"), str(tmp_path / "orc_splits"))
    _same_tree(tmp_path / "ref", tmp_path / "orc", "*/*.ply")
    for i in range(1, 7):
        assert (tmp_path / "cwd" / "splits" / "stanford" / f"area{i}.txt").read_bytes() == (tmp_path / "orc_splits" / f"area{i}.txt").read_bytes()


def test_scannet_restatement_writes_the_original_bytes(tmp_path):
    for k, name in enumerate(("scene0270_00", "scene0384_00", "scene0001_00")):
        synth.write_scannet_raw_scene(tmp_path / "raw", "scans", name, k, n=500)
    synth.write_scannet_raw_scene(tmp_path / "raw", "scans_test", "scene0707_00", 7, n=300, labels=False)
    R.scannet(tmp_path / "raw", tmp_path / "ref")
    O.convert_scannet(tmp_path / "raw", tmp_path / "orc")
    _same_tree(tmp_path / "ref", tmp_path / "orc", "*/*.ply")
