"""S3DIS preprocessing on the GPU (pcb_text_lines, pcb_s3dis_parse, pcb_ply_rows through semseg_prep) against the numpy restatement
(oracle/semseg_prep_cpu.py) bit for bit, and against the original's output bytes (tests/golden/semseg_prep.npz)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import semseg_prep_cpu as O
from pointcontrast_b200 import semseg_data as S, semseg_prep as P, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "semseg_prep.npz")

# every separator, rounding edges, skipped lines
EXACT = (b"-0.000 0.005 -0.005 1 2 3\n0.010 -0.010 0.015 4 5 6\r\n1e-3 +.5 5. 7 8 9\r"
         b"12.345\t6.789\x0b-1.001\x0c10 11 12\x1c\n3.141\x1d2.718\x1e1.414\x1f13 14 15 \n"
         b"1.2.3 0 0 0 0 0\n1\x102 0 0 0 0 0\n0.009999 0.019999 -0.0099 200 100 50\n-49.995 49.995 0.0050 255.9 0.0 1e2\n"
         b"0.005 0.005 -0.005 9 9 9")
# lines the device hands to the host
HOST = (b"1_0 0.1 0.2 16 17 18\n0.12345678901234567890 1.5 2.5 0 1 2\n0.1 0.2 0.3 256 -1 255.9\n0.1 0.2 0.3 inf nan 1\n"
        b"1e400 2 3 4 5 6 7 x\n0.5 0.5 0.5 1 2 3" + b" " * 600 + b"\n")
NONASCII = "0.001 0.002 0.003 1 2 3\n0.004 0.005 0.006 4 5 6  \n".encode("utf-8")


def _room(tmp_path, contents):
    ann = tmp_path / "room" / "Annotations"
    ann.mkdir(parents=True, exist_ok=True)
    files = []
    for name, data in contents:
        (ann / name).write_bytes(data)
        files.append(str(ann / name))
    return files


def _oracle(files):
    xs, rs, ls = [], [], []
    for f in files:
        x, r = O.read_txt(f)
        xs.append(x), rs.append(r), ls.append(np.full(len(x), O.CLASSES.index(os.path.basename(f).split("_")[0]), np.int32))
    x = np.concatenate(xs)
    return x, np.concatenate(rs), np.concatenate(ls), np.floor(x.astype(np.float64) / 0.01).astype(np.int32)


def _check(files):
    got = [t.cpu().numpy() for t in P.parse_room(P._load_room(files), torch.device("cuda"))]
    want = _oracle(files)
    assert got[0].shape == want[0].shape
    assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32))           # bits: the sign of -0.000 included
    for g, w in zip(got[1:], want[1:]):
        assert np.array_equal(g, w)
    return got


def test_parse_matches_the_oracle_on_adversarial_text(tmp_path):
    got = _check(_room(tmp_path, [("wall_1.txt", EXACT), ("chair_1.txt", HOST), ("door_1.txt", NONASCII), ("beam_2.txt", EXACT[:52])]))
    assert np.signbit(got[0][0, 0]) and got[3][0].tolist() == [0, 0, -1]


@pytest.mark.parametrize("data,match", [(b"1 2 3 4 5\n", "6 values"), (b"1 2 3 4 5 6\n\n1 2 3 4 5 6\n", "6 values"), (b"", "no parsed line"),
                                        (b"x y z\n", "no parsed line"), (b"1 2 3 4 5 inf 7\n", "values")])
def test_parse_raises_where_the_original_raises(tmp_path, data, match):
    files = _room(tmp_path, [("wall_1.txt", EXACT), ("floor_1.txt", data)])
    with pytest.raises(Exception):
        O.read_txt(files[1])
    with pytest.raises(ValueError, match=match):
        P.parse_room(P._load_room(files), torch.device("cuda"))


def test_unknown_class_raises(tmp_path):
    with pytest.raises(ValueError, match="unknown S3DIS class"):
        P._load_room(_room(tmp_path, [("roof_1.txt", EXACT)]))


def test_sizes_across_block_and_chunk_boundaries(tmp_path):
    rng = np.random.default_rng(5)
    many = [(f"{O.CLASSES[k % 14]}_{k}.txt", b"%d.%03d 0.5 -0.25 %d 7 8%s" % (k % 17 - 8, k % 1000, k % 256, b"\n" if k % 3 else b""))
            for k in range(700)]
    long_line = (b"1.000" + b" " * 40 + b"2.000\t\t\t3.000 4 5 6\n") * 3
    mm = rng.integers(-50000, 50000, size=(70001, 3))
    big = b"".join(b"%.3f %.3f %.3f %d %d %d\n" % (x / 1000, y / 1000, z / 1000, x % 256, y % 256, z % 256) for x, y, z in mm.tolist())
    _check(_room(tmp_path, many[:350] + [("window_1.txt", long_line), ("table_1.txt", big)] + many[350:]))


def test_whole_rooms_match_the_oracle(tmp_path):
    synth.write_s3dis_tree(tmp_path / "in", 1, areas=(1, 5), rooms_per_area=2, points_per_room=30000)
    P.convert_stanford(str(tmp_path / "in"), str(tmp_path / "ours"), log=None)
    O.convert_stanford(str(tmp_path / "in"), str(tmp_path / "orc"))
    n = 0
    for a in ("Area_1", "Area_5"):
        for f in sorted(os.listdir(tmp_path / "orc" / a)):
            assert (tmp_path / "ours" / a / f).read_bytes() == (tmp_path / "orc" / a / f).read_bytes(), f
            labels = S.read_ply(tmp_path / "ours" / a / f)["label"]
            n += 1
            assert (labels == 255).any() and (labels < 14).any()            # mixed-label voxels and plain ones
    assert n == 4 and not os.path.exists(tmp_path / "ours" / "Area_1" / "storage_1.ply")


def test_golden_original_output(tmp_path):
    z = np.load(GOLDEN)
    text, off = z["text"].tobytes(), z["text_off"]
    for k, rel in enumerate(z["paths"].tolist()):
        p = tmp_path / "in" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(text[off[k]:off[k + 1]])
    P.convert_stanford(str(tmp_path / "in"), str(tmp_path / "out"), log=None)
    out, ooff = z["out"].tobytes(), z["out_off"]
    for k, rel in enumerate(z["outputs"].tolist()):
        assert (tmp_path / "out" / rel).read_bytes() == out[ooff[k]:ooff[k + 1]], rel


def test_cli_end_to_end_and_area5_loader(tmp_path):
    synth.write_s3dis_tree(tmp_path / "in", 2, areas=(1, 2, 5), rooms_per_area=1, points_per_room=20000)
    cmd = [sys.executable, "-m", "pointcontrast_b200.semseg_prep", "stanford", "--input", str(tmp_path / "in"), "--output", str(tmp_path / "out")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, check=True)
    assert "has 0 files." in r.stdout and r.stdout.count(" -> ") == 3
    plys = sorted(p.relative_to(tmp_path / "out").as_posix() for p in (tmp_path / "out").glob("Area_*/*.ply"))
    assert plys == ["Area_1/office_1.ply", "Area_2/office_1.ply", "Area_5/office_1.ply"]
    assert (tmp_path / "out" / "splits" / "area5.txt").read_text() == "Area_5/office_1.ply"
    before = {p: (p.read_bytes(), p.stat().st_mtime_ns) for p in (tmp_path / "out").rglob("*.ply")}
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, check=True)
    assert r.stdout.count("exists") == 3
    assert {p: (p.read_bytes(), p.stat().st_mtime_ns) for p in (tmp_path / "out").rglob("*.ply")} == before
    from tests import refload
    cfg = refload.Cfg(data=dict(stanford3d_path=str(tmp_path / "out"), ignore_label=255, return_transformation=False, voxel_size=None),
                      augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05))
    loader = S.initialize_data_loader(S.StanfordArea5Dataset, cfg, "train", shuffle=True, augment_data=True, batch_size=2, limit_numpoints=0)
    assert len(loader.dataset) == 2
    coords, feats, labels = next(iter(loader))[0]
    assert coords.is_cuda and coords.shape[1] == 4 and len(coords) == len(feats) == len(labels) > 0
    val = S.initialize_data_loader(S.StanfordArea5Dataset, cfg, "val", shuffle=False, augment_data=False, batch_size=1, limit_numpoints=0,
                                   repeat=False)
    assert len(val.dataset) == 1
