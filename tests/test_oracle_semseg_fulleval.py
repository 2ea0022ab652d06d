"""Semantic segmentation on the original point cloud, without a GPU: the oracle (oracle/semseg_fulleval_cpu.py) on hand-checked cases
and against its own brute force, the transformation collate, and the host argument checks of `pcb_nearest` / `pcb_label_transfer`."""
import os

import numpy as np
import pytest
import torch

from oracle import semseg_fulleval_cpu as O


def test_nearest_tie_rule_by_hand():
    ref = np.array([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [1.0, 0, 0], [5.0, 5, 5]])
    q = np.array([[0.0, 0, 0], [1.0, 0, 0], [0.5, 0.5, 0], [4.0, 4, 4], [2.0, 0, 0]])
    want = [0, 0, 0, 4, 0]                    # equal d2: the smallest index; duplicates 0 / 3: index 0
    assert list(O.nearest_brute(ref, q)) == want
    assert list(O.nearest(ref, q)) == want


def test_nearest_kdtree_equals_brute_force():
    g = np.random.default_rng(0)
    c = (np.arange(5) + 0.5) * 0.25
    lattice = np.stack(np.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3)
    h = np.arange(11) * 0.125
    ties = np.stack(np.meshgrid(h, h, h, indexing="ij"), -1).reshape(-1, 3)
    for ref, q in ((g.random((700, 3)), g.random((900, 3)) * 1.4 - 0.2), (lattice, ties),
                   (np.concatenate([lattice, lattice[::-1]]), ties), (g.random((300, 3)) + 1e4, g.random((200, 3)) + 1e4)):
        assert np.array_equal(O.nearest(ref, q), O.nearest_brute(ref, q))


def test_fast_hist_and_label_transfer():
    label_map = {0: 255, 1: 0, 2: 1, 3: 255, 4: 2, 255: 255}
    lut = O.label_lut(label_map)
    assert list(O.decode_lut(label_map, 3)) == [1, 2, 4]
    idx = np.array([0, 1, 2, 2, 0])
    ref_label = np.array([1, 2, 4])
    gt = np.array([1, 2, 255, 3, 4])
    pl, h = O.label_transfer(idx, ref_label, gt, lut, 3)
    assert list(pl) == [1, 2, 4, 4, 1]
    want = np.zeros((3, 3), np.int64)
    want[0, 0] += 1; want[1, 1] += 1; want[2, 0] += 1        # gt 255 and ignored gt 3 do not count
    assert np.array_equal(h, want)
    assert np.array_equal(O.fast_hist(np.array([0, 1, 2]), np.array([2, 255, 0]), 3), [[0, 0, 1], [0, 0, 0], [1, 0, 0]])
    for bad in ([1, 2, 300, 3, 4], [1, 2, -1, 3, 4], [1, 2, 5, 3, 4]):
        with pytest.raises(KeyError):
            O.label_transfer(idx, ref_label, np.array(bad), lut, 3)
    with pytest.raises(KeyError):                                          # a counted prediction that masks to 255
        O.label_transfer(idx, np.array([0, 2, 4]), gt, lut, 3)


def test_centres_and_groups():
    T = np.diag([50.0, 50.0, 50.0, 1.0]).astype(np.float32)
    T[:3, 3] = [3, 4, 5]
    c = O.centres(np.array([[0, 0, 0], [1, 2, 3]]), T.reshape(16))
    assert np.allclose(c, [[(0.5 - 3) / 50, (0.5 - 4) / 50, (0.5 - 5) / 50], [(1.5 - 3) / 50, (2.5 - 4) / 50, (3.5 - 5) / 50]], rtol=1e-6)
    paths = [os.path.join("Area_1", f) for f in ("conferenceRoom_1.ply", "office_1.ply", "office_10.ply", "office_2.ply")]
    paths.append(os.path.join("Area_2", "office_1.ply"))
    groups = O.s3dis_groups(paths)
    assert list(groups.items()) == [(("Area_1", "conferenceRoom"), [0]), (("Area_1", "office"), [1, 2, 3]), (("Area_2", "office"), [4])]
    assert O.scannet_output_id("scene0707_00_vh_clean_2.ply") == "scene0707_00"


def test_cflt_collate_on_host():
    from pointcontrast_b200 import semseg_data as D
    g = np.random.default_rng(2)
    items = []
    for n in (5, 7, 4):
        items.append((torch.from_numpy(g.integers(0, 9, (n, 3)).astype(np.int32)), torch.from_numpy(g.random((n, 3)).astype(np.float32)),
                      torch.from_numpy(g.integers(0, 20, n).astype(np.int32)), g.random(16).astype(np.float32)))
    coords, feats, labels, T = D.cflt_collate_fn_factory(0)(items)
    assert T.dtype == torch.float32 and tuple(T.shape) == (3, 17)
    assert np.array_equal(T[:, :16].numpy(), np.stack([it[3] for it in items])) and list(T[:, 16].numpy()) == [0, 1, 2]
    assert list(coords[:, 0].numpy()) == [0] * 5 + [1] * 7 + [2] * 4
    coords, feats, labels, T = D.cflt_collate_fn_factory(11)(items)       # truncated at the scene that exceeds 11 points
    assert tuple(T.shape) == (1, 17) and len(coords) == 5


def test_host_argument_checks():
    from pointcontrast_b200 import _lib
    L = _lib.lib
    assert L.pcb_nearest_ws_bytes(-1, 5) == 0 and L.pcb_nearest_ws_bytes(5, 1 << 31) == 0
    assert L.pcb_nearest_ws_bytes(0, 0) > 0
    buf = np.zeros(64, np.float64)
    p = buf.ctypes.data
    # n == 0 returns before anything else; m == 0 < n, bad cell sizes, NULL pointers and short workspaces are rejected
    assert L.pcb_nearest(None, 0, None, 0, 0.05, None, None, None, 0, None) == 0
    assert L.pcb_nearest(p, 0, p, 3, 0.05, p, p, p, 1 << 30, None) == 2
    for cell in (0.0, -1.0, float("inf"), float("nan")):
        assert L.pcb_nearest(p, 3, p, 3, cell, p, p, p, 1 << 30, None) == 2
    assert L.pcb_nearest(p, 3, p, 3, 0.05, None, p, p, 1 << 30, None) == 2
    assert L.pcb_nearest(p, 3, p, 3, 0.05, p, p, p, L.pcb_nearest_ws_bytes(3, 3) - 1, None) == 2
    assert L.pcb_label_transfer(None, None, 0, None, 0, None, 0, 0, None, None, None, None) == 0
    assert L.pcb_label_transfer(p, p, 3, p, 3, p, 0, 20, p, p, p, None) == 2            # lut_n < 1
    assert L.pcb_label_transfer(p, p, 3, p, 3, p, 256, 0, p, p, p, None) == 2           # C < 1
    assert L.pcb_label_transfer(p, p, 3, p, 3, p, 256, 20, p, None, p, None) == 2       # no histogram
    assert L.pcb_label_transfer(p, p, 3, None, 3, None, 0, 0, p, None, None, None) == 2  # no status
    assert L.pcb_label_transfer(p, p, 3, None, -1, None, 0, 0, p, None, p, None) == 2
    assert L.pcb_label_transfer(p, p, -1, None, 3, None, 0, 0, p, None, p, None) == 2             # m < 0


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "semseg_fulleval.npz")


@pytest.mark.parametrize("kind", ["scannet", "s3dis"])
def test_oracle_matches_reference_golden(tmp_path, kind):
    """The reference's staged `save_predictions` and `test_pointcloud` (tests/golden/make_semseg_fulleval_golden.py) against the oracle:
    the same npy arrays bit for bit, the same submission files byte for byte, the same histogram."""
    from tests.golden import make_semseg_fulleval_golden as G
    z = np.load(GOLDEN)
    s = G.write_plys(z, kind, str(tmp_path / "data"))
    label_map, C = G.KINDS[kind]
    pred_dir = tmp_path / "pred"
    pred_dir.mkdir()
    for i, (coords, pred) in enumerate(zip(s["coords"], s["pred"])):
        got = O.save_predictions(coords.reshape(-1, 4), pred, s["T"][i:i + 1], label_map, C, i, str(pred_dir))
        assert np.array_equal(got[0], s["npy"][i].reshape(-1, 4))
    preds = [a.reshape(-1, 4) for a in s["npy"]]
    if kind == "scannet":
        edir = tmp_path / "eval"
        edir.mkdir()
        hist, _ = O.test_pointcloud_scannet(preds, s["names"], str(tmp_path / "data"), label_map, C, str(edir))
        for name, txt in zip(s["names"], s["txt"]):
            assert (edir / (name[:12] + ".txt")).read_bytes() == txt
        hist_b, _ = O.test_pointcloud_scannet(preds, s["names"], str(tmp_path / "data"), label_map, C, nearest_fn=O.nearest_brute)
        assert np.array_equal(hist_b, hist)
    else:
        hist, _ = O.test_pointcloud_s3dis(preds, s["names"], str(tmp_path / "data"), label_map, C)
    assert hist.sum() > 0
    assert np.array_equal(hist, s["hist"])
