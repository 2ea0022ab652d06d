"""Semantic segmentation on the original point cloud on the GPU: `pcb_nearest` index for index against oracle/semseg_fulleval_cpu.py
(ties, duplicates, the brute-force pass, clustered and offset clouds, three cell sizes, ScanNet size), its argument checks,
`pcb_label_transfer` against `fast_hist`, and `semseg.test` with `test.save_prediction` / `test.test_original_pointcloud` on synthetic
ScanNet and S3DIS rooms against the oracle, with `semseg.test_pointcloud` on the saved files."""
import os

import numpy as np
import pytest
import torch

from oracle import semseg_fulleval_cpu as O
from tests import refload

pytestmark = pytest.mark.gpu


def _nn(ref, query, cell):
    from pointcontrast_b200 import semseg
    return semseg.nearest(torch.from_numpy(np.ascontiguousarray(ref, np.float64)).cuda(),
                          torch.from_numpy(np.ascontiguousarray(query, np.float64)).cuda(), cell).cpu().numpy().astype(np.int64)


def _lattice(k=6, v=0.25):
    """Voxel centres (i + 0.5) v of a k^3 lattice and queries on every face, edge and corner between them (exact dyadic values, so
    the tied distances are equal in fp64), on the centres themselves and inside the voxels."""
    c = (np.arange(k) + 0.5) * v
    ref = np.stack(np.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3)
    h = np.arange(2 * k + 1) * (v / 2)
    q = np.stack(np.meshgrid(h, h, h, indexing="ij"), -1).reshape(-1, 3)
    return ref, np.concatenate([q, q + v / 8])


def _cases():
    g = np.random.default_rng(7)
    ref_u, q_u = g.random((3000, 3)) * 4, g.random((5000, 3)) * 4.5 - 0.25
    ref_l, q_l = _lattice()
    dup = g.random((400, 3))
    ref_d = np.concatenate([dup, dup[::-1], dup[:100]])
    perm = g.permutation(len(ref_d))
    q_d = np.concatenate([g.random((1000, 3)), dup[:50]])
    ref_far, q_far = g.random((2000, 3)), np.concatenate([g.random((300, 3)), [[100.0, -40.0, 3.0], [-7.5, 0.5, 0.5]]])
    centres = g.random((20, 3)) * 3
    ref_c = (centres[:, None, :] + g.normal(0, 2e-3, (20, 300, 3))).reshape(-1, 3)
    q_c = g.random((3000, 3)) * 3
    return [("uniform", ref_u, q_u, 0.1), ("lattice-ties", ref_l, q_l, 0.25), ("lattice-ties-small-cell", ref_l, q_l, 0.03125),
            ("duplicates", ref_d[perm], q_d, 0.05), ("m1", g.random((1, 3)), g.random((500, 3)) * 10, 0.05),
            ("far-query", ref_far, q_far, 0.05), ("clustered", ref_c, q_c, 0.5),
            ("offset-1e4", ref_u * 0.1 + 1e4, q_u * 0.1 + 1e4, 0.02)]


@pytest.mark.parametrize("name,ref,query,cell", _cases(), ids=[c[0] for c in _cases()])
def test_nearest_matches_oracle(name, ref, query, cell):
    got = _nn(ref, query, cell)
    want = O.nearest_brute(ref, query)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (name, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _room(seed=3, n_raw=60_000, voxel=0.05):
    """ScanNet-like surfaces: voxel centres of the points (the predicted cloud) and the points themselves (the queries)."""
    from pointcontrast_b200 import synth
    xyz = synth.synth_labelled_room(seed, n_raw, scale=1.0)[0].astype(np.float64)
    cells = np.unique(np.floor(xyz / voxel), axis=0)
    return (cells + 0.5) * voxel, xyz


@pytest.mark.parametrize("mult", [0.125, 1.0, 64.0])
def test_nearest_independent_of_cell_size(mult):
    ref, query = _room()
    want = O.nearest(ref, query)
    got = _nn(ref, query, 0.05 * mult)
    assert np.array_equal(got, want)


def test_nearest_scannet_size():
    g = np.random.default_rng(11)
    ref, query = _room(seed=5, n_raw=400_000, voxel=0.02)
    ref = ref[g.permutation(len(ref))[:120_000]]
    query = query[g.permutation(len(query))[:150_000]]
    assert np.array_equal(_nn(ref, query, 0.02), O.nearest(ref, query))


def test_nearest_arguments():
    from pointcontrast_b200 import _lib, semseg
    L = _lib.lib
    g = np.random.default_rng(1)
    ref = torch.from_numpy(g.random((5000, 3))).cuda()
    query = torch.from_numpy(g.random((7000, 3)) * 1.2 - 0.1).cuda()
    m, n = len(ref), len(query)
    q = L.pcb_nearest_ws_bytes(m, n)
    ws = torch.empty(q, dtype=torch.uint8, device="cuda")
    idx = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(L.pcb_nearest(ref.data_ptr(), m, query.data_ptr(), n, 0.03, idx.data_ptr(), status.data_ptr(), ws.data_ptr(), q, _lib.stream()))
    assert int(status.item()) == 0
    assert np.array_equal(idx.cpu().numpy(), O.nearest_brute(ref.cpu().numpy(), query.cpu().numpy()))
    # m == 0 < n and a bad cell size are rejected before anything is launched: idx keeps its sentinel
    idx = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    for args in ((0, 0.03), (m, 0.0), (m, float("inf")), (m, float("nan"))):
        assert L.pcb_nearest(ref.data_ptr(), args[0], query.data_ptr(), n, args[1], idx.data_ptr(), status.data_ptr(), ws.data_ptr(), q,
                             _lib.stream()) == 2
    assert L.pcb_nearest(ref.data_ptr(), m, query.data_ptr(), 0, 0.03, None, None, None, 0, _lib.stream()) == 0      # n == 0: no-op
    torch.cuda.synchronize()
    assert bool((idx == -7).all()) and int(status.item()) == 0
    # a non-finite coordinate or a cell outside +-2^20 sets the status bit, which the wrapper raises
    for bad in (float("nan"), float("inf"), 1e6):
        qq = query.clone()
        qq[3, 1] = bad
        with pytest.raises(_lib.PcbError):
            semseg.nearest(ref, qq, 0.03)
        rr = ref.clone()
        rr[10, 2] = bad
        with pytest.raises(_lib.PcbError):
            semseg.nearest(rr, query, 0.03)


def _scannet_maps():
    from pointcontrast_b200 import semseg_data as D
    label_map, n_used = {}, 0
    for l in range(41):
        if l in D.ScannetVoxelizationDataset.IGNORE_LABELS:
            label_map[l] = 255
        else:
            label_map[l] = n_used
            n_used += 1
    label_map[255] = 255
    return label_map, n_used


def test_label_transfer_matches_fast_hist():
    from pointcontrast_b200 import _lib, semseg
    label_map, C = _scannet_maps()
    lut = O.label_lut(label_map)
    g = np.random.default_rng(4)
    m, n = 3000, 50_000
    ref_label = O.decode_lut(label_map, C)[g.integers(0, C, m)]
    idx = g.integers(0, m, n)
    gt = g.integers(0, 41, n)
    gt[g.random(n) < 0.1] = 255
    dev = lambda a: torch.from_numpy(np.asarray(a, np.int32)).cuda()
    hist = torch.zeros(C * C, dtype=torch.int64, device="cuda")
    base = g.integers(0, 1000, C * C)
    hist += torch.from_numpy(base).cuda()                               # accumulated onto, not overwritten
    pl, status = semseg.label_transfer(dev(idx), dev(ref_label), dev(gt), dev(lut), C, hist)
    want_pl, want_h = O.label_transfer(idx, ref_label, gt, lut, C)
    assert int(status.item()) == 0
    assert np.array_equal(pl.cpu().numpy(), want_pl)
    assert np.array_equal(hist.cpu().numpy(), base + want_h.reshape(-1))
    # without query labels only the transfer runs
    pl2, status = semseg.label_transfer(dev(idx), dev(ref_label))
    assert np.array_equal(pl2.cpu().numpy(), want_pl) and int(status.item()) == 0
    # an index outside [0, m) is reported and that row is neither transferred nor counted
    for bad in (m, -1):
        bad_idx = idx.copy()
        bad_idx[7] = bad
        h = torch.zeros(C * C, dtype=torch.int64, device="cuda")
        pl3, status = semseg.label_transfer(dev(bad_idx), dev(ref_label), dev(gt), dev(lut), C, h)
        assert int(status.item()) & _lib.NEAREST_RANGE and int(pl3[7]) == -1
    # a label outside the table, a label without an entry, and a counted prediction that maps to 255 are reported
    for bad_gt, bad_ref in ((300, None), (-1, None), (None, 0)):
        gt2, ref2 = gt.copy(), ref_label.copy()
        if bad_gt is not None:
            gt2[5] = bad_gt
        else:
            counted = np.flatnonzero((gt < 41) & (lut[np.minimum(gt, 255)] < C))[0]
            ref2[idx[counted]] = bad_ref                                     # original id 0 is ignored: masked 255 against a valid gt
        with pytest.raises(KeyError):
            O.label_transfer(idx, ref2, gt2, lut, C)
        h = torch.zeros(C * C, dtype=torch.int64, device="cuda")
        _, status = semseg.label_transfer(dev(idx), dev(ref2), dev(gt2), dev(lut), C, h)
        assert int(status.item()) & _lib.LABEL_RANGE
    # C above the shared-memory bins: the global-atomic path gives the same histogram
    C2 = 80
    lut2 = np.arange(C2 + 1, dtype=np.int64)
    lut2[C2] = 255
    r2, g2 = g.integers(0, C2, m), g.integers(0, C2 + 1, n)
    h = torch.zeros(C2 * C2, dtype=torch.int64, device="cuda")
    _, status = semseg.label_transfer(dev(idx), dev(r2), dev(g2), dev(lut2), C2, h)
    assert int(status.item()) == 0
    assert np.array_equal(h.cpu().numpy(), O.label_transfer(idx, r2, g2, lut2, C2)[1].reshape(-1))


# ------------------------------------------------------------------------------------------------ semseg.test end to end

def _scannet_rooms(root, n=4, n_raw=20_000):
    from pointcontrast_b200 import synth
    (root / "splits").mkdir(exist_ok=True)
    names = []
    for k in range(n):
        xyz, rgb, lab = synth.synth_labelled_room(300 + k, n_raw, scale=0.8 + 0.1 * k)
        synth.write_ply(root / f"scene{k:04d}_00_vh_clean_2.ply", xyz, rgb, lab if k != 2 else None)    # scene 2: test split, no label
        names.append(f"scene{k:04d}_00_vh_clean_2.ply")
    (root / "splits" / "scannetv2_val.txt").write_text("\n".join(names) + "\n")


def _s3dis_rooms(root):
    from pointcontrast_b200 import synth
    (root / "Area_5").mkdir(parents=True, exist_ok=True)
    (root / "splits").mkdir(exist_ok=True)
    names = []
    shared = None
    for k, name in enumerate(("office_1", "office_2", "hallway_1")):
        xyz, rgb, lab = synth.synth_labelled_room(400 + k, 15_000, scale=0.7 + 0.1 * k, num_labels=14)
        if k == 0:
            shared = (xyz[:2000], rgb[:2000], lab[:2000])
            xyz, rgb, lab = (np.concatenate([a, b[:500]]) for a, b in zip((xyz, rgb, lab), shared))     # duplicate rows inside one room
        if k == 1:
            xyz, rgb, lab = (np.concatenate([a, b]) for a, b in zip((xyz, rgb, lab), shared))          # and across the office group
        synth.write_ply(root / "Area_5" / f"{name}.ply", xyz, rgb, lab)
        names.append(f"Area_5/{name}.ply")
    (root / "splits" / "val.txt").write_text("\n".join(names) + "\n")


def _config(root, pred_dir, save, full, transformation=True):
    return refload.Cfg(
        data=dict(scannet_path=str(root), stanford3d_path=str(root), ignore_label=255, return_transformation=transformation),
        augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
        net=dict(model="Res16UNet34C", wrapper_type=None), misc=dict(seed=123), train=dict(),
        test=dict(test_stat_freq=1, save_prediction=save, save_pred_dir=str(pred_dir), test_original_pointcloud=full,
                  evaluate_original_pointcloud=False))


def _loader(root, cfg, stanford, batch_size, shuffle=False):
    from pointcontrast_b200 import semseg_data as D
    if stanford:
        return D.initialize_data_loader(D.StanfordDataset, cfg, "val", shuffle=shuffle, augment_data=False, batch_size=batch_size,
                                        limit_numpoints=0, repeat=False)
    return D.initialize_data_loader(D.ScannetVoxelization2cmDataset, cfg, "val", shuffle=shuffle, augment_data=False,
                                    batch_size=batch_size, limit_numpoints=0, split_dir=str(root / "splits"), repeat=False)


def _net(C, seed=1):
    from pointcontrast_b200.model import load_model
    from tests.helpers import det_init
    mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
    net = load_model("Res16UNet34C")(3, C, mcfg, D=3).cuda()
    det_init(net, seed)
    return net


def _oracle_predictions(net, loader, dataset, out_dir):
    """The oracle's `save_predictions` of every batch, from the model's logits (argmax on the host)."""
    from pointcontrast_b200 import me as ME
    from oracle.semseg_eval_cpu import argmax_first
    net.eval()
    files = []
    with torch.no_grad():
        for it, (coords, feats, target, T) in enumerate(loader):
            out = net(ME.SparseTensor(feats, coords).to("cuda")).F.cpu().numpy()
            files += O.save_predictions(coords.cpu().numpy(), argmax_first(out), T.numpy(), dataset.label_map, dataset.NUM_LABELS, it,
                                        str(out_dir))
    return files


@pytest.mark.parametrize("stanford", [False, True], ids=["scannet", "s3dis"])
def test_semseg_test_original_pointcloud(tmp_path, stanford):
    from pointcontrast_b200 import semseg
    root = tmp_path / "data"
    root.mkdir()
    (_s3dis_rooms if stanford else _scannet_rooms)(root)
    C = 13 if stanford else 20
    net = _net(C)
    plain = semseg.test(net, _loader(root, _config(root, tmp_path / "none", False, False, False), stanford, 1),
                        _config(root, tmp_path / "none", False, False, False))
    pred_dir = tmp_path / "pred"
    cfg = _config(root, pred_dir, True, True)
    loader = _loader(root, cfg, stanford, 1)
    ev = semseg.PointCloudEvaluator(loader.dataset, "cuda", eval_path=str(pred_dir / "fulleval") if not stanford else None)
    got = semseg.test(net, loader, cfg, evaluator=ev)
    assert np.array_equal(np.array(got, np.float64), np.array(plain, np.float64), equal_nan=True), "the voxel-level result changed"
    res = ev.result()
    # the saved predictions against the oracle's
    odir = tmp_path / "oracle"
    odir.mkdir()
    want_files = _oracle_predictions(net, loader, loader.dataset, odir)
    names = sorted(f for f in os.listdir(pred_dir) if f.endswith(".npy"))
    assert names == sorted(os.listdir(odir)) and len(names) == len(loader.dataset)
    for f in names:
        a, b = np.load(pred_dir / f), np.load(odir / f)
        assert a.dtype == np.float64 and a.shape == b.shape
        assert np.array_equal(a[:, 3], b[:, 3])
        assert np.abs(a[:, :3] - b[:, :3]).max() <= 2.0 ** -50 * np.abs(b[:, :3]).max()
    # the full-resolution histogram and submission files against the oracle, from the GPU's own saved centres
    ds = loader.dataset
    preds = [np.load(pred_dir / f) for f in names]
    if stanford:
        want_hist, _ = O.test_pointcloud_s3dis(preds, ds.data_paths, ds.data_root, ds.label_map, C)
    else:
        edir = tmp_path / "oracle_eval"
        edir.mkdir()
        want_hist, labels = O.test_pointcloud_scannet(preds, ds.data_paths, ds.data_root, ds.label_map, C, str(edir))
        txt = sorted(os.listdir(pred_dir / "fulleval"))
        assert txt == sorted(os.listdir(edir)) == [f"scene{k:04d}_00.txt" for k in range(4)]
        for f in txt:
            assert (pred_dir / "fulleval" / f).read_bytes() == (edir / f).read_bytes(), f
    assert want_hist.sum() > 0
    assert np.array_equal(res.hist, want_hist)
    # the saved directory through test_pointcloud, and the in-memory path with two items per batch
    again = semseg.test_pointcloud(ds, str(pred_dir))
    assert np.array_equal(again.hist, want_hist)
    cfg2 = _config(root, tmp_path / "pred2", False, True)
    ev2 = semseg.PointCloudEvaluator(ds, "cuda")
    semseg.test(net, _loader(root, cfg2, stanford, 2), cfg2, evaluator=ev2)
    assert np.array_equal(ev2.result().hist, want_hist)


def test_semseg_test_original_pointcloud_rejections(tmp_path):
    from pointcontrast_b200 import semseg
    root = tmp_path / "data"
    root.mkdir()
    _scannet_rooms(root, n=1, n_raw=5000)
    net = _net(20)
    cfg = _config(root, tmp_path / "pred", False, True, transformation=False)
    with pytest.raises(ValueError):
        semseg.test(net, _loader(root, cfg, False, 1), cfg)
    cfg = _config(root, tmp_path / "pred", False, True)
    with pytest.raises(ValueError):
        semseg.test(net, _loader(root, cfg, False, 1, shuffle=True), cfg)
    cfg = _config(root, tmp_path / "pred", True, False)
    (tmp_path / "pred").mkdir()
    (tmp_path / "pred" / "old.npy").write_bytes(b"")
    with pytest.raises(ValueError):
        semseg.test(net, _loader(root, cfg, False, 1), cfg)
    cfg = _config(root, tmp_path / "pred4", False, True)
    loader = _loader(root, cfg, False, 1)
    loader.dataset.IS_FULL_POINTCLOUD_EVAL = False                    # a dataset without full point-cloud evaluation
    with pytest.raises(ValueError, match="does not support"):
        semseg.test(net, loader, cfg)
    cfg = _config(root, tmp_path / "pred3", False, False)
    cfg["test"]["evaluate_original_pointcloud"] = True
    with pytest.raises(NotImplementedError):
        semseg.test(net, _loader(root, cfg, False, 1), cfg)


# ------------------------------------------------------------------------------------------------ against the reference's golden

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "semseg_fulleval.npz")


class _GoldenModel(torch.nn.Module):
    """Returns logits whose argmax is the golden's prediction of the batch the loader just yielded."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.logits = None

    def forward(self, sinput):
        import types
        return types.SimpleNamespace(F=self.logits)


class _GoldenLoader:
    """The golden's collated items (batch size 1, in dataset order) for `dataset`."""

    def __init__(self, dataset, s, model):
        self.dataset, self.s, self.model, self.batch_size, self.shuffle = dataset, s, model, 1, False

    def __len__(self):
        return len(self.s["coords"])

    def __iter__(self):
        C = self.dataset.NUM_LABELS
        for i in range(len(self)):
            c = torch.from_numpy(self.s["coords"][i].reshape(-1, 4).astype(np.int32)).cuda()
            p = torch.from_numpy(self.s["pred"][i].astype(np.int64)).cuda()
            logits = torch.zeros(len(c), C, device="cuda")
            logits[torch.arange(len(c), device="cuda"), p] = 1.0
            self.model.logits = logits
            yield (c, torch.zeros(len(c), 3, device="cuda"), torch.full((len(c),), 255, dtype=torch.int32, device="cuda"),
                   torch.from_numpy(self.s["T"][i:i + 1].copy()))


@pytest.mark.parametrize("kind", ["scannet", "s3dis"])
def test_semseg_test_matches_reference_golden(tmp_path, kind):
    """`semseg.test` with `test.save_prediction` and `test.test_original_pointcloud` on the inputs of the reference's golden run
    (tests/golden/make_semseg_fulleval_golden.py): its npy files within 2^-50 relative, its submission files byte for byte, its
    histogram exactly; then `test_pointcloud` on the saved directory."""
    from pointcontrast_b200 import semseg, semseg_data as D
    from tests.golden import make_semseg_fulleval_golden as G
    s = G.write_plys(np.load(GOLDEN), kind, str(tmp_path / "data"))
    root, pred_dir = tmp_path / "data", tmp_path / "pred"
    cfg = _config(root, pred_dir, True, True)
    if kind == "scannet":
        ds = D.ScannetVoxelization2cmDataset(cfg, augment_data=False, phase="val", split_dir=str(root / "splits"))
    else:
        ds = D.StanfordDataset(cfg, augment_data=False, phase="val")
    assert ds.data_paths == s["names"]
    model = _GoldenModel()
    ev = semseg.PointCloudEvaluator(ds, "cuda", eval_path=str(pred_dir / "fulleval") if kind == "scannet" else None)
    semseg.test(model, _GoldenLoader(ds, s, model), cfg, evaluator=ev)
    for i, want in enumerate(s["npy"]):
        want = want.reshape(-1, 4)
        got = np.load(pred_dir / ("pred_%04d_00.npy" % i))
        assert got.dtype == np.float64 and got.shape == want.shape
        assert np.array_equal(got[:, 3], want[:, 3])
        assert np.abs(got[:, :3] - want[:, :3]).max() <= 2.0 ** -50 * np.abs(want[:, :3]).max()
    if kind == "scannet":
        for name, txt in zip(s["names"], s["txt"]):
            assert (pred_dir / "fulleval" / (name[:12] + ".txt")).read_bytes() == txt, name
    assert np.array_equal(ev.result().hist, s["hist"])
    assert np.array_equal(semseg.test_pointcloud(ds, str(pred_dir)).hist, s["hist"])
