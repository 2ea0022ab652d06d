"""The semseg finetune data path on the GPU (pointcontrast_b200/semseg_data.py, csrc/augment.cu, `pcb_voxelize_labels`) against the
oracle (oracle/semseg_data_cpu.py) and against the reference's own augmentation replayed from tests/golden/semseg_augment.npz;
then PLY scenes on disk -> dataset -> loader -> one `SegmentationTrainer.train_step`."""
import random

import numpy as np
import pytest
import torch

from oracle import semseg_data_cpu as O
from tests import refload
from tests.test_oracle_semseg_data import GOLDEN

pytestmark = pytest.mark.gpu


def _labelled_voxels(n, rng):
    """n points with integer coordinates; besides random points, voxels built to hold mixed labels, only ignore labels, and
    ignore mixed with one real label."""
    c = rng.integers(-40, 40, size=(n, 3)).astype(np.int32)
    lab = rng.integers(0, 20, n).astype(np.int32)
    if n >= 40:                                                            # outside the random points' range [-40, 40)
        c[:8] = [50, 50, 50]; lab[:8] = [3, 3, 4, 3, 3, 3, 3, 3]           # mixed
        c[8:16] = [-57, 0, 59]; lab[8:16] = 255                            # all ignore
        c[16:24] = [0, -53, 51]; lab[16:24] = [255, 6, 255, 6, 6, 255, 6, 6]   # ignore + one real label
        c[24:32] = [61, 62, 63]; lab[24:32] = 9                            # agree
        p = rng.permutation(40)
        c[:40], lab[:40] = c[p], lab[p]
    return c, lab


@pytest.mark.parametrize("n", [1, 1000, 300_000])
def test_voxelize_labels_matches_oracle(n):
    from pointcontrast_b200 import semseg_data as S
    rng = np.random.default_rng(n)
    c, lab = _labelled_voxels(n, rng)
    sel, colab = O.sparse_quantize(c, labels=lab, ignore_label=255, return_index=True)
    vc, vsel, vlab = S.voxelize_labels(torch.from_numpy(c).cuda(), torch.from_numpy(lab).cuda(), 255)
    assert (vsel.cpu().numpy() == sel).all()
    assert (vc.cpu().numpy() == c[sel]).all() and (vlab.cpu().numpy() == colab).all()
    if n >= 40:
        got = {tuple(k): l for k, l in zip(vc.cpu().numpy().tolist(), vlab.cpu().numpy().tolist())}
        assert got[(50, 50, 50)] == 255 and got[(-57, 0, 59)] == 255 and got[(0, -53, 51)] == 255 and got[(61, 62, 63)] == 9


def test_affine_floor_is_exact_away_from_integers():
    from pointcontrast_b200 import semseg_data as S
    rng = np.random.default_rng(5)
    xyz = (rng.random((300_000, 3)) * np.array([6.0, 5.0, 3.0]) - 1.0).astype(np.float32)
    M_v, M_r = O.transformation_matrix(0.02, [0.03, -0.04, 2.1], [2, 0, 1], 1.07)
    T = M_r @ M_v
    T[:3, 3] = [3.3, -1.25, 0.5]
    ref, mn, pre = O.affine_floor(xyz, T)
    got, gmn = S.affine_floor(torch.from_numpy(xyz).cuda(), T)
    diff = (got.cpu().numpy() != ref).any(1)
    borderline = (np.abs(pre - np.round(pre)) < 1e-9).any(1)
    assert (gmn == mn).all() or borderline.any()
    assert not (diff & ~borderline).any(), "a floor differs away from an integer"
    assert borderline.sum() <= 1e-4 * len(xyz), borderline.sum()
    blas = np.floor(np.hstack((xyz, np.ones((len(xyz), 1), np.float32))) @ T.T[:, :3]) - mn     # the reference's own expression
    assert ((got.cpu().numpy() != blas).any(1) & ~borderline).sum() == 0


def test_elastic_distortion_matches_scipy():
    """Same noise grid: the blurred grid and the moved points are bit-identical to scipy's (the oracle equals scipy bit for bit,
    tests/test_oracle_semseg_data.py)."""
    import scipy.interpolate
    import scipy.ndimage
    from pointcontrast_b200 import semseg_data as S
    rng = np.random.default_rng(7)
    coords = (rng.random((200_000, 3)) * np.array([5.0, 4.0, 2.5])).astype(np.float32)
    for g, m in ((0.2, 0.4), (0.8, 1.6)):
        noise_dim, cmin = O.noise_shape(coords, g)
        noise = rng.standard_normal((*noise_dim, 3)).astype(np.float32)
        ref = noise
        for _ in range(2):
            for shape in ((3, 1, 1, 1), (1, 3, 1, 1), (1, 1, 3, 1)):
                ref = scipy.ndimage.convolve(ref, np.ones(shape).astype("float32") / 3, mode="constant", cval=0)
        axes = O.grid_axes(cmin, g, noise_dim)
        want = coords.copy()
        want += scipy.interpolate.RegularGridInterpolator(axes, ref, bounds_error=0, fill_value=0)(coords) * m
        dims, gaxes = S.ElasticDistortion.grid(torch.from_numpy(coords).cuda(), g)
        assert (dims == noise_dim).all() and all(np.array_equal(a, b) for a, b in zip(gaxes, axes))
        x, gn = torch.from_numpy(coords).cuda(), torch.from_numpy(noise).cuda()
        S.ElasticDistortion(((g, m),)).elastic_distortion(x, None, None, g, m, noise=gn)
        assert np.array_equal(gn.cpu().numpy(), ref)
        got = x.cpu().numpy()
        rel = np.abs(got.astype(np.float64) - want) / np.maximum(np.abs(want), 1e-3)
        assert rel.max() <= 1e-6 and np.array_equal(got, want), (rel.max(), (got != want).sum())
        coords = want


@pytest.mark.parametrize("contrast", [True, False])
def test_input_transform_matches_oracle(contrast):
    from pointcontrast_b200 import semseg_data as S
    z = np.load(GOLDEN)
    c, f = z["s0_vox_coords"], z["s0_vox_feats"].astype(np.float32)
    rng = np.random.default_rng(2)
    inds = rng.permutation(len(c))[: int(len(c) * 0.8)]
    c, f = c[inds], f[inds]
    tr = O.translation_offset(rng.random((1, 3)), 0.1)
    noise = rng.standard_normal((len(c), 3))
    want_c = O.horizontal_flip(c, [0, 1])
    want_f = O.auto_contrast(f, 0.37) if contrast else f
    want_f = O.jitter(O.translate(want_f, tr), noise, 0.05)
    gc, gf = torch.from_numpy(c.copy()).cuda(), torch.from_numpy(f.copy()).cuda()
    S.input_transform(gc, gf, flip_mask=3, contrast=contrast, blend=0.37, translation=tr[0], jitter_noise=torch.from_numpy(noise).cuda(),
                      jitter_scale=0.05 * 255)
    assert (gc.cpu().numpy() == want_c).all() and np.array_equal(gf.cpu().numpy(), want_f)
    S.input_transform(None, gf, normalize=True)
    assert np.array_equal(gf.cpu().numpy(), (torch.from_numpy(want_f) / 255. - 0.5).numpy())       # `lib/train.py:114` on torch
    with pytest.raises(Exception, match="colour maximum"):
        S.input_transform(gc, torch.full_like(gf, 0.5), contrast=True, blend=0.5)


def _cfg(root, **data):
    d = dict(scannet_path=str(root), stanford3d_path=str(root), ignore_label=255, return_transformation=False, voxel_size=None)
    d.update(data)
    return refload.Cfg(data=d, augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
                       optimizer=dict(optimizer="SGD", lr=0.01, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=2,
                                      scheduler="PolyLR", max_iter=100, poly_power=0.9))


@pytest.mark.parametrize("s", [0, 1])
def test_pipeline_replays_the_reference(tmp_path, s):
    """The golden scene as a `.ply` on disk, through the dataset class with the recorded draws: the reference's voxels, features,
    labels and transformation."""
    from pointcontrast_b200 import semseg_data as S, synth
    z = np.load(GOLDEN)
    pre = f"s{s}_"
    name = str(z[pre + "name"])
    (tmp_path / "splits").mkdir()
    synth.write_ply(tmp_path / "scene.ply", z[pre + "xyz"], z[pre + "rgb"], z[pre + "label"])
    cls = S.ScannetVoxelization2cmDataset if name == "scannet2cm" else S.StanfordDataset
    (tmp_path / "splits" / cls.DATA_PATH_FILE["Train"]).write_text("scene.ply\n")
    draws = S.ReplayDraws(O.read_draws(z, pre), "cuda")
    kw = dict(split_dir=str(tmp_path / "splits")) if name == "scannet2cm" else {}
    loader = S.initialize_data_loader(cls, _cfg(tmp_path, return_transformation=True), "train", shuffle=False, augment_data=True,
                                      batch_size=1, limit_numpoints=0, draws=draws, **kw)
    coords, feats, labels, trans = loader.dataset[0]
    assert draws.pos == len(draws.record)
    assert coords.shape == z[pre + "coords"].shape and (coords.cpu().numpy() == z[pre + "coords"]).all()
    assert (labels.cpu().numpy() == z[pre + "labels"]).all()
    assert np.array_equal(feats.cpu().numpy(), z[pre + "feats"])
    assert np.abs(trans - z[pre + "transformation"]).max() <= 1e-6 * np.abs(z[pre + "transformation"]).max()


def _scenes(root, n_scenes=4, n_raw=60_000):
    from pointcontrast_b200 import synth
    (root / "splits").mkdir(exist_ok=True)
    names = []
    for k in range(n_scenes):
        xyz, rgb, lab = synth.synth_labelled_room(100 + k, n_raw, scale=1.0 + 0.1 * k)
        synth.write_ply(root / f"scene{k:04d}_00.ply", xyz, rgb, lab)
        names.append(f"scene{k:04d}_00.ply")
    (root / "splits" / "scannetv2_train.txt").write_text("\n".join(names) + "\n")


def _seed(k):
    random.seed(k); np.random.seed(k); torch.manual_seed(k)


def _loader(root, draws, **kw):
    from pointcontrast_b200 import semseg_data as S
    args = dict(shuffle=True, augment_data=True, batch_size=2, limit_numpoints=0, iter_size=2, normalize_color=True)
    args.update(kw)
    return S.initialize_data_loader(S.ScannetVoxelization2cmDataset, _cfg(root), "train", draws=draws, split_dir=str(root / "splits"), **args)


def test_end_to_end_train_step_and_determinism(tmp_path):
    """PLY scenes + split file -> `ScannetVoxelization2cmDataset` -> loader (batch 2, iter_size 2) -> one finetune step; then the
    collate's `limit_numpoints` truncation; then a second run with the same seeds gives identical batches."""
    from pointcontrast_b200 import semseg, semseg_data as S
    from pointcontrast_b200.model import load_model
    from tests.helpers import det_init
    _scenes(tmp_path)
    _seed(0)
    gen = torch.Generator(device="cuda"); gen.manual_seed(0)
    loader = _loader(tmp_path, S.Draws("cuda", gen))
    batch = next(iter(loader))
    assert len(batch) == 2
    for coords, feats, target in batch:
        assert coords.dtype == torch.int32 and coords.shape[1] == 4 and feats.shape == (len(coords), 3) and len(target) == len(coords)
        assert coords[:, 0].unique().tolist() == [0, 1]
        assert (coords[:, 0][1:] >= coords[:, 0][:-1]).all()                       # scenes concatenated in order
        t = target.cpu()
        assert (((t >= 0) & (t < 20)) | (t == 255)).all() and (t == 255).any() and (t < 20).any()
        assert feats.min() >= -0.5 and feats.max() <= 0.5 + 1e-5                    # normalize_color
    mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
    net = load_model("Res16UNet34C")(3, 20, mcfg, D=3)
    det_init(net, 1)
    tr = semseg.SegmentationTrainer(net, _cfg(tmp_path))
    loss = float(tr.train_step(batch))
    assert np.isfinite(loss) and 0 < loss < 20

    # limit_numpoints (`transforms.py:251-283`): the batch stops before the scene that would exceed the limit
    items = [loader.dataset[k] for k in range(3)]
    sizes = [len(it[0]) for it in items]
    col = S.cfl_collate_fn_factory(sizes[0] + sizes[1] + sizes[2] // 2)
    c, f, l = col(items)
    assert len(c) == sizes[0] + sizes[1] and c[:, 0].max() == 1
    assert torch.equal(c[:, 1:], torch.cat([items[0][0], items[1][0]])) and torch.equal(f, torch.cat([items[0][1], items[1][1]]))
    c, _, _ = S.cfl_collate_fn_factory(0)(items)
    assert len(c) == sum(sizes) and c[:, 0].max() == 2

    # determinism: the same seeds give the same batches
    runs = []
    for _ in range(2):
        _seed(3)
        gen = torch.Generator(device="cuda"); gen.manual_seed(3)
        it = iter(_loader(tmp_path, S.Draws("cuda", gen)))
        runs.append([next(it) for _ in range(2)])
    for b0, b1 in zip(runs[0], runs[1]):
        for x0, x1 in zip(b0, b1):
            for a, b in zip(x0, x1):
                assert torch.equal(a, b)
