"""csrc/det_data.cu and pointcontrast_b200.det_data on the GPU: floor heights bit for bit against numpy, the choice sets' properties, a
replay of tests/golden/det_data.npz (the original's items under recorded draws), ragged batches of several scenes against the numpy
restatement (oracle/det_data_cpu.py) scene by scene, and the loader end to end into one VoteNet step.

Comparison rule: integers and masks exact; fp32 values equal (`==`: the signed zeros of padded box rows are not pinned) or 1 ulp apart,
where numpy's BLAS sums the three fp64 products of a rotation in another order (with FMA), at most 0.3 % of the elements; fp64
`max_gt_bboxes` within 8e-14 (that BLAS rounding of a rotated centre whose terms reach ~5 m, before any cancellation)."""
import numpy as np
import pytest
import torch

from oracle import det_data_cpu as O
from pointcontrast_b200 import det_data, detection, synth
from pointcontrast_b200.semseg_data import Draws, ReplayDraws
from tests.test_oracle_det_data import NUM_POINTS, SCANNET, SUNRGBD, cases, draws_of, golden, parse  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_floor_height_matches_numpy(dtype):
    rng = np.random.default_rng(0)
    # n = 1, ties, negative z, and sizes around which the 0.99th percentile's interpolation weight crosses 0.5
    sizes = [1, 2, 3, 50, 51, 52, 101, 102, 152, 153, 1000, 5051, 40000]
    scenes = []
    for i, n in enumerate(sizes):
        z = rng.normal(-1.0, 2.0, n)
        if i % 3 == 0:
            z = np.round(z * 4) / 4                 # many ties
        scenes.append(z.astype(dtype))
    rows = np.zeros((sum(sizes), 6), dtype)
    rows[:, 2] = np.concatenate(scenes)
    off = np.zeros(len(sizes) + 1, np.int64)
    off[1:] = np.cumsum(sizes)
    got = det_data.floor_height(torch.from_numpy(rows).cuda()[:, 2], off).cpu().numpy()
    want = np.array([np.percentile(z, 0.99) for z in scenes])
    assert np.array_equal(got, want.astype(np.float64)), (got - want)
    crosses = [(np.float32(0.99) / np.float32(100) * np.float32(n - 1)) % 1 >= 0.5 for n in sizes]
    assert any(crosses) and not all(crosses)


def test_choice_sets():
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    d = Draws("cuda", g)
    ns, k = [10, 1000, 3, 250, 40000], 250
    a = d.choices(ns, k).cpu().numpy()
    assert a.shape == (len(ns), k)
    for n, c in zip(ns, a):
        assert c.min() >= 0 and c.max() < n
        if n >= k:
            assert len(np.unique(c)) == k
    g.manual_seed(5)
    assert np.array_equal(Draws("cuda", g).choices(ns, k).cpu().numpy(), a)
    assert not np.array_equal(d.choices(ns, k).cpu().numpy(), a)
    # frequencies over many draws: each of 6 points lands in each of the 3 ordered slots 1/6 of the time; iid indices uniform
    hits, iid = np.zeros((6, 3)), np.zeros(4)
    T = 4000
    for _ in range(T // 50):
        c = d.choices([6] * 50 + [4] * 50, 3).cpu().numpy()
        for row in c[:50]:
            hits[row, np.arange(3)] += 1
        iid += np.bincount(c[50:].ravel(), minlength=4)
    assert np.abs(hits / T - 1 / 6).max() < 0.03
    assert np.abs(iid / iid.sum() - 0.25).max() < 0.02


def _config(dataset):
    from oracle import det_data_ref
    mods = det_data_ref.load()
    if mods is None:
        pytest.skip("the original dataset configs are not staged under oracle/_ref/")
    return mods, (mods[0].DC if dataset == "scannet" else mods[1].DC)


def _library_record(records):
    """The original's per-scene draws in the order this library asks for them: every scene's scalars and colour arrays, then one
    choice-set draw for all scenes."""
    out, choices = [], []
    for record in records:
        for kind, v in record:
            if kind == "choice":
                choices.append(v)
            elif v.ndim == 0 or len(v) == 3:
                out.append(("rand", v))
            else:
                out.append(("rand_device", v))
    return out + [("choices", choices)]


def _compare(got, want, where):
    """(elements 1 ulp apart, elements compared) under the module's comparison rule; asserts the rest."""
    off_by_ulp, total = 0, 0
    for k, w in want.items():
        g = got[k].cpu().numpy()
        w = np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape, (where, k)
        if w.dtype.kind in "iu" or k == "box_label_mask":
            assert np.array_equal(g, w), (where, k)
            continue
        diff = g != w
        if diff.any():
            tol = 8e-14 if w.dtype == np.float64 else np.spacing(np.abs(w[diff]).astype(w.dtype)).astype(np.float64)
            ulp = np.abs(g[diff].astype(np.float64) - w[diff]) <= tol
            assert ulp.all(), (where, k, g[diff][~ulp][:5], w[diff][~ulp][:5])
            off_by_ulp += int(diff.sum())
        total += g.size
    return off_by_ulp, total


def _dataset(dataset, path, dc, opt, draws, num_points=NUM_POINTS):
    if dataset == "scannet":
        split = path / "split.txt"
        split.write_text("\n".join(SCANNET) + "\n")
        return det_data.ScannetDetectionDataset("train", num_points, use_height=opt["h"], augment=opt["a"], data_path=str(path),
                                                split_file=str(split), dataset_config=dc, draws=draws)
    return det_data.SunrgbdDetectionVotesDataset("train", num_points, use_color=opt["c"], use_height=opt["h"], augment=opt["a"],
                                                 data_path=str(path), dataset_config=dc, draws=draws)


@pytest.mark.parametrize("dataset", ["scannet", "sunrgbd"])
def test_golden_replay(golden, dataset, tmp_path):  # noqa: F811
    mods, dc = _config(dataset)
    from tests.golden.make_det_data_golden import write_scenes
    write_scenes(str(tmp_path))
    off_by_ulp, total = 0, 0
    for case in cases(golden, dataset + "_"):
        s, opt = parse(case)
        ds = _dataset(dataset, tmp_path, dc, opt, ReplayDraws(_library_record([draws_of(golden, case)])))
        want = {k.split("/", 1)[1]: golden[k] for k in golden if k.startswith(case + "/") and "draw" not in k}
        o, t = _compare(ds[s], want, case)
        off_by_ulp, total = off_by_ulp + o, total + t
    assert off_by_ulp <= 3e-3 * total, (off_by_ulp, total)


class _ScannetConfig:
    nyu40ids = np.array(synth.SCANNET_NYU40IDS)
    mean_size_arr = np.random.default_rng(1).uniform(0.2, 2.0, (18, 3))
    num_heading_bin = 1
    type2class = {str(i): i for i in range(18)}


class _SunConfig:
    mean_size_arr = np.random.default_rng(2).uniform(0.2, 2.0, (10, 3))
    num_heading_bin = 12
    type2class = {str(i): i for i in range(10)}


# (points, boxes) per scene: N above and below num_points (300), N equal to it, K = 0 and K = 64
BATCH_SCENES = ((520, 5), (140, 0), (300, 64), (900, 17), (31, 2))


@pytest.mark.parametrize("dataset,opt", [("scannet", dict(a=True, h=True, c=False)), ("scannet", dict(a=True, h=False, c=False)),
                                         ("scannet", dict(a=False, h=True, c=False)), ("sunrgbd", dict(a=True, h=True, c=True)),
                                         ("sunrgbd", dict(a=True, h=False, c=False)), ("sunrgbd", dict(a=False, h=True, c=True))])
def test_ragged_batch_matches_oracle(dataset, opt, tmp_path):
    """One `_assemble` call over five ragged scenes (replayed draws) equals the numpy restatement of each scene's item under the same
    draws, scene by scene: a per-scene indexing slip (offsets, params, box offsets, floor heights, colour draws, or instance ids
    merged across scenes -- every scene holds instance ids 0 and 2^32 - 1) shows as a wrong slice."""
    k, sun = 300, dataset == "sunrgbd"
    names = [f"{i + 1:06d}" if sun else f"scene{i:04d}_00" for i in range(len(BATCH_SCENES))]
    for j, (name, (n, K)) in enumerate(zip(names, BATCH_SCENES)):
        if sun:
            synth.write_sunrgbd_detection_scene(str(tmp_path), name, 50 + j, n, K)
        else:
            synth.write_scannet_detection_scene(str(tmp_path), name, 50 + j, n, K)
    dc = _SunConfig() if sun else _ScannetConfig()
    rng = np.random.RandomState(11)
    records = []
    for n, _ in BATCH_SCENES:               # each scene's draws in the original's call order
        rec = [] if sun else [("choice", rng.choice(n, k, replace=n < k))]
        if opt["a"]:
            rec += [("random", np.asarray(rng.random_sample())) for _ in range(2 if sun else 3)]
            if sun and opt["c"]:
                rec += [("random", rng.random_sample(3)), ("random", rng.random_sample(3)), ("random", rng.random_sample(n)),
                        ("random", rng.random_sample(n))]
            if sun:
                rec += [("random", np.asarray(rng.random_sample()))]
        if sun:
            rec += [("choice", rng.choice(n, k, replace=n < k))]
        records.append(rec)
    if sun:
        ds = det_data.SunrgbdDetectionVotesDataset("train", k, use_color=opt["c"], use_height=opt["h"], augment=opt["a"],
                                                   data_path=str(tmp_path), dataset_config=dc, draws=ReplayDraws(_library_record(records)))
    else:
        split = tmp_path / "split.txt"
        split.write_text("\n".join(names) + "\n")
        ds = det_data.ScannetDetectionDataset("train", k, use_height=opt["h"], augment=opt["a"], data_path=str(tmp_path),
                                              split_file=str(split), dataset_config=dc, draws=ReplayDraws(_library_record(records)))
    idxs = list(range(len(names)))
    items = ds._read_batch(idxs)
    if not sun:
        common = set(items[0]["ins"])
        for it in items[1:]:
            common &= set(it["ins"])
        assert {0, 2 ** 32 - 1} <= common
    batch = ds._assemble(items, idxs)
    off_by_ulp, total = 0, 0
    for b, (it, record) in enumerate(zip(items, records)):
        it_draws = iter(record)

        def draws(kind, *a, **kw):
            kk, v = next(it_draws)
            assert kk == kind
            return v[()] if v.ndim == 0 else v.copy()
        if sun:
            want = O.sunrgbd_item(it["pc"], it["votes"], it["bbox"], dc.num_heading_bin, dc.mean_size_arr, k, opt["c"], opt["h"], opt["a"],
                                  b, draws)
        else:
            want = O.scannet_item(it["vert"], it["sem"], it["ins"], it["bbox"], dc.nyu40ids, dc.mean_size_arr, k, opt["h"], opt["a"], b,
                                  draws)
        o, t = _compare({key: v[b] for key, v in batch.items()}, want, (dataset, b))
        off_by_ulp, total = off_by_ulp + o, total + t
    assert off_by_ulp <= 3e-3 * total, (off_by_ulp, total)


@pytest.mark.parametrize("dataset", ["scannet", "sunrgbd"])
def test_loader_end_to_end(dataset, tmp_path):
    """Synthetic scenes on disk -> DetectionLoader(voxel_size=0.025): default_collate's keys, dtypes and shapes of the original's items,
    voxel fields equal to voxelize_batch on the same clouds, and one VoteNet training step with a finite loss."""
    mods, dc = _config(dataset)
    from oracle import det_data_ref
    from torch.utils.data import default_collate
    n_pts = 20000
    names = SCANNET if dataset == "scannet" else SUNRGBD
    for j, name in enumerate(names):
        if dataset == "scannet":
            synth.write_scannet_detection_scene(str(tmp_path), name, j, 30000 + 5000 * j, 10 + j, n_inst=30)
        else:
            synth.write_sunrgbd_detection_scene(str(tmp_path), name, j, 50000, 10)
    ds = _dataset(dataset, tmp_path, dc, {"h": False, "a": True, "c": False}, None, n_pts)
    loader = det_data.DetectionLoader(ds, 2, shuffle=True, voxel_size=0.025)
    batches = list(loader)
    assert len(batches) == 2 and [len(b["scan_idx"]) for b in batches] == [2, 1]
    cls = mods[0].ScannetDetectionDataset if dataset == "scannet" else mods[1].SunrgbdDetectionVotesDataset
    rng = np.random.RandomState(0)
    orig = [det_data_ref.item(cls, str(tmp_path), names, n_pts, False, False, True, i,
                              lambda kind, *a, **kw: rng.random_sample(*a) if kind == "random" else rng.choice(*a, **kw))
            for i in (0, 1)]
    want = default_collate(orig)
    b = batches[0]
    for k, v in want.items():
        assert k in b and b[k].dtype == v.dtype and tuple(b[k].shape) == tuple(v.shape) and b[k].is_cuda, k
        assert b[k].cuda() is b[k]
    assert set(b) - set(want) == {"voxel_coords", "voxel_inds", "voxel_feats"}
    ref = detection.voxelize_batch({"point_clouds": b["point_clouds"].clone()}, 0.025)
    for k in ("voxel_coords", "voxel_inds", "voxel_feats"):
        assert torch.equal(ref[k], b[k]), k
    # one training step: the sparse-conv backbone + the original VoteNet heads + det_loss
    from oracle import det_loss_ref
    if not det_loss_ref.available():
        pytest.skip("the original VoteNet heads are not staged under oracle/_ref/")
    import importlib
    from pointcontrast_b200 import det_loss
    from tests.test_host_detection import original_backbone_module
    original_backbone_module()
    votenet = importlib.import_module("models.votenet")
    torch.manual_seed(0)
    net = votenet.VoteNet(dc.num_class, dc.num_heading_bin, dc.num_size_cluster, dc.mean_size_arr, input_feature_dim=0,
                          num_proposal=256, vote_factor=1, sampling="vote_fps", backbone="sparseconv").cuda().train()
    end_points = net({k: b[k] for k in ("point_clouds", "voxel_coords", "voxel_inds", "voxel_feats")})
    for k, v in b.items():
        if k not in end_points:
            end_points[k] = v
    loss, end_points = det_loss.get_loss(end_points, dc)
    loss.backward()
    assert torch.isfinite(loss)
    assert sum(p.grad.abs().sum() for p in net.parameters() if p.grad is not None) > 0
