"""pointcontrast_b200.det_eval and csrc/det_eval.cu against the oracle (oracle/det_eval_cpu.py) and the original's numbers
(tests/golden/detection_eval.npz): decoding, points per box, NMS masks, oriented IoU and VOC AP; at
ScanNet-val batch size; and, where oracle/det_eval_ref.py staged the original, its unmodified `lib/test.py::test` with and without
`det_eval.install()`.

The oracle's softmax takes each fp32 `exp` from fp64 `exp`, as the kernel does, so the 2-ulp score check against the oracle mostly
confirms that shared choice; agreement with the reference's own numpy fp32 `exp` rests on the 4-ulp oracle-vs-golden check of
tests/test_oracle_det_eval.py and on the end-to-end comparison below."""
import logging
import sys
import types

import numpy as np
import pytest
import torch

from oracle import det_eval_cpu as O
from tests.test_oracle_det_eval import DATASETS, GOLDEN, VARIANTS, flatten, golden, ulps

pytestmark = pytest.mark.gpu


class Config:
    """The dataset-config surface det_eval reads (model_util_scannet.py / model_util_sunrgbd.py)."""

    def __init__(self, dname, mean_size):
        d = DATASETS[dname]
        self.num_class, self.num_heading_bin, self.num_size_cluster = d["num_class"], d["H"], len(mean_size)
        self.mean_size_arr, self.rule = mean_size, d["rule"]
        self.class2type = {c: f"c{c}" for c in range(self.num_class)}

    def class2angle(self, pred_cls, residual, to_label_format=True):
        return O.class2angle(self.rule, pred_cls, residual, self.num_heading_bin)


def cuda(ep):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.items()}


@pytest.fixture(scope="module")
def det():
    from pointcontrast_b200 import det_eval
    return det_eval


@pytest.mark.parametrize("dname", sorted(DATASETS))
@pytest.mark.parametrize("vname", sorted(VARIANTS))
def test_parse_matches_oracle(det, dname, vname):
    z, ep = golden(dname)
    cfg = Config(dname, z[f"{dname}/mean_size"])
    cd = dict(VARIANTS[vname], dataset_config=cfg)
    e = cuda(ep)
    pred = det.parse_predictions(e, cd)
    gt = det.parse_groundtruths(e, cd)
    ocfg = dict(VARIANTS[vname], mean_size=cfg.mean_size_arr, rule=cfg.rule, num_class=cfg.num_class)
    mask_o, lists_o, corners_o = O.parse_predictions(ep, ocfg)
    assert np.array_equal(e["pred_mask"], mask_o)
    assert np.array_equal(e["pred_mask"], z[f"{dname}/{vname}/pred_mask"])
    assert np.abs(pred.corners.cpu().numpy() - corners_o).max() <= 1e-12
    got, want = flatten([pred[i] for i in range(len(pred))]), flatten(lists_o)
    assert [(i, c) for i, c, _, _ in got] == [(i, c) for i, c, _, _ in want]
    assert ulps([s for *_, s in got], [s for *_, s in want]).max(initial=0) <= 2
    _, gl = O.decode_gt(ep, cfg.mean_size_arr, cfg.rule, cfg.num_heading_bin)
    gg = [gt[i] for i in range(len(gt))]
    assert [(i, c) for i, lst in enumerate(gg) for c, _ in lst] == [(i, c) for i, lst in enumerate(gl) for c, _ in lst]
    assert max(np.abs(a[1] - b[1]).max() for la, lb in zip(gg, gl) for a, b in zip(la, lb)) <= 1e-12
    for thr in (0.25, 0.5):
        calc = det.APCalculator(thr, cfg.class2type)
        calc.step(pred, gt)
        m = calc.compute_metrics()
        mo = O.metrics(lists_o, gl, thr, cfg.class2type)
        assert list(m) == list(mo)
        np.testing.assert_allclose([m[k] for k in m], [mo[k] for k in mo], rtol=0, atol=1e-12, equal_nan=True)


@pytest.mark.parametrize("dname", sorted(DATASETS))
def test_points_per_box_exact(det, dname):
    z, ep = golden(dname)
    cfg = Config(dname, z[f"{dname}/mean_size"])
    _, params, *_ = O.decode_pred(ep, cfg.mean_size_arr, cfg.rule)
    e = cuda(ep)
    _, box, *_ = det.decode_predictions(e, cfg)
    counts = det.points_in_boxes(e["point_clouds"], box).cpu().numpy()
    pc = ep["point_clouds"][:, :, :3]
    want = np.array([[O.points_in_box(pc[i], params[i, j]) for j in range(params.shape[1])] for i in range(params.shape[0])])
    assert np.array_equal(counts, want)


@pytest.mark.parametrize("dname", sorted(DATASETS))
@pytest.mark.parametrize("vname", sorted(VARIANTS))
def test_ap_on_reference_detections(det, dname, vname):
    """APCalculator fed the golden's own (reference) detection and ground-truth lists: the reference's metric dict within 1e-12."""
    z, _ = golden(dname)
    key = f"{dname}/{vname}"
    B = int(max(z[key + "/gt"][:, 0].max(initial=0), z[key + "/pred"][:, 0].max(initial=0))) + 1
    preds, gts = [[] for _ in range(B)], [[] for _ in range(B)]
    for (i, c, s), b in zip(z[key + "/pred"], z[key + "/pred_corners"]):
        preds[int(i)].append((int(c), b, np.float32(s)))
    for (i, c), b in zip(z[key + "/gt"], z[key + "/gt_corners"]):
        gts[int(i)].append((int(c), b))
    for thr in (0.25, 0.5):
        calc = det.APCalculator(thr)
        calc.step(preds, gts)
        m = calc.compute_metrics()
        np.testing.assert_allclose([float(v) for v in m.values()], z[f"{key}/metrics_{thr}/values"], rtol=0, atol=1e-12, equal_nan=True)


def box(c, size, a=0.0):
    return O.get_3d_box(size, a, c)


def test_ap_ties_equal_oracle(det):
    """Saturated scores: many exact ties of 1.0 across scans and classes; AP and recall equal to the oracle's stable order."""
    g = np.random.default_rng(7)
    preds, gts = [], []
    for s in range(6):
        centers = g.uniform(-3, 3, (8, 3))
        gts.append([(int(g.integers(0, 3)), box(c, [1, 1, 1], g.uniform(-1, 1))) for c in centers])
        preds.append([(int(g.integers(0, 3)), box(centers[g.integers(0, 8)] + g.normal(0, 0.2, 3), [1, 1, 1], g.uniform(-1, 1)),
                       np.float32(1.0) if g.random() < 0.6 else np.float32(g.random())) for _ in range(20)])
    for thr in (0.25, 0.5):
        calc = det.APCalculator(thr)
        calc.step(preds, gts)
        m = calc.compute_metrics()
        mo = O.metrics(preds, gts, thr)
        assert list(m) == list(mo)
        np.testing.assert_allclose([m[k] for k in m], [mo[k] for k in mo], rtol=0, atol=1e-12, equal_nan=True)


def test_nms_ties_zero_area_and_modes(det):
    """Equal scores pick the larger index first; NaN scores rank above every number; a zero-area box (0/0 overlap) never suppresses or
    is suppressed."""
    g = np.random.default_rng(11)
    B, K = 3, 200
    c = g.uniform(-2, 2, (B, K, 3))
    size = g.uniform(0.2, 1.5, (B, K, 3))
    size[:, ::17] = 0.0
    corners = np.array([[box(c[i, j], size[i, j], g.uniform(-np.pi, np.pi)) for j in range(K)] for i in range(B)])
    score = np.round(g.random((B, K)) * 8).astype(np.float32) / 8
    score[:, ::23] = np.nan                                                 # a NaN objectness (diverged net): picked first, as np.argsort
    score[:, 5::29] = -0.0                                                  # -0.0 ties +0.0
    cls = g.integers(0, 4, (B, K)).astype(np.int32)
    counts = g.integers(0, 10, (B, K)).astype(np.int32)
    for mode_name, mode in (("2d", 0), ("3d", 1), ("3d_samecls", 2)):
        for old in (False, True):
            got = det.nms(torch.from_numpy(corners).cuda(), torch.from_numpy(score).cuda(), torch.from_numpy(cls).cuda(),
                          torch.from_numpy(counts).cuda(), mode_name, old, 0.25).cpu().numpy()
            for i in range(B):
                inds = np.where(counts[i] >= 5)[0]
                want = np.zeros(K, np.int32)
                want[inds[O.nms(O.nms_boxes(corners[i, inds], mode), score[i, inds], mode, 0.25, old, cls[i, inds])]] = 1
                assert np.array_equal(got[i], want), (mode_name, old, i)


def test_det_ap_matches_oracle(det):
    import ctypes
    from pointcontrast_b200 import _lib
    g = np.random.default_rng(3)
    P, D, G, C = 300, 900, 120, 7
    prop = torch.from_numpy(np.array([box(g.uniform(-2, 2, 3), g.uniform(0.3, 1.5, 3), g.uniform(-3, 3)) for _ in range(P)])).cuda()
    gtc = torch.from_numpy(np.array([box(g.uniform(-2, 2, 3), g.uniform(0.3, 1.5, 3), g.uniform(-3, 3)) for _ in range(G)])).cuda()
    t = lambda a, dt: torch.from_numpy(np.asarray(a, dt)).cuda()
    row, cls = t(g.integers(0, P, D), np.int32), t(g.integers(-1, C, D), np.int32)
    score, scan = t(np.round(g.random(D) * 16) / 16, np.float32), t(np.sort(g.integers(0, 4, D)), np.int32)     # accumulation order
    gscan, gcls = t(g.integers(0, 4, G), np.int32), t(g.integers(-1, C, G), np.int32)
    thr = (ctypes.c_double * 3)(0.1, 0.25, 0.5)
    q = _lib.lib.pcb_det_ap_ws_bytes(D, G, C, 3)
    ws = torch.empty(q, dtype=torch.uint8, device="cuda")
    out = torch.empty(3, C, 4, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib.pcb_det_ap(prop.data_ptr(), P, row.data_ptr(), cls.data_ptr(), score.data_ptr(), scan.data_ptr(), D, gtc.data_ptr(),
                                   gscan.data_ptr(), gcls.data_ptr(), G, C, ctypes.addressof(thr), 3, out.data_ptr(), ws.data_ptr(), q,
                                   _lib.stream()))
    out = out.cpu().numpy()
    pc, gc = prop.cpu().numpy(), gtc.cpu().numpy()
    rn, cn, sn, scn = row.cpu().numpy(), cls.cpu().numpy(), score.cpu().numpy(), scan.cpu().numpy()
    preds = [[(int(cn[d]), pc[rn[d]], sn[d]) for d in range(D) if scn[d] == s and cn[d] >= 0] for s in range(4)]
    gts = [[(int(c), gc[j]) for j, c in enumerate(gcls.cpu().numpy()) if gscan[j] == s and c >= 0] for s in range(4)]
    for ti, th in enumerate((0.1, 0.25, 0.5)):
        res = O.eval_det(preds, gts, th)
        for c in range(C):
            if c in res:
                np.testing.assert_allclose(out[ti, c], res[c], rtol=0, atol=1e-12, equal_nan=True)
            else:
                assert out[ti, c, 2] == 0 and out[ti, c, 3] == 0


def box_iou(det, c1, c2):
    from pointcontrast_b200 import _lib
    a, b = (torch.from_numpy(np.ascontiguousarray(c, np.float64)).cuda() for c in (c1, c2))
    out = torch.empty(len(a), dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib.pcb_det_box_iou(a.data_ptr(), b.data_ptr(), len(a), out.data_ptr(), _lib.stream()))
    return out.cpu().numpy()


def test_box_iou_kernel_on_golden_and_seeded_pairs(det):
    """The kernel's box3d_iou: within 1e-12 of the reference on the golden pairs, and of the oracle on seeded rotated and mirrored
    (negative-size) boxes, nested and disjoint ones included."""
    z = np.load(GOLDEN)
    pairs = z["iou/pairs"]
    assert np.abs(box_iou(det, pairs[:, 0], pairs[:, 1]) - z["iou/value"]).max() <= 1e-12
    g = np.random.default_rng(21)
    c1, c2 = [], []
    for _ in range(400):
        c = g.uniform(-1, 1, 3)
        c1.append(box(c, g.uniform(0.3, 2, 3) * g.choice([-1, 1], 3, p=[0.2, 0.8]), g.uniform(-np.pi, np.pi)))
        c2.append(box(c + g.normal(0, 0.4, 3), g.uniform(0.3, 2, 3) * g.choice([-1, 1], 3, p=[0.2, 0.8]), g.uniform(-np.pi, np.pi)))
    got = box_iou(det, np.array(c1), np.array(c2))
    want = np.array([O.box3d_iou(a, b) for a, b in zip(c1, c2)])
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12, equal_nan=True)


class ScanNetLike:
    """ScanNet's config shape (18 classes, one heading bin, class2angle 0) with seeded mean sizes."""
    num_class, num_heading_bin, num_size_cluster = 18, 1, 18
    rule = 0

    def __init__(self):
        self.mean_size_arr = np.random.default_rng(0).uniform(0.3, 2.0, (18, 3))
        self.class2type = {c: f"class{c}" for c in range(18)}

    def class2angle(self, pred_cls, residual, to_label_format=True):
        return 0


def scannet_val_batch(seed, cfg, B=8, K=256, N=40000, K2=64):
    g = np.random.default_rng(seed)
    gt_center = np.concatenate([g.uniform(-3, 3, (B, K2, 2)), g.uniform(0.2, 1.7, (B, K2, 1))], -1).astype(np.float32)
    src = g.integers(0, K2, (B, K))
    sc = g.integers(0, 18, (B, K2))
    f = lambda a: np.asarray(a, np.float32)
    return {
        "center": f(np.take_along_axis(gt_center, src[..., None].repeat(3, -1), 1) + g.normal(0, 0.15, (B, K, 3))),
        "heading_scores": f(g.normal(0, 1, (B, K, 1))), "heading_residuals": f(g.normal(0, 0.1, (B, K, 1))),
        "size_scores": f(g.normal(0, 1, (B, K, 18))), "size_residuals": f(g.normal(0, 0.1, (B, K, 18, 3))),
        "sem_cls_scores": f(g.normal(0, 2, (B, K, 18))), "objectness_scores": f(g.normal(0, 2, (B, K, 2))),
        "point_clouds": f(np.concatenate([g.uniform(-3.5, 3.5, (B, N, 2)), g.uniform(0, 2, (B, N, 1)), g.random((B, N, 1))], -1)),
        "center_label": gt_center, "heading_class_label": np.zeros((B, K2), np.int64), "heading_residual_label": f(np.zeros((B, K2))),
        "size_class_label": sc, "size_residual_label": f(g.normal(0, 0.05, (B, K2, 3))), "sem_cls_label": sc,
        "box_label_mask": f(g.random((B, K2)) < 0.4),
    }


@pytest.mark.parametrize("vname", ["test", "train"])
def test_scannet_val_size_against_oracle(det, vname):
    """One batch at the ScanNet-val shape (B = 8, K = 256, 18 classes, 40 000 points, 64 label slots): masks, detection sets and the
    metric dicts at 0.25 / 0.5 against the oracle."""
    cfg = ScanNetLike()
    ep = scannet_val_batch(5, cfg)
    cd = dict(VARIANTS[vname], dataset_config=cfg)
    e = cuda(ep)
    pred, gt = det.parse_predictions(e, cd), det.parse_groundtruths(e, cd)
    mask_o, lists_o, _ = O.parse_predictions(ep, dict(VARIANTS[vname], mean_size=cfg.mean_size_arr, rule=0, num_class=18))
    assert np.array_equal(e["pred_mask"], mask_o)
    got, want = flatten([pred[i] for i in range(len(pred))]), flatten(lists_o)
    assert [(i, c) for i, c, _, _ in got] == [(i, c) for i, c, _, _ in want]
    assert ulps([s for *_, s in got], [s for *_, s in want]).max(initial=0) <= 2
    _, gl = O.decode_gt(ep, cfg.mean_size_arr, 0, 1)
    for thr in (0.25, 0.5):
        calc = det.APCalculator(thr, cfg.class2type)
        calc.step(pred, gt)
        m, mo = calc.compute_metrics(), O.metrics(lists_o, gl, thr, cfg.class2type)
        assert list(m) == list(mo)
        np.testing.assert_allclose([m[k] for k in m], [mo[k] for k in mo], rtol=0, atol=1e-12, equal_nan=True)


def test_out_of_range_label_raises(det):
    """A kept ground-truth slot with a size class outside the config raises when the labels are read; a dropped slot may hold anything."""
    z, ep = golden("scannet")
    cfg = Config("scannet", z["scannet/mean_size"])
    cd = dict(VARIANTS["test"], dataset_config=cfg)
    ep = dict(ep, size_class_label=ep["size_class_label"].copy(), box_label_mask=ep["box_label_mask"].copy())
    ep["box_label_mask"][0, 0] = 0
    ep["size_class_label"][0, 0] = 99                                       # dropped slot: ignored, as the reference skips it
    e = cuda(ep)
    calc = det.APCalculator(0.25)
    calc.step(det.parse_predictions(e, cd), det.parse_groundtruths(e, cd))
    calc.compute_metrics()
    ep["box_label_mask"][0, 0] = 1                                          # kept slot: an error
    e = cuda(ep)
    gt = det.parse_groundtruths(e, cd)
    with pytest.raises(Exception, match="outside the dataset config"):
        gt[0]
    calc = det.APCalculator(0.25)
    calc.step(det.parse_predictions(e, cd), gt)
    with pytest.raises(Exception, match="outside the dataset config"):
        calc.compute_metrics()


# ------------------------------------------------------------------------------------------------ the original's lib/test.py::test

def _run_reference_test(ref_ap, det, install, dname, vname, ep_batches, cfg):
    """The original's unmodified lib/test.py::test over ep_batches, fed by a stand-in net (the batch's predictions) and criterion (a
    constant loss); the PLY dump of batch 0 is out of scope and replaced by a no-op.  Returns the logged 'eval <key>: <value>' lines."""
    import importlib
    pkg = sys.modules["models"]
    saved = sys.modules["models.ap_helper"]
    pred_keys = ("center", "heading_scores", "heading_residuals", "size_scores", "size_residuals", "sem_cls_scores", "objectness_scores")
    try:
        if install:
            det.install()
        sys.modules.pop("lib.test", None)
        T = importlib.import_module("lib.test")
        calls = iter(range(len(ep_batches)))

        class Net:
            def eval(self):
                return self

            def __call__(self, inputs):
                i = next(calls)
                return {k: torch.from_numpy(np.ascontiguousarray(ep_batches[i][k])).cuda() for k in pred_keys}

        def criterion(end_points, dataset_config):
            end_points["loss"] = torch.tensor(0.5, device="cuda")
            return end_points["loss"], end_points

        T.criterion = criterion
        T.dump_results = lambda *a, **k: None
        loader = [{k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in b.items() if k not in pred_keys} for b in ep_batches]
        v = VARIANTS[vname]
        config = types.SimpleNamespace(test=types.SimpleNamespace(
            use_cls_nms=v["cls_nms"], use_3d_nms=v["use_3d_nms"], faster_eval=not v["remove_empty_box"], nms_iou=v["nms_iou"],
            use_old_type_nms=v["use_old_type_nms"], per_class_proposal=v["per_class_proposal"], conf_thresh=v["conf_thresh"],
            ap_iou_thresholds=[0.25, 0.5]))
        lines = []
        handler = logging.Handler(logging.INFO)
        handler.emit = lambda r: lines.append(r.getMessage())
        root = logging.getLogger()
        old_level = root.level
        root.addHandler(handler)
        root.setLevel(logging.INFO)
        try:
            T.test(Net(), loader, cfg, config)
        finally:
            root.removeHandler(handler)
            root.setLevel(old_level)
        assert T.APCalculator is (det.APCalculator if install else ref_ap.APCalculator)
    finally:
        sys.modules["models.ap_helper"] = saved
        pkg.ap_helper = saved
        sys.modules.pop("lib.test", None)
    return [l for l in lines if l.startswith("eval ") or l.startswith("-")]


@pytest.mark.parametrize("dname", sorted(DATASETS))
@pytest.mark.parametrize("vname", sorted(VARIANTS))
def test_reference_test_loop_with_and_without_install(det, dname, vname):
    """lib/test.py::test logs the same metrics (as it prints them, %f) with the original's ap_helper and after det_eval.install(), on
    the golden scenes split into two batches, with the dataset's own model-util config."""
    from oracle import det_eval_ref
    ref_ap = det_eval_ref.load()
    if ref_ap is None:
        pytest.skip("the original VoteNet evaluation code is not staged (oracle/det_eval_ref.py)")
    import importlib
    mod = importlib.import_module("lib.datasets.%s.model_util_%s" % (dname, dname))
    cfg = (mod.ScannetDatasetConfig if dname == "scannet" else mod.SunrgbdDatasetConfig)()
    _, ep = golden(dname)
    batches = [{k: v[i:i + 1] for k, v in ep.items()} for i in range(ep["center"].shape[0])]
    ref = _run_reference_test(ref_ap, det, False, dname, vname, batches, cfg)
    ours = _run_reference_test(ref_ap, det, True, dname, vname, batches, cfg)
    assert len(ref) == len(ours) and len(ref) > 4
    for a, b in zip(ref, ours):
        ka, _, va = a.rpartition(": ")
        kb, _, vb = b.rpartition(": ")
        assert ka == kb
        if ka.startswith("eval "):
            fa, fb = float(va), float(vb)
            assert (np.isnan(fa) and np.isnan(fb)) or abs(fa - fb) <= 1.5e-6, (a, b)
