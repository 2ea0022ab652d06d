"""The detection-evaluation oracle (oracle/det_eval_cpu.py) against the original's own `ap_helper` / `nms` / `eval_det` / `box_util`
(tests/golden/detection_eval.npz), its point-in-box test against scipy's Delaunay, and the argument checks of the pcb_det_* entry
points, which run before anything touches the device."""
import os

import numpy as np
import pytest
import torch

from oracle import det_eval_cpu as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "detection_eval.npz")
VARIANTS = {
    "test": dict(remove_empty_box=True, use_3d_nms=False, nms_iou=0.25, use_old_type_nms=False, cls_nms=False, per_class_proposal=False,
                 conf_thresh=0.05),
    "test_old": dict(remove_empty_box=True, use_3d_nms=False, nms_iou=0.25, use_old_type_nms=True, cls_nms=False, per_class_proposal=False,
                     conf_thresh=0.05),
    "train": dict(remove_empty_box=False, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=False, cls_nms=True, per_class_proposal=True,
                  conf_thresh=0.05),
    "train_old": dict(remove_empty_box=False, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=True, cls_nms=True, per_class_proposal=True,
                      conf_thresh=0.05),
}
DATASETS = {"scannet": dict(rule=0, num_class=18, H=1), "sunrgbd": dict(rule=1, num_class=10, H=12)}
SCORE_ULP = 4       # fp32 exp rounded from fp64 against numpy's own fp32 exp (within 2 ulp), through the row sum and the division


def golden(dname):
    z = np.load(GOLDEN)
    ep = {k.split("/")[-1]: z[k] for k in z.files if k.startswith(dname + "/in/")}
    return z, ep


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def flatten(lists):
    return [(i, c, b, s) for i, lst in enumerate(lists) for c, b, s in lst]


@pytest.mark.parametrize("dname", sorted(DATASETS))
@pytest.mark.parametrize("vname", sorted(VARIANTS))
def test_oracle_reproduces_reference_parse_and_ap(dname, vname):
    z, ep = golden(dname)
    d = DATASETS[dname]
    cfg = dict(VARIANTS[vname], mean_size=z[f"{dname}/mean_size"], rule=d["rule"], num_class=d["num_class"])
    pred_mask, lists, _ = O.parse_predictions(ep, cfg)
    key = f"{dname}/{vname}"
    assert np.array_equal(pred_mask, z[key + "/pred_mask"])
    det = flatten(lists)
    ref = z[key + "/pred"]
    assert len(det) == len(ref)
    assert [(i, c) for i, c, _, _ in det] == [(int(i), int(c)) for i, c, _ in ref]
    assert ulps([s for *_, s in det], ref[:, 2]).max(initial=0) <= SCORE_ULP
    assert np.abs(np.array([b for _, _, b, _ in det]).reshape(-1, 8, 3) - z[key + "/pred_corners"]).max(initial=0) <= 1e-12
    gt_corners, gt_lists = O.decode_gt(ep, z[f"{dname}/mean_size"], d["rule"], d["H"])
    assert [(i, c) for i, lst in enumerate(gt_lists) for c, _ in lst] == [tuple(x) for x in z[key + "/gt"].tolist()]
    assert np.abs(np.array([b for lst in gt_lists for _, b in lst]).reshape(-1, 8, 3) - z[key + "/gt_corners"]).max(initial=0) <= 1e-12
    # AP fed the reference's own detections (its scores and corners): the metric dict within 1e-12
    B = len(lists)
    ref_lists = [[] for _ in range(B)]
    for (i, c, s), b in zip(ref, z[key + "/pred_corners"]):
        ref_lists[int(i)].append((int(c), b, np.float32(s)))
    gt_ref = [[] for _ in range(B)]
    for (i, c), b in zip(z[key + "/gt"], z[key + "/gt_corners"]):
        gt_ref[int(i)].append((int(c), b))
    for thr in (0.25, 0.5):
        m = O.metrics(ref_lists, gt_ref, thr, dict(enumerate(z[f"{dname}/class_names"].tolist())))
        keys, vals = z[f"{key}/metrics_{thr}/keys"], z[f"{key}/metrics_{thr}/values"]
        assert list(m) == keys.tolist()
        np.testing.assert_allclose(np.array([float(v) for v in m.values()]), vals, rtol=0, atol=1e-12, equal_nan=True)


def test_oracle_iou_matches_reference_pairs():
    z = np.load(GOLDEN)
    got = np.array([O.box3d_iou(a, b) for a, b in z["iou/pairs"]])
    assert np.abs(got - z["iou/value"]).max() <= 1e-12


def test_stable_tie_orders():
    """NMS: among equal scores the larger index is picked first; AP: equal scores keep accumulation order."""
    c = np.array([[0, 0, 1, 1], [0.1, 0.1, 1.1, 1.1], [5, 5, 6, 6]], np.float64)
    assert O.nms(c, [0.5, 0.5, 0.5], 0, 0.25, False) == [2, 1]
    box = O.get_3d_box([1, 1, 1], 0.0, [0, 0, 0])
    far = O.get_3d_box([1, 1, 1], 0.0, [9, 0, 0])
    # two detections of one gt with the same score: the first accumulated is the true positive
    ap = O.eval_det([[(0, box, np.float32(1.0)), (0, far, np.float32(1.0))]], [[(0, box)]], 0.25)[0]
    assert ap[0] == 1.0
    ap = O.eval_det([[(0, far, np.float32(1.0)), (0, box, np.float32(1.0))]], [[(0, box)]], 0.25)[0]
    assert ap[0] == 0.5


def test_empty_class_rules():
    box = O.get_3d_box([1, 1, 1], 0.0, [0, 0, 0])
    r = O.eval_det([[(1, box, np.float32(0.9))]], [[(0, box)]], 0.25)
    assert np.isnan(r[1][0]) and np.isnan(r[1][1])           # predictions, no ground truth: NaN
    assert r[0][:2] == (0.0, 0.0)                             # ground truth, no predictions: 0


def test_points_in_box_matches_delaunay():
    spatial = pytest.importorskip("scipy.spatial")
    g = np.random.default_rng(5)
    pc = g.uniform(-2, 2, (4000, 3)).astype(np.float32)
    for _ in range(12):
        params = [*g.uniform(-0.5, 0.5, 3), *(g.uniform(0.4, 2.0, 3) * g.choice([-1, 1], 3)), g.uniform(-np.pi, np.pi)]
        corners = O.get_3d_box(params[3:6], params[6], params[:3])
        depth = np.stack([corners[:, 0], corners[:, 2], -corners[:, 1]], 1)             # flip_axis_to_depth
        inside = spatial.Delaunay(depth).find_simplex(pc.astype(np.float64)) >= 0
        assert O.points_in_box(pc, params) == int(inside.sum())


# ------------------------------------------------------------------------------------------------ argument checks (no GPU needed)

def _lib():
    from pointcontrast_b200 import _lib
    return _lib.lib


def test_det_entry_points_reject_bad_arguments():
    L = _lib()
    f = torch.zeros(64)
    p = f.data_ptr()
    for rc in (L.pcb_det_decode_pred(p, p, p, p, p, p, p, 0, 4, 1, 1, 1, p, 0, p, p, p, p, p, None),
               L.pcb_det_decode_pred(p, p, p, p, p, p, p, 1, 4, 1, 1, 1025, p, 0, p, p, p, p, p, None),
               L.pcb_det_decode_pred(p, p, p, p, p, p, p, 1, 4, 1, 1, 1, p, 2, p, p, p, p, p, None),
               L.pcb_det_decode_pred(None, p, p, p, p, p, p, 1, 4, 1, 1, 1, p, 0, p, p, p, p, p, None),
               L.pcb_det_decode_gt(p, p, p, p, p, 1, 0, 1, 1, p, 0, p, p, p, None),
               L.pcb_det_decode_gt(p, p, p, p, p, 1, 4, 1, 1, p, 3, p, p, p, None),
               L.pcb_det_points_in_box(p, 1, 10, 2, p, 4, p, None),
               L.pcb_det_points_in_box(p, 1, 0, 3, p, 4, p, None),
               L.pcb_det_points_in_box(p, 1, 65536 * 4096, 3, p, 4, p, None),          # more point splits than gridDim.z holds
               L.pcb_det_box_iou(p, p, 0, p, None),
               L.pcb_det_box_iou(p, None, 4, p, None),
               L.pcb_det_nms(p, p, p, None, 5, 1, 1025, 0, 0, 0.25, p, None),
               L.pcb_det_nms(p, p, p, None, 5, 1, 16, 3, 0, 0.25, p, None),
               L.pcb_det_nms(None, p, p, None, 5, 1, 16, 0, 0, 0.25, p, None)):
        assert rc == 2 and b"bad argument" in L.pcb_last_error()


def test_det_ap_rejects_bad_arguments():
    L = _lib()
    D, G, C, T = 100, 20, 18, 2
    q = L.pcb_det_ap_ws_bytes(D, G, C, T)
    assert q > 0 and L.pcb_det_ap_ws_bytes(0, G, C, T) == 0
    ws = torch.empty(q, dtype=torch.uint8)
    f = torch.zeros(64)
    p = f.data_ptr()
    thr = torch.tensor([0.25, 0.5], dtype=torch.float64)

    def call(D=D, G=G, C=C, T=T, b=q, t=thr.data_ptr(), prop=p):
        return L.pcb_det_ap(prop, 4, p, p, p, p, D, p, p, p, G, C, t, T, p, ws.data_ptr(), b, None)
    for rc in (call(D=0), call(G=0), call(C=0), call(C=1025), call(T=0), call(T=65), call(b=q - 1), call(t=None), call(prop=None)):
        assert rc == 2 and b"bad argument" in L.pcb_last_error()
