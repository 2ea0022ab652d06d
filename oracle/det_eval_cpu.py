"""numpy restatement of VoteNet's detection evaluation (`downstream/votenet_det_new/models/ap_helper.py`, `lib/utils/nms.py`,
`lib/utils/eval_det.py`, `lib/utils/box_util.py`), the oracle of pointcontrast_b200/det_eval.py and csrc/det_eval.cu.

It follows the reference line by line, with three deliberate choices (DESIGN.md section 5):
  * corners are built with one rounding per operation, not with np.dot (whose BLAS may fuse or reorder);
  * ties sort stably: AP in accumulation order, NMS larger proposal index first (numpy's default argsort is not stable);
  * a clip with fewer than 3 non-collinear vertices has area 0 (Qhull raises there).
Softmax exponentials are fp64 `exp` rounded to fp32, as the kernel computes them (numpy's fp32 `np.exp` is within 2 ulp of that).
"""
import math

import numpy as np


# ------------------------------------------------------------------------------------------------ decoding (ap_helper.py:18-38, 57-83)
def softmax(x):
    """ap_helper.py:33-38 in fp32: exp(x - max) (fp64 exp rounded to fp32), divided by numpy's row sum."""
    x = np.asarray(x, np.float32)
    e = np.exp((x - np.max(x, axis=-1, keepdims=True)).astype(np.float64)).astype(np.float32)
    return e / np.sum(e, axis=-1, keepdims=True)


def argmax_first(x):
    """torch.argmax: first maximal index, NaN maximal (np.argmax's rule too)."""
    return np.argmax(np.asarray(x), -1)


def class2angle(rule, cls, residual, H):
    """model_util_scannet.py:45-49 (rule 0), model_util_sunrgbd.py:67-74 (rule 1)."""
    if rule == 0:
        return 0.0
    a = float(cls) * (2 * np.pi / float(H)) + float(residual)
    return a - 2 * np.pi if a > np.pi else a


def get_3d_box(box_size, heading_angle, center):
    """box_util.py:210-225: rows of roty(angle) times the corner table, one rounding per operation."""
    c, s = math.cos(heading_angle), math.sin(heading_angle)
    l, w, h = (float(v) for v in box_size)
    xs = [l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2]
    ys = [h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2]
    zs = [w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2]
    out = np.empty((8, 3))
    for k in range(8):
        out[k, 0] = ((c * xs[k] + 0.0 * ys[k]) + s * zs[k]) + float(center[0])
        out[k, 1] = ((0.0 * xs[k] + 1.0 * ys[k]) + 0.0 * zs[k]) + float(center[1])
        out[k, 2] = ((-s * xs[k] + 0.0 * ys[k]) + c * zs[k]) + float(center[2])
    return out


def flip_axis_to_camera(pc):
    """ap_helper.py:18-25: (x, y, z) -> (x, -z, y)."""
    pc = np.asarray(pc)
    return np.stack([pc[..., 0], -pc[..., 2], pc[..., 1]], -1)


def decode_pred(ep, mean_size, rule):
    """ap_helper.py:57-83 plus the softmaxes of lines 67 and 103: corners [B,K,8,3], params [B,K,7] (center cam, l, w, h, angle),
    sem_cls [B,K], obj_prob fp32 [B,K], sem_prob fp32 [B,K,C]."""
    center = np.asarray(ep["center"], np.float32)
    B, K = center.shape[:2]
    hc = argmax_first(ep["heading_scores"])
    sc = argmax_first(ep["size_scores"])
    H = ep["heading_scores"].shape[-1]
    hr = np.take_along_axis(np.asarray(ep["heading_residuals"], np.float32), hc[..., None], 2)[..., 0]
    sr = np.take_along_axis(np.asarray(ep["size_residuals"], np.float32), sc[..., None, None].repeat(3, -1), 2)[:, :, 0]
    cam = flip_axis_to_camera(center)
    corners, params = np.zeros((B, K, 8, 3)), np.zeros((B, K, 7))
    for i in range(B):
        for j in range(K):
            a = class2angle(rule, hc[i, j], hr[i, j], H)
            size = mean_size[sc[i, j]] + sr[i, j].astype(np.float64)
            corners[i, j] = get_3d_box(size, a, cam[i, j])
            params[i, j] = [*cam[i, j], *size, a]
    return corners, params, argmax_first(ep["sem_cls_scores"]), softmax(ep["objectness_scores"])[..., 1], softmax(ep["sem_cls_scores"])


def decode_gt(ep, mean_size, rule, H):
    """ap_helper.py:196-221: corners [B,K2,8,3] of every slot, and the (cls, corners) lists of the slots with box_label_mask == 1."""
    center = np.asarray(ep["center_label"], np.float32)[:, :, 0:3]
    B, K = center.shape[:2]
    cam = flip_axis_to_camera(center)
    corners = np.zeros((B, K, 8, 3))
    hr = np.asarray(ep["heading_residual_label"], np.float32)
    sr = np.asarray(ep["size_residual_label"], np.float32)
    for i in range(B):
        for j in range(K):
            a = class2angle(rule, ep["heading_class_label"][i, j], hr[i, j], H)
            corners[i, j] = get_3d_box(mean_size[int(ep["size_class_label"][i, j])] + sr[i, j].astype(np.float64), a, cam[i, j])
    mask = np.asarray(ep["box_label_mask"])
    lists = [[(int(ep["sem_cls_label"][i, j]), corners[i, j]) for j in range(K) if mask[i, j] == 1] for i in range(B)]
    return corners, lists


def points_in_box(pc, params):
    """extract_pc_in_box3d (sunrgbd_utils.py:214-223) on one box: points of pc [N, 3] (depth) within the box, as the kernel tests it
    (local coordinates in fp64, |.| <= half size)."""
    cx, cy, cz, l, w, h, a = params
    c, s = math.cos(a), math.sin(a)
    p = np.asarray(pc, np.float32).astype(np.float64)
    dx, dy, dz = p[:, 0] - cx, -p[:, 2] - cy, p[:, 1] - cz
    lx, lz = c * dx - s * dz, s * dx + c * dz
    return int(np.count_nonzero((np.abs(lx) <= abs(l) / 2) & (np.abs(dy) <= abs(h) / 2) & (np.abs(lz) <= abs(w) / 2)))


# ------------------------------------------------------------------------------------------------ NMS (nms.py:44-155)
def nms(boxes, score, mode, thresh, old_type, cls=None):
    """nms_2d_faster (mode 0, boxes [n, 4] = x1, y1, x2, y2), nms_3d_faster (1) and nms_3d_faster_samecls (2, boxes [n, 6]); returns
    the picked indices.  Order: ascending score, ties by index, picked from the end (a stable argsort)."""
    boxes = np.asarray(boxes, np.float64)
    score = np.asarray(score, np.float64)
    d = 2 if mode == 0 else 3
    lo, hi = boxes[:, :d], boxes[:, d:]
    area = (hi[:, 0] - lo[:, 0]) * (hi[:, 1] - lo[:, 1])
    if d == 3:
        area = area * (hi[:, 2] - lo[:, 2])
    I = np.lexsort((np.arange(len(score)), score))
    pick = []
    with np.errstate(invalid="ignore", divide="ignore"):
        while I.size:
            i = I[-1]
            pick.append(i)
            r = I[:-1]
            ext = [np.maximum(0, np.minimum(hi[i, k], hi[r, k]) - np.maximum(lo[i, k], lo[r, k])) for k in range(d)]
            inter = ext[0] * ext[1] if d == 2 else (ext[0] * ext[1]) * ext[2]
            o = inter / area[r] if old_type else inter / (area[i] + area[r] - inter)
            if mode == 2:
                o = o * (cls[i] == cls[r])
            I = np.delete(I, np.concatenate(([I.size - 1], np.where(o > thresh)[0])))
    return pick


def nms_boxes(corners, mode):
    c = np.asarray(corners)
    if mode == 0:
        return np.stack([c[:, :, 0].min(1), c[:, :, 2].min(1), c[:, :, 0].max(1), c[:, :, 2].max(1)], 1)
    return np.concatenate([c.min(1), c.max(1)], 1)


# ------------------------------------------------------------------------------------------------ oriented IoU (box_util.py:16-117)
def polygon_clip(subject, clip):
    """box_util.py:16-62, verbatim in arithmetic."""
    def inside(p):
        return (cp2[0] - cp1[0]) * (p[1] - cp1[1]) > (cp2[1] - cp1[1]) * (p[0] - cp1[0])

    def isect():
        dc = [cp1[0] - cp2[0], cp1[1] - cp2[1]]
        dp = [s[0] - e[0], s[1] - e[1]]
        n1 = cp1[0] * cp2[1] - cp1[1] * cp2[0]
        n2 = s[0] * e[1] - s[1] * e[0]
        den = dc[0] * dp[1] - dc[1] * dp[0]
        n3 = 1.0 / den if den != 0 else math.copysign(math.inf, den)
        return [(n1 * dp[0] - n2 * dc[0]) * n3, (n1 * dp[1] - n2 * dc[1]) * n3]

    out = subject
    cp1 = clip[-1]
    for cp2 in clip:
        inp, out = out, []
        s = inp[-1]
        for e in inp:
            if inside(e):
                if not inside(s):
                    out.append(isect())
                out.append(e)
            elif inside(s):
                out.append(isect())
            s = e
        cp1 = cp2
        if not out:
            return None
    return out


def hull_area(pts):
    """ConvexHull(pts).volume: monotone chain, shoelace; fewer than 3 non-collinear points -> 0."""
    p = sorted((float(x), float(y)) for x, y in pts)

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    h = []
    for q in p:
        while len(h) >= 2 and cross(h[-2], h[-1], q) <= 0:
            h.pop()
        h.append(q)
    t = len(h) + 1
    for q in reversed(p[:-1]):
        while len(h) >= t and cross(h[-2], h[-1], q) <= 0:
            h.pop()
        h.append(q)
    h = h[:-1]
    if len(h) < 3:
        return 0.0
    a = 0.0
    for i in range(len(h)):
        u, v = h[i], h[(i + 1) % len(h)]
        a += u[0] * v[1] - u[1] * v[0]
    return abs(a) / 2


def box3d_vol(c):
    def ln(i, j):
        d = [float(c[i, k]) - float(c[j, k]) for k in range(3)]
        return math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    return (ln(0, 1) * ln(1, 2)) * ln(0, 4)


def box3d_iou(c1, c2):
    """box_util.py:92-117, the 3-D IoU."""
    r1 = [(float(c1[i, 0]), float(c1[i, 2])) for i in range(3, -1, -1)]
    r2 = [(float(c2[i, 0]), float(c2[i, 2])) for i in range(3, -1, -1)]
    inter = polygon_clip(r1, r2)
    inter_area = hull_area(inter) if inter is not None else 0.0
    ymax = min(float(c1[0, 1]), float(c2[0, 1]))
    ymin = max(float(c1[4, 1]), float(c2[4, 1]))
    inter_vol = inter_area * max(0.0, ymax - ymin)
    den = box3d_vol(c1) + box3d_vol(c2) - inter_vol
    return inter_vol / den if den != 0 else (math.nan if inter_vol == 0 else math.copysign(math.inf, inter_vol))


# ------------------------------------------------------------------------------------------------ AP (eval_det.py:24-55, 77-161, 210-256)
def eval_class(dets, gts, thresh):
    """eval_det_cls for one class: dets = [(scan, corners, score)] in accumulation order, gts = {scan: [corners]}.  Returns (rec, ap)
    with the stable descending sort."""
    npos = sum(len(v) for v in gts.values())
    order = sorted(range(len(dets)), key=lambda d: -float(dets[d][2]))          # Python's sort is stable
    used = {s: [False] * len(v) for s, v in gts.items()}
    tp = np.zeros(len(dets))
    for r, d in enumerate(order):
        scan, bb, _ = dets[d]
        ovmax, jmax = -np.inf, -1
        for j, g in enumerate(gts.get(scan, [])):
            iou = box3d_iou(bb, g)
            if iou > ovmax:
                ovmax, jmax = iou, j
        if ovmax > thresh and not used[scan][jmax]:
            tp[r], used[scan][jmax] = 1, True
    fp = np.cumsum(1 - tp)
    tp = np.cumsum(tp)
    with np.errstate(invalid="ignore", divide="ignore"):
        rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    mrec = np.concatenate(([0.0], rec, [1.0]))
    mpre = np.concatenate(([0.0], prec, [0.0]))
    for i in range(mpre.size - 1, 0, -1):
        mpre[i - 1] = max(mpre[i - 1], mpre[i])
    i = np.where(mrec[1:] != mrec[:-1])[0]
    with np.errstate(invalid="ignore"):
        ap = float(np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1]))
    return rec, ap


def eval_det(pred_all, gt_all, thresh):
    """eval_det_multiprocessing: pred_all / gt_all = lists (one per scan) of (cls, corners, score) / (cls, corners).  Returns
    {cls: (ap, recall, npos, ndet)}."""
    pred, gt = {}, {}
    for scan, lst in enumerate(pred_all):
        for c, bb, s in lst:
            pred.setdefault(c, []).append((scan, bb, s))
            gt.setdefault(c, {})
    for scan, lst in enumerate(gt_all):
        for c, bb in lst:
            gt.setdefault(c, {}).setdefault(scan, []).append(bb)
    out = {}
    for c in gt:
        npos = sum(len(v) for v in gt[c].values())
        if c in pred:
            rec, ap = eval_class(pred[c], gt[c], thresh)
            out[c] = (ap, rec[-1], npos, len(pred[c]))
        else:
            out[c] = (0.0, 0.0, npos, 0)
    return out


def metrics(pred_all, gt_all, thresh, class2type_map=None):
    """APCalculator.compute_metrics (ap_helper.py:252-271)."""
    res = eval_det(pred_all, gt_all, thresh)
    ret = {}
    for c in sorted(res):
        ret["%s Average Precision" % (class2type_map[c] if class2type_map else str(c))] = res[c][0]
    ret["mAP"] = np.mean([res[c][0] for c in sorted(res)])
    for c in sorted(res):
        ret["%s Recall" % (class2type_map[c] if class2type_map else str(c))] = res[c][1]
    ret["AR"] = np.mean([res[c][1] for c in sorted(res)])
    return ret


# ------------------------------------------------------------------------------------------------ parse_predictions (ap_helper.py:40-177)
def parse_predictions(ep, cfg):
    """cfg: the config_dict keys of ap_helper.py plus mean_size (fp64 [S, 3]), rule and num_class.  Returns (pred_mask [B, K], the
    per-scene detection lists, corners)."""
    corners, params, sem_cls, obj_prob, sem_prob = decode_pred(ep, cfg["mean_size"], cfg["rule"])
    B, K = obj_prob.shape
    nonempty = np.ones((B, K), bool)
    if cfg["remove_empty_box"]:
        pc = np.asarray(ep["point_clouds"], np.float32)[:, :, 0:3]
        for i in range(B):
            for j in range(K):
                nonempty[i, j] = points_in_box(pc[i], params[i, j]) >= 5
    mode = 0 if not cfg["use_3d_nms"] else (2 if cfg["cls_nms"] else 1)
    pred_mask = np.zeros((B, K))
    for i in range(B):
        inds = np.where(nonempty[i])[0]
        pick = nms(nms_boxes(corners[i, inds], mode), obj_prob[i, inds], mode, cfg["nms_iou"], cfg["use_old_type_nms"], sem_cls[i, inds])
        assert len(pick) > 0
        pred_mask[i, inds[pick]] = 1
    lists = []
    thr = np.float32(cfg["conf_thresh"])
    for i in range(B):
        keep = [j for j in range(K) if pred_mask[i, j] == 1 and obj_prob[i, j] > thr]
        if cfg["per_class_proposal"]:
            lists.append([(c, corners[i, j], sem_prob[i, j, c] * obj_prob[i, j]) for c in range(cfg["num_class"]) for j in keep])
        else:
            lists.append([(int(sem_cls[i, j]), corners[i, j], obj_prob[i, j]) for j in keep])
    return pred_mask, lists, corners
