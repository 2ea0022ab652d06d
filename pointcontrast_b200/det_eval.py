"""VoteNet detection evaluation on the GPU, behind the interface of the original's `models/ap_helper.py`.

    parse_predictions(end_points, config_dict)     proposal decoding, empty-box removal, NMS (csrc/det_eval.cu)
    parse_groundtruths(end_points, config_dict)    label decoding with the same box routine
    APCalculator(ap_iou_thresh, class2type_map)    VOC average precision of the accumulated batches, one kernel pass per call
    DetectionMetrics(thresholds, config_dict, ...)  the same evaluation with no per-batch host read at all
    install()                                      registers this module as `models.ap_helper`

After `install()`, VoteNet's unmodified `lib/test.py::test` and `lib/train.py::evaluate_one_epoch` run this evaluation.  The numerics
(fp32 scores, fp64 corners and IoU, the tie order, degenerate clips) are stated in DESIGN.md section 5.
"""
import ctypes
import importlib
import sys
import types

import numpy as np
import torch

from ._lib import PcbError, check, lib, ptr, require_cuda, stream, workspace

NMS_MODES = {"2d": 0, "3d": 1, "3d_samecls": 2}
MIN_POINTS = 5                                          # ap_helper.py:98: a box with fewer points is empty


def heading_rule(dataset_config):
    """0 when `class2angle` always returns 0 (ScanNet), 1 when it is cls * 2 pi / H + residual wrapped above pi (SUN RGB-D).  Probed
    on the host; any other config raises."""
    H = int(dataset_config.num_heading_bin)
    probes = [(0, 0.0), (1 % H, 0.25), (H - 1, 0.5), (H // 2, -0.125)]
    got = [float(dataset_config.class2angle(np.array(c), np.float32(r))) for c, r in probes]
    if all(g == 0.0 for g in got):
        return 0
    want = []
    for c, r in probes:
        a = c * (2 * np.pi / float(H)) + float(np.float32(r))
        want.append(a - 2 * np.pi if a > np.pi else a)
    if all(abs(g - w) <= 1e-12 for g, w in zip(got, want)):
        return 1
    raise PcbError("det_eval: dataset_config.class2angle matches neither the ScanNet nor the SUN RGB-D heading rule")


def _mean_size(dataset_config, device):
    return torch.as_tensor(np.asarray(dataset_config.mean_size_arr, np.float64), device=device).contiguous()


def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def decode_predictions(end_points, dataset_config):
    """Device tensors of every proposal: corners fp64 [B,K,8,3], box params fp64 [B,K,8], sem_cls int32 [B,K], obj_prob fp32 [B,K],
    sem_prob fp32 [B,K,C]."""
    center = _f32(end_points["center"])
    require_cuda(center)
    B, K = center.shape[:2]
    hs, hr = _f32(end_points["heading_scores"]), _f32(end_points["heading_residuals"])
    ss, sr = _f32(end_points["size_scores"]), _f32(end_points["size_residuals"])
    cs, obj = _f32(end_points["sem_cls_scores"]), _f32(end_points["objectness_scores"])
    H, S, C = hs.shape[-1], ss.shape[-1], cs.shape[-1]
    dev = center.device
    corners = torch.empty(B, K, 8, 3, dtype=torch.float64, device=dev)
    box = torch.empty(B, K, 8, dtype=torch.float64, device=dev)
    sem_cls = torch.empty(B, K, dtype=torch.int32, device=dev)
    obj_prob = torch.empty(B, K, dtype=torch.float32, device=dev)
    sem_prob = torch.empty(B, K, C, dtype=torch.float32, device=dev)
    check(lib.pcb_det_decode_pred(ptr(center), ptr(hs), ptr(hr), ptr(ss), ptr(sr), ptr(cs), ptr(obj), B, K, H, S, C,
                                  ptr(_mean_size(dataset_config, dev)), heading_rule(dataset_config), ptr(corners), ptr(box), ptr(sem_cls),
                                  ptr(obj_prob), ptr(sem_prob), stream()))
    return corners, box, sem_cls, obj_prob, sem_prob


def decode_groundtruths(end_points, dataset_config):
    """Corners fp64 [B,K2,8,3] of every label slot, and the device int32 status of pcb_det_decode_gt.  Slots that box_label_mask drops
    are decoded with class 0 (the reference skips them, so whatever they hold is never out of range); a kept slot with a size or
    heading class out of range sets status to PCB_ERR_RANGE and keeps zero corners."""
    center = _f32(end_points["center_label"][:, :, 0:3])
    require_cuda(center)
    B, K = center.shape[:2]
    dev = center.device
    keep = end_points["box_label_mask"] == 1
    hc = torch.where(keep, end_points["heading_class_label"].to(torch.int64), 0).contiguous()
    hr = _f32(end_points["heading_residual_label"])
    sc = torch.where(keep, end_points["size_class_label"].to(torch.int64), 0).contiguous()
    sr = _f32(end_points["size_residual_label"])
    corners = torch.zeros(B, K, 8, 3, dtype=torch.float64, device=dev)
    box = torch.zeros(B, K, 8, dtype=torch.float64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.pcb_det_decode_gt(ptr(center), ptr(hc), ptr(hr), ptr(sc), ptr(sr), B, K, int(dataset_config.num_heading_bin),
                                int(np.asarray(dataset_config.mean_size_arr).shape[0]), ptr(_mean_size(dataset_config, dev)),
                                heading_rule(dataset_config), ptr(corners), ptr(box), ptr(status), stream()))
    return corners, status


def points_in_boxes(points, box):
    """int32 [B, K]: points of points [B, N, >=3] inside each box of box params [B, K, 8]."""
    points = _f32(points)
    require_cuda(points)
    B, N, ld = points.shape
    K = box.shape[1]
    counts = torch.empty(B, K, dtype=torch.int32, device=points.device)
    check(lib.pcb_det_points_in_box(ptr(points), B, N, ld, ptr(box.contiguous()), K, ptr(counts), stream()))
    return counts


def nms(corners, score, sem_cls, counts, mode, old_type, nms_iou):
    """int32 [B, K] keep mask; candidates are the proposals with counts >= 5 (all when counts is None)."""
    B, K = score.shape
    mask = torch.empty(B, K, dtype=torch.int32, device=score.device)
    check(lib.pcb_det_nms(ptr(corners), ptr(score), ptr(sem_cls), ptr(counts), MIN_POINTS, B, K, NMS_MODES[mode], int(bool(old_type)),
                          float(nms_iou), ptr(mask), stream()))
    return mask


def _nms_mode(config_dict):
    if not config_dict["use_3d_nms"]:
        return "2d"
    return "3d_samecls" if config_dict["cls_nms"] else "3d"


class BatchPredictions:
    """parse_predictions' result, kept on the device.  len() is the batch size; [i] builds the reference's list of
    (cls, corners (8, 3), score) tuples of scene i on demand."""

    def __init__(self, corners, sem_cls, obj_prob, sem_prob, mask, conf_thresh, per_class):
        self.corners, self.sem_cls, self.obj_prob, self.sem_prob, self.mask = corners, sem_cls, obj_prob, sem_prob, mask
        self.conf_thresh, self.per_class = float(conf_thresh), bool(per_class)

    def __len__(self):
        return self.corners.shape[0]

    def detections(self):
        """(row, cls, score) int32 / int32 / fp32 device tensors over every slot of the batch, in the reference's list order per scene,
        scene-major; cls -1 marks a slot that is not a detection.  Per-class: slots [B, C, K] with score sem_prob * obj_prob (fp32);
        else [B, K] with the argmax class and obj_prob.  The `obj_prob > conf_thresh` test runs in fp32, as numpy compares them."""
        B, K = self.obj_prob.shape
        keep = (self.mask == 1) & (self.obj_prob > torch.tensor(self.conf_thresh, dtype=torch.float32))
        rows = torch.arange(B * K, dtype=torch.int32, device=self.mask.device).view(B, K)
        if self.per_class:
            C = self.sem_prob.shape[-1]
            score = (self.sem_prob * self.obj_prob.unsqueeze(-1)).transpose(1, 2)                # [B, C, K], fp32 product
            cls = torch.arange(C, dtype=torch.int32, device=rows.device).view(1, C, 1).expand(B, C, K)
            cls = torch.where(keep.unsqueeze(1), cls, -1)
            rows = rows.unsqueeze(1).expand(B, C, K)
        else:
            score, cls = self.obj_prob, torch.where(keep, self.sem_cls, -1)
        return rows.reshape(-1).contiguous(), cls.reshape(-1).contiguous(), score.reshape(-1).contiguous()

    def __getitem__(self, i):
        rows, cls, score = (t.view(len(self), -1)[i].cpu().numpy() for t in self.detections())
        corners = self.corners.view(-1, 8, 3).cpu().numpy()
        return [(int(c), corners[r], np.float32(s)) for r, c, s in zip(rows, cls, score) if c >= 0]


def _check_status(status):
    if int(status) != 0:
        raise PcbError("det_eval: a ground-truth box has a size or heading class outside the dataset config's range")


class BatchGroundTruths:
    """parse_groundtruths' result on the device; [i] builds the reference's list of (cls, corners) tuples of scene i.  status: the
    decode status (device int32), checked wherever the labels are read on the host."""

    def __init__(self, corners, cls, status):
        self.corners, self.cls, self.status = corners, cls, status

    def __len__(self):
        return self.corners.shape[0]

    def __getitem__(self, i):
        _check_status(self.status)
        c = self.cls[i].cpu().numpy()
        k = self.corners[i].cpu().numpy()
        return [(int(c[j]), k[j]) for j in range(len(c)) if c[j] >= 0]


def _predict(end_points, config_dict):
    cfg = config_dict["dataset_config"]
    corners, box, sem_cls, obj_prob, sem_prob = decode_predictions(end_points, cfg)
    counts = points_in_boxes(end_points["point_clouds"], box) if config_dict["remove_empty_box"] else None
    mask = nms(corners, obj_prob, sem_cls, counts, _nms_mode(config_dict), config_dict["use_old_type_nms"], config_dict["nms_iou"])
    return BatchPredictions(corners, sem_cls, obj_prob, sem_prob, mask, config_dict["conf_thresh"], config_dict["per_class_proposal"])


def parse_predictions(end_points, config_dict):
    """`ap_helper.py:40-177` on the device.  Sets end_points['pred_mask'] (numpy fp64 [B, K], the one host read) and
    end_points['batch_pred_map_cls'], and returns the BatchPredictions."""
    pred = _predict(end_points, config_dict)
    pred_mask = pred.mask.cpu().numpy().astype(np.float64)
    assert (pred_mask.sum(1) > 0).all()                 # ap_helper.py:118: assert(len(pick)>0) per scene
    end_points["pred_mask"] = pred_mask
    end_points["batch_pred_map_cls"] = pred
    return pred


def _gt(end_points, config_dict):
    corners, status = decode_groundtruths(end_points, config_dict["dataset_config"])
    valid = end_points["box_label_mask"] == 1
    cls = torch.where(valid, end_points["sem_cls_label"].to(torch.int32), -1).contiguous()
    return BatchGroundTruths(corners, cls, status)


def parse_groundtruths(end_points, config_dict):
    """`ap_helper.py:179-221` on the device; sets end_points['batch_gt_map_cls'] and returns the BatchGroundTruths."""
    gt = _gt(end_points, config_dict)
    end_points["batch_gt_map_cls"] = gt
    return gt


def _from_lists(batch_pred, batch_gt, device):
    """The reference's plain lists as one device batch: predictions as their own proposals (one row per tuple)."""
    B = len(batch_pred)
    rows, cls, score, corners = [], [], [], []
    for i in range(B):
        for c, bb, s in batch_pred[i]:
            rows.append(len(corners))
            corners.append(np.asarray(bb, np.float64))
            cls.append(int(c))
            score.append(np.float32(s))
    K2 = max([len(g) for g in batch_gt] + [1])
    gc = np.zeros((B, K2, 8, 3))
    gcls = np.full((B, K2), -1, np.int32)
    for i in range(B):
        for j, (c, bb) in enumerate(batch_gt[i]):
            gc[i, j], gcls[i, j] = bb, int(c)
    n = [len(p) for p in batch_pred]
    t = lambda a, dt: torch.as_tensor(np.asarray(a, dt), device=device)
    pc = t(np.stack(corners) if corners else np.zeros((1, 8, 3)), np.float64)
    return (pc, t(rows, np.int32), t(cls, np.int32), t(score, np.float32), t(np.repeat(np.arange(B), n), np.int32),
            t(gc, np.float64), t(gcls, np.int32))


class _Accumulator:
    """Device tensors of every batch stepped so far; compute() runs pcb_det_ap once over all of them."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.parts = []
        self.scan_cnt = 0
        self.rows = 0
        self.max_cls = -1
        self.status = []

    def add(self, prop_corners, det_row, det_cls, det_score, det_scan, gt_corners, gt_cls, num_class=None, status=None):
        B = gt_corners.shape[0]
        if status is not None:
            self.status.append(status.view(1))
        self.parts.append((prop_corners.reshape(-1, 8, 3), det_row + self.rows, det_cls, det_score, det_scan + self.scan_cnt,
                           gt_corners.reshape(-1, 8, 3), gt_cls.reshape(-1),
                           (torch.arange(B, dtype=torch.int32, device=gt_cls.device) + self.scan_cnt).repeat_interleave(gt_cls.shape[1])))
        self.rows += prop_corners.reshape(-1, 8, 3).shape[0]
        self.scan_cnt += B
        if num_class is not None:
            self.max_cls = max(self.max_cls, int(num_class) - 1)

    def compute(self, thresholds, num_class=None):
        """fp64 numpy [T, C, 4] = (AP, recall, npos, ndet) per threshold and class.  Raises when a stepped batch had a ground-truth
        label out of range (read with the results, in the same copy)."""
        if not self.parts:
            raise PcbError("det_eval: nothing accumulated")
        cat = [torch.cat([p[k] for p in self.parts]).contiguous() for k in range(8)]
        prop, row, cls, score, scan, gtc, gcls, gscan = cat
        C = num_class if num_class is not None else self.max_cls + 1
        if C < 1:
            raise PcbError("det_eval: no class seen")
        dev = prop.device
        if cls.numel() == 0:                              # no slot at all: one that is not a detection
            row, cls, score, scan = (torch.zeros(1, dtype=d, device=dev) for d in (torch.int32, torch.int32, torch.float32, torch.int32))
            cls -= 1
        if gcls.numel() == 0:
            gtc, gcls, gscan = torch.zeros(1, 8, 3, dtype=torch.float64, device=dev), torch.full((1,), -1, dtype=torch.int32, device=dev), \
                torch.zeros(1, dtype=torch.int32, device=dev)
        T = len(thresholds)
        D, G, P = cls.numel(), gcls.numel(), prop.shape[0]
        out = torch.empty(T, C, 4, dtype=torch.float64, device=dev)
        wsb = lib.pcb_det_ap_ws_bytes(D, G, C, T)
        ws = workspace(wsb, dev)
        thr = (ctypes.c_double * T)(*[float(x) for x in thresholds])           # host array: the entry point copies it
        check(lib.pcb_det_ap(ptr(prop), P, ptr(row), ptr(cls), ptr(score), ptr(scan), D, ptr(gtc), ptr(gscan), ptr(gcls), G, C,
                             ctypes.addressof(thr), T, ptr(out), ptr(ws), wsb, stream()))
        status = torch.cat(self.status).max().double().view(1) if self.status else torch.zeros(1, dtype=torch.float64, device=dev)
        host = torch.cat([out.view(-1), status]).cpu().numpy()
        _check_status(host[-1])
        return host[:-1].reshape(T, C, 4)


def metrics_dict(res, class2type_map=None):
    """`APCalculator.compute_metrics`' dict from one threshold's [C, 4] rows: the classes that have a detection or a ground-truth box,
    in sorted order."""
    ret, ap, rec = {}, [], []
    present = [c for c in range(res.shape[0]) if res[c, 2] > 0 or res[c, 3] > 0]
    for c in present:
        name = class2type_map[c] if class2type_map else str(c)
        ret["%s Average Precision" % name] = res[c, 0]
        ap.append(res[c, 0])
    ret["mAP"] = np.mean(ap)
    for c in present:
        name = class2type_map[c] if class2type_map else str(c)
        ret["%s Recall" % name] = res[c, 1]
        rec.append(res[c, 1])
    ret["AR"] = np.mean(rec)
    return ret


class APCalculator:
    """`ap_helper.py:223-276`: step() appends a batch (device results of parse_predictions / parse_groundtruths, or the reference's plain
    lists); compute_metrics() returns the reference's dict from one kernel pass and one host read."""

    def __init__(self, ap_iou_thresh=0.25, class2type_map=None):
        self.ap_iou_thresh = ap_iou_thresh
        self.class2type_map = class2type_map
        self.acc = _Accumulator()

    def step(self, batch_pred_map_cls, batch_gt_map_cls):
        assert len(batch_pred_map_cls) == len(batch_gt_map_cls)
        if isinstance(batch_pred_map_cls, BatchPredictions) and isinstance(batch_gt_map_cls, BatchGroundTruths):
            p, g = batch_pred_map_cls, batch_gt_map_cls
            row, cls, score = p.detections()
            scan = torch.div(row.long(), p.corners.shape[1], rounding_mode="floor").to(torch.int32)
            self.acc.add(p.corners, row, cls, score, scan, g.corners, g.cls, p.sem_prob.shape[-1], g.status)
            return
        dev = torch.device("cuda", torch.cuda.current_device())
        pc, row, cls, score, scan, gc, gcls = _from_lists(list(batch_pred_map_cls[i] for i in range(len(batch_pred_map_cls))),
                                                          list(batch_gt_map_cls[i] for i in range(len(batch_gt_map_cls))), dev)
        seen = [int(x) for x in cls.tolist()] + [int(x) for x in gcls.flatten().tolist() if x >= 0]
        if any(c < 0 for c in seen):
            raise PcbError("det_eval: class ids must be non-negative integers")
        self.acc.add(pc, row, cls, score, scan, gc, gcls, (max(seen) + 1) if seen else None)

    def compute_metrics(self):
        return metrics_dict(self.acc.compute([self.ap_iou_thresh])[0], self.class2type_map)

    def reset(self):
        self.acc.reset()


class DetectionMetrics:
    """The evaluation of `lib/test.py` for several IoU thresholds at once, with no host read per batch: update() decodes, removes empty
    boxes, runs NMS and accumulates on the device; result() returns one metrics dict per threshold."""

    def __init__(self, thresholds, config_dict, class2type_map=None):
        self.thresholds = list(thresholds)
        self.config_dict = config_dict
        self.class2type_map = class2type_map
        self.acc = _Accumulator()

    def update(self, end_points):
        p = _predict(end_points, self.config_dict)
        g = _gt(end_points, self.config_dict)
        row, cls, score = p.detections()
        scan = torch.div(row.long(), p.corners.shape[1], rounding_mode="floor").to(torch.int32)
        self.acc.add(p.corners, row, cls, score, scan, g.corners, g.cls, p.sem_prob.shape[-1], g.status)

    def result(self):
        res = self.acc.compute(self.thresholds)
        return [metrics_dict(r, self.class2type_map) for r in res]


def install(name="models.ap_helper"):
    """Register this module as `name` (and as the attribute of its parent package), so that `from models.ap_helper import
    APCalculator, parse_predictions, parse_groundtruths` -- VoteNet's lib/test.py and lib/train.py -- resolves here.  Returns the module."""
    return register(sys.modules[__name__], name)


def register(mod, name):
    """Make `import name` resolve to mod: sys.modules[name], and the attribute of its parent package (created empty when it cannot be
    imported).  Returns mod."""
    parent, _, child = name.rpartition(".")
    if parent:
        try:
            pkg = importlib.import_module(parent)
        except ImportError:
            pkg = types.ModuleType(parent)
            pkg.__path__ = []
            sys.modules[parent] = pkg
        setattr(pkg, child, mod)
    sys.modules[name] = mod
    return mod
