"""Writes tests/golden/detection_eval.npz from the original VoteNet evaluation code, run unmodified:

    python tests/golden/make_detection_eval_golden.py <root>      (<root>: the original repository)

Loads `models/ap_helper.py` (with `lib/utils/{nms,eval_det,box_util}.py`) and the ScanNet / SUN RGB-D model-util configs by path, with
stubs for the modules they import but this path never uses (plyfile, trimesh, matplotlib, cv2).  Inputs are seeded `end_points` of two
small scenes per dataset; for the four `config_dict` variants of lib/test.py (2-D NMS, empty-box removal) and lib/train.py (3-D
per-class NMS, per-class proposals), each with and without old_type NMS, it records pred_mask, the flattened detection and
ground-truth lists and compute_metrics at IoU 0.25 and 0.5.  It also records `box3d_iou` on rotated, mirrored, nested, disjoint and
near-threshold pairs.  It asserts that its data has no exact score ties and no Qhull-degenerate overlap.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "detection_eval.npz")
VARIANTS = [  # (name, config_dict without dataset_config)
    ("test", dict(remove_empty_box=True, use_3d_nms=False, nms_iou=0.25, use_old_type_nms=False, cls_nms=False, per_class_proposal=False,
                  conf_thresh=0.05)),
    ("test_old", dict(remove_empty_box=True, use_3d_nms=False, nms_iou=0.25, use_old_type_nms=True, cls_nms=False,
                      per_class_proposal=False, conf_thresh=0.05)),
    ("train", dict(remove_empty_box=False, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=False, cls_nms=True, per_class_proposal=True,
                   conf_thresh=0.05)),
    ("train_old", dict(remove_empty_box=False, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=True, cls_nms=True,
                       per_class_proposal=True, conf_thresh=0.05)),
]


class _Anything:
    """Stands for any attribute of a stubbed module (`pyplot.cm.jet` in a default argument, PlyData, ...); never called here."""
    def __getattr__(self, attr):
        return self


def _stub_attr(attr):
    if attr.startswith("__"):
        raise AttributeError(attr)
    return _Anything()


def load(root):
    base = os.path.join(root, "downstream", "votenet_det_new")
    for name in ("plyfile", "trimesh", "matplotlib", "matplotlib.pyplot", "cv2"):
        try:
            __import__(name)
        except ImportError:
            stub = types.ModuleType(name)
            stub.__getattr__ = _stub_attr                                    # `from plyfile import PlyData, PlyElement` etc.
            sys.modules[name] = stub
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.path[:0] = [base, os.path.join(base, "lib", "utils")]
    from models import ap_helper
    from lib.utils import box_util
    from lib.datasets.scannet.model_util_scannet import ScannetDatasetConfig
    from lib.datasets.sunrgbd.model_util_sunrgbd import SunrgbdDatasetConfig
    return ap_helper, box_util, ScannetDatasetConfig(), SunrgbdDatasetConfig()


def end_points(cfg, seed, B=2, K=48, K2=12, N=5000):
    """Proposals scattered around the ground-truth boxes of a room; points sampled inside half of the boxes and over the room."""
    g = np.random.default_rng(seed)
    C, H, S = cfg.num_class, cfg.num_heading_bin, cfg.num_size_cluster
    ms = np.asarray(cfg.mean_size_arr)
    ep = {}
    sc_l = g.integers(0, S, (B, K2))
    ep["center_label"] = np.concatenate([g.uniform(-3, 3, (B, K2, 2)), g.uniform(0.3, 1.5, (B, K2, 1))], -1).astype(np.float32)
    ep["heading_class_label"] = g.integers(0, H, (B, K2))
    ep["heading_residual_label"] = g.uniform(-0.2, 0.2, (B, K2)).astype(np.float32) * (H > 1)
    ep["size_class_label"] = sc_l
    ep["size_residual_label"] = (g.uniform(-0.15, 0.15, (B, K2, 3)) * ms[sc_l]).astype(np.float32)
    ep["sem_cls_label"] = sc_l.copy()
    ep["box_label_mask"] = (g.random((B, K2)) < 0.85).astype(np.float32)
    src = g.integers(0, K2, (B, K))
    jit = g.normal(0, 0.15, (B, K, 3))
    ep["center"] = (np.take_along_axis(ep["center_label"], src[..., None].repeat(3, -1), 1) + jit).astype(np.float32)
    ep["heading_scores"] = g.normal(0, 2, (B, K, H)).astype(np.float32)
    ep["heading_residuals"] = g.uniform(-0.3, 0.3, (B, K, H)).astype(np.float32)
    ss = g.normal(0, 1, (B, K, S))
    np.put_along_axis(ss, np.take_along_axis(sc_l, src, 1)[..., None], 4.0, -1)
    ep["size_scores"] = ss.astype(np.float32)
    sr = g.uniform(-0.25, 0.25, (B, K, S, 3)) * ms[None, None]
    sr[g.random((B, K)) < 0.05, :, 0] -= 3 * ms.max()                       # mirrored boxes: a negative length after the residual
    ep["size_residuals"] = sr.astype(np.float32)
    cls = g.normal(0, 1.5, (B, K, C))
    ep["sem_cls_scores"] = cls.astype(np.float32)
    ep["objectness_scores"] = g.normal(0, 2, (B, K, 2)).astype(np.float32)
    room = g.uniform([-3.5, -3.5, 0], [3.5, 3.5, 2], (B, N // 2, 3))
    near = ep["center_label"][:, g.integers(0, K2, N - N // 2)] + g.normal(0, 0.3, (B, N - N // 2, 3))
    ep["point_clouds"] = np.concatenate([room, near], 1).astype(np.float32)
    return ep


def to_torch(ep):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in ep.items()}


def iou_pairs(box_util, seed):
    g = np.random.default_rng(seed)
    pairs = []
    def box(c, size, a):
        return box_util.get_3d_box(size, a, c)
    for _ in range(40):                                                      # rotated, overlapping
        c = g.uniform(-1, 1, 3)
        pairs.append((box(c, g.uniform(0.5, 2, 3), g.uniform(-np.pi, np.pi)), box(c + g.normal(0, 0.3, 3), g.uniform(0.5, 2, 3),
                                                                                    g.uniform(-np.pi, np.pi))))
    for _ in range(8):                                                       # mirrored (negative sizes)
        c = g.uniform(-1, 1, 3)
        s = g.uniform(0.5, 2, 3) * g.choice([-1, 1], 3)
        pairs.append((box(c, s, g.uniform(-np.pi, np.pi)), box(c + g.normal(0, 0.2, 3), g.uniform(0.5, 2, 3), g.uniform(-np.pi, np.pi))))
    pairs.append((box(np.zeros(3), [2, 2, 2], 0.3), box(np.zeros(3), [1, 1, 1], 0.7)))          # nested
    pairs.append((box(np.zeros(3), [1, 1, 1], 0.0), box(np.array([5.0, 0, 0]), [1, 1, 1], 0.2)))  # disjoint
    pairs.append((box(np.zeros(3), [1, 1, 1], 0.0), box(np.array([0.5, 0.0, 0.1]), [1, 1, 1], 0.0)))
    pairs.append((box(np.zeros(3), [1, 1, 1], 0.0), box(np.array([0.0, 0.0, 0.6]), [1, 1, 1], 0.0)))  # IoU 0.25
    return np.array(pairs)


def main(root):
    ap_helper, box_util, scannet, sunrgbd = load(root)
    rec = {}
    for dname, cfg, seed in (("scannet", scannet, 1), ("sunrgbd", sunrgbd, 2)):
        ep = end_points(cfg, seed)
        for k, v in ep.items():
            rec[f"{dname}/in/{k}"] = v
        rec[f"{dname}/mean_size"] = np.asarray(cfg.mean_size_arr, np.float64)
        rec[f"{dname}/class_names"] = np.array([cfg.class2type[c] for c in range(cfg.num_class)])
        for vname, v in VARIANTS:
            cd = dict(v, dataset_config=cfg)
            e = to_torch(ep)
            preds = ap_helper.parse_predictions(e, cd)
            gts = ap_helper.parse_groundtruths(e, cd)
            key = f"{dname}/{vname}"
            rec[key + "/pred_mask"] = np.asarray(e["pred_mask"])
            rec[key + "/pred"] = np.array([(i, c, float(s)) for i, lst in enumerate(preds) for c, _, s in lst]).reshape(-1, 3)
            rec[key + "/pred_corners"] = np.array([b for lst in preds for _, b, _ in lst]).reshape(-1, 8, 3)
            rec[key + "/gt"] = np.array([(i, c) for i, lst in enumerate(gts) for c, _ in lst]).reshape(-1, 2)
            rec[key + "/gt_corners"] = np.array([b for lst in gts for _, b in lst]).reshape(-1, 8, 3)
            for i, lst in enumerate(preds):
                per = {}
                for c, _, s in lst:
                    per.setdefault(c, []).append(s)
                for c, s in per.items():
                    assert len(set(np.float32(s).tolist())) == len(s), f"{key}: exact score tie in scene {i} class {c}"
            for thr in (0.25, 0.5):
                calc = ap_helper.APCalculator(thr, cfg.class2type)
                calc.step(preds, gts)
                m = calc.compute_metrics()
                rec[f"{key}/metrics_{thr}/keys"] = np.array(list(m.keys()))
                rec[f"{key}/metrics_{thr}/values"] = np.array([float(x) for x in m.values()])
    pairs = iou_pairs(box_util, 3)
    rec["iou/pairs"] = pairs
    rec["iou/value"] = np.array([box_util.box3d_iou(a, b)[0] for a, b in pairs])      # raises on a Qhull-degenerate overlap
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
