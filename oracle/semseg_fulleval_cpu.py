"""numpy / scipy restatement of semantic segmentation on the original point cloud (`downstream/semseg/lib/utils.py:304-349`
`save_predictions`, `lib/datasets/scannet.py:131-172` and `stanford.py:41-84` `test_pointcloud`), the checker of `pcb_nearest`,
`pcb_label_transfer` and `pointcontrast_b200.semseg.PointCloudEvaluator`.  The decisions it restates (DESIGN.md section 5):

* nearest centre: idx[i] = the smallest j whose d2 = ((dx dx + dy dy) + dz dz) (fp64, each operation rounded once) is minimal over all
  references -- scipy's KD-tree leaves the order of ties unspecified.  `nearest` takes cKDTree candidates within a slightly widened
  radius of its distance and applies that rule to their exact d2; `nearest_brute` scans every reference, in chunks;
* centres: inv(T) @ (c + 0.5, 1) with T the float32 4x4 of the collated transformation and inv its float32 `np.linalg.inv`, the product
  in fp64 (`utils.py:326-330`); coords batch-first, as the collate writes them;
* labels: predictions decoded to original ids through the inverse label map (`utils.py:336-341`); the histogram maps prediction and
  ground truth through the dataset's label map (original -> masked, ignored classes -> 255) and counts rows with 0 <= gt < C
  (`fast_hist`);
* ScanNet: one scene per group, `<scene>.txt` of the per-point original ids (`np.savetxt(fmt='%i')`), a scene without a `label`
  property adds nothing to the histogram;
* S3DIS: the group key is (area, file stem without its last "_" field), so all rooms of one type in an area are searched together;
  the group's query rows [x, y, z, r, g, b, label] are de-duplicated by exact equality (`stanford.py:63`).
"""
import collections
import os

import numpy as np


def d2(ref, q):
    """((dx dx + dy dy) + dz dz) between rows of ref [k, 3] and one point q [3], fp64."""
    d = np.asarray(ref, np.float64) - np.asarray(q, np.float64)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def _pick(cand, dd):
    """The smallest candidate index among those with the minimal d2 (cand ascending or not)."""
    best = dd.min()
    return int(cand[dd == best].min())


def nearest_brute(ref, query, chunk=2048):
    """idx int64 [n]: exact nearest reference by the d2 / smallest-index rule, every reference compared (small cases)."""
    ref, query = np.asarray(ref, np.float64), np.asarray(query, np.float64)
    out = np.empty(len(query), np.int64)
    for a in range(0, len(query), chunk):
        q = query[a:a + chunk]
        d = ref[None, :, :] - q[:, None, :]
        dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]          # [chunk, m]
        out[a:a + chunk] = np.argmin(dd, axis=1)                                             # argmin: the first minimum
    return out


def nearest(ref, query):
    """idx int64 [n], the same rule as `nearest_brute` for any size: cKDTree distance r, then every reference within r (1 + 1e-9) +
    1e-300 is a candidate and the exact d2 decides."""
    from scipy.spatial import cKDTree
    ref, query = np.asarray(ref, np.float64), np.asarray(query, np.float64)
    tree = cKDTree(ref)
    dist, out = tree.query(query)
    out = out.astype(np.int64)
    r = dist * (1 + 1e-9) + 1e-300
    many = np.flatnonzero(tree.query_ball_point(query, r, return_length=True) > 1)      # one candidate: the tree's answer is it
    for i, c in zip(many, tree.query_ball_point(query[many], r[many])):
        c = np.asarray(c, np.int64)
        out[i] = _pick(c, d2(ref[c], query[i]))
    return out


def fast_hist(pred, label, n):
    """`utils.py:131-133`: hist[label, pred] over the rows with 0 <= label < n (int64)."""
    pred, label = np.asarray(pred, np.int64), np.asarray(label, np.int64)
    k = (label >= 0) & (label < n)
    return np.bincount(n * label[k] + pred[k], minlength=n ** 2).reshape(n, n)


def per_class_iu(hist):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))


def label_lut(label_map):
    """The label map {original: masked} as an int64 table, -1 where it has no entry."""
    lut = np.full(max(label_map) + 1, -1, np.int64)
    for k, v in label_map.items():
        lut[k] = v
    return lut


def decode_lut(label_map, C):
    """`utils.py:336-339`: masked prediction -> original id (the last original id mapped to it)."""
    dec = {}
    for k, v in label_map.items():
        dec[v] = k
    return np.array([dec[v] for v in range(C)], np.int64)


def map_labels(lut, x):
    """lut[x]; a label outside the table or without an entry raises (the reference's KeyError / IndexError)."""
    x = np.asarray(x, np.int64)
    if len(x) and (x.min() < 0 or x.max() >= len(lut) or (lut[x] < 0).any()):
        raise KeyError("label outside the dataset's label map")
    return lut[x]


def label_transfer(idx, ref_label, query_label, lut, C):
    """(point_label = ref_label[idx], hist of the mapped labels or None without query_label)."""
    point_label = np.asarray(ref_label, np.int64)[np.asarray(idx, np.int64)]
    if query_label is None:
        return point_label, None
    gt, pred = map_labels(lut, query_label), map_labels(lut, point_label)
    k = (gt >= 0) & (gt < C)
    if (pred[k] >= C).any():
        raise KeyError("a counted prediction lies outside [0, C)")
    return point_label, fast_hist(pred, gt, C)


def centres(coords, T):
    """`utils.py:326-330` for one batch item: coords int [M, 3] (x, y, z), T the float32 [16] transformation -> fp64 [M, 3]."""
    inv = np.linalg.inv(np.asarray(T, np.float32).reshape(4, 4))
    xyz = np.hstack((np.asarray(coords)[:, :3] + 0.5, np.ones((len(coords), 1))))
    return (inv @ xyz.T).T[:, :3]


def save_predictions(coords, pred, transformation, label_map, C, iteration, save_pred_dir):
    """`utils.py:304-349` with batch-first coords int [N, 4] and transformation float32 [B, 17]: `pred_%04d_%02d.npy` fp64 [M, 4] per
    batch item.  Returns the written arrays."""
    coords, pred = np.asarray(coords), np.asarray(pred, np.int64)
    dec = decode_lut(label_map, C)
    out = []
    for i in range(int(coords[:, 0].max()) + 1):
        mask = coords[:, 0] == i
        full = np.hstack((centres(coords[mask, 1:4], transformation[i, :16]), dec[pred[mask]][:, None]))
        np.save(os.path.join(save_pred_dir, "pred_%04d_%02d.npy" % (iteration, i)), full)
        out.append(full)
    return out


def read_cloud(path):
    """A semseg PLY as (fp64 [n, 7] = x, y, z, r, g, b, label; whether it has a label property).  Without a label the column is 0."""
    from pointcontrast_b200.semseg_data import read_ply
    v = read_ply(path)
    has = "label" in v.dtype.names
    cols = [v[k] for k in ("x", "y", "z", "red", "green", "blue")] + [v["label"] if has else np.zeros(len(v))]
    return np.stack([np.asarray(c, np.float64) for c in cols], 1), has


def scannet_output_id(data_path):
    """`scannet.py:121-122`."""
    return "_".join(os.path.splitext(os.path.basename(data_path))[0].split("_")[:2])


def s3dis_groups(data_paths):
    """`stanford.py:43-49`: {(area, room type): [dataset indices]} in order of first appearance."""
    groups = collections.OrderedDict()
    for i, p in enumerate(data_paths):
        area, room = p.split(os.sep)
        room = os.path.splitext(room)[0]
        groups.setdefault((area, "_".join(room.split("_")[:-1])), []).append(i)
    return groups


def test_pointcloud_scannet(preds, data_paths, data_root, label_map, C, eval_path=None, nearest_fn=nearest):
    """`scannet.py:131-172`: preds[i] = the fp64 [M, 4] prediction of dataset item i.  Writes `<eval_path>/<scene>.txt` when eval_path is
    given.  Returns (hist int64 [C, C], {scene: per-point original ids})."""
    lut = label_lut(label_map)
    hist = np.zeros((C, C), np.int64)
    labels = {}
    for i, p in enumerate(data_paths):
        pred = np.asarray(preds[i])
        cloud, has = read_cloud(os.path.join(data_root, p))
        idx = nearest_fn(pred[:, :3], cloud[:, :3])
        point_label, h = label_transfer(idx, pred[:, 3].astype(np.int64), cloud[:, 6] if has else None, lut, C)
        room_id = scannet_output_id(p)
        labels[room_id] = point_label
        if eval_path is not None:
            np.savetxt(os.path.join(eval_path, room_id + ".txt"), point_label, fmt="%i")
        if h is not None:
            hist += h
    return hist, labels


def test_pointcloud_s3dis(preds, data_paths, data_root, label_map, C, nearest_fn=nearest):
    """`stanford.py:41-84`: returns (hist int64 [C, C], the cumulative histogram after each group)."""
    lut = label_lut(label_map)
    hist = np.zeros((C, C), np.int64)
    after = []
    for rooms in s3dis_groups(data_paths).values():
        pred = np.vstack([np.asarray(preds[i]) for i in rooms])
        cloud = np.vstack([read_cloud(os.path.join(data_root, data_paths[i]))[0] for i in rooms])
        cloud = np.unique(cloud, axis=0)
        idx = nearest_fn(pred[:, :3], cloud[:, :3])
        _, h = label_transfer(idx, pred[:, 3].astype(np.int64), cloud[:, 6], lut, C)
        hist += h
        after.append(hist.copy())
    return hist, after
