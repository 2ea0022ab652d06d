"""numpy restatement of the two VoteNet detection `__getitem__`s (`lib/datasets/scannet/scannet_detection_dataset.py`,
`lib/datasets/sunrgbd/sunrgbd_detection_dataset.py`) with the random draws passed in: `draws(kind, *args)` answers
("random",) / ("random", 3) / ("choice", n, k, replace=...) in the original's call order.  Written from the original's semantics for the
tests of pointcontrast_b200.det_data; nothing under pointcontrast_b200/ imports it.
"""
import numpy as np

MAX_NUM_OBJ = 64


def _rotz(t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def _choice(draws, n, k):
    return np.asarray(draws("choice", n, k, replace=n < k))


def scannet_item(vert, sem, ins, bbox, nyu40ids, mean_size_arr, num_points, use_height, augment, idx, draws):
    pc = vert[:, 0:3]
    color = vert[:, 3:6]
    if use_height:
        pc = np.concatenate([pc, (pc[:, 2] - np.percentile(pc[:, 2], 0.99))[:, None]], 1)
    K = bbox.shape[0]
    boxes = np.zeros((MAX_NUM_OBJ, 6))
    boxes[:K] = bbox[:, 0:6]
    ch = _choice(draws, pc.shape[0], num_points)
    pc, sem, ins, color = pc[ch], sem[ch], ins[ch], color[ch]
    if augment:
        if draws("random") > 0.5:
            pc[:, 0] = -pc[:, 0]
            boxes[:, 0] = -boxes[:, 0]
        if draws("random") > 0.5:
            pc[:, 1] = -pc[:, 1]
            boxes[:, 1] = -boxes[:, 1]
        R = _rotz(draws("random") * np.pi / 18 - np.pi / 36)
        pc[:, 0:3] = pc[:, 0:3] @ R.T
        half = np.zeros((4, MAX_NUM_OBJ, 3))
        for i, (sx, sy) in enumerate(((-1, -1), (1, -1), (1, 1), (-1, 1))):
            half[i, :, 0], half[i, :, 1] = sx * (boxes[:, 3] / 2.0), sy * (boxes[:, 4] / 2.0)
        rot = half @ R.T
        boxes = np.concatenate([boxes[:, 0:3] @ R.T, np.stack([2.0 * rot[:, :, 0].max(0), 2.0 * rot[:, :, 1].max(0), boxes[:, 5]], 1)], 1)
    votes = np.zeros((num_points, 3))
    mask = np.zeros(num_points)
    for i in np.unique(ins):
        rows = np.flatnonzero(ins == i)
        if np.isin(sem[rows[0]], nyu40ids):
            x = pc[rows, 0:3]
            votes[rows] = 0.5 * (x.min(0) + x.max(0)) - x
            mask[rows] = 1
    cls = np.array([np.flatnonzero(nyu40ids == v)[0] for v in bbox[:, 6]], np.int64)
    size_cls = np.zeros(MAX_NUM_OBJ, np.int64)
    size_res = np.zeros((MAX_NUM_OBJ, 3))
    size_cls[:K] = cls
    size_res[:K] = boxes[:K, 3:6] - mean_size_arr[cls]
    box_mask = np.zeros(MAX_NUM_OBJ)
    box_mask[:K] = 1
    return {"point_clouds": pc.astype(np.float32), "center_label": boxes[:, 0:3].astype(np.float32),
            "heading_class_label": np.zeros(MAX_NUM_OBJ, np.int64), "heading_residual_label": np.zeros(MAX_NUM_OBJ, np.float32),
            "size_class_label": size_cls, "size_residual_label": size_res.astype(np.float32), "sem_cls_label": size_cls.copy(),
            "box_label_mask": box_mask.astype(np.float32), "vote_label": np.tile(votes, (1, 3)).astype(np.float32),
            "vote_label_mask": mask.astype(np.int64), "scan_idx": np.array(idx, np.int64), "pcl_color": color}


def _angle2class(angle, nh):
    apc = 2 * np.pi / float(nh)
    shifted = (angle % (2 * np.pi) + apc / 2) % (2 * np.pi)
    c = int(shifted / apc)
    return c, shifted - (c * apc + apc / 2)


def sunrgbd_item(pc, votes, bbox, num_heading_bin, mean_size_arr, num_points, use_color, use_height, augment, idx, draws):
    pc = pc[:, 0:6].copy() if use_color else pc[:, 0:3].copy()
    votes, bbox = votes.copy(), bbox.copy()
    if use_color:
        pc[:, 3:] = pc[:, 3:] - 0.5
    if use_height:
        pc = np.concatenate([pc, (pc[:, 2] - np.percentile(pc[:, 2], 0.99))[:, None]], 1)
    if augment:
        if draws("random") > 0.5:
            pc[:, 0] = -pc[:, 0]
            bbox[:, 0] = -bbox[:, 0]
            bbox[:, 6] = np.pi - bbox[:, 6]
            votes[:, [1, 4, 7]] = -votes[:, [1, 4, 7]]
        angle = draws("random") * np.pi / 3 - np.pi / 6
        R = _rotz(angle)
        ends = [(pc[:, 0:3] + votes[:, 1 + 3 * j:4 + 3 * j]) @ R.T for j in range(3)]
        pc[:, 0:3] = pc[:, 0:3] @ R.T
        bbox[:, 0:3] = bbox[:, 0:3] @ R.T
        bbox[:, 6] -= angle
        for j in range(3):
            votes[:, 1 + 3 * j:4 + 3 * j] = ends[j] - pc[:, 0:3]
        if use_color:
            rgb = pc[:, 3:6] + 0.5
            rgb *= 1 + 0.4 * draws("random", 3) - 0.2
            rgb += 0.1 * draws("random", 3) - 0.05
            rgb += (0.05 * draws("random", pc.shape[0]) - 0.025)[:, None]
            rgb = np.clip(rgb, 0, 1)
            rgb *= (draws("random", pc.shape[0]) > 0.3)[:, None]
            pc[:, 3:6] = rgb - 0.5
        s = draws("random") * 0.3 + 0.85
        pc[:, 0:3] *= s
        bbox[:, 0:6] *= s
        votes[:, 1:10] *= s
        if use_height:
            pc[:, -1] *= s
    K = bbox.shape[0]
    centers = np.zeros((MAX_NUM_OBJ, 3))
    hcls, hres, scls = (np.zeros(MAX_NUM_OBJ) for _ in range(3))
    sres = np.zeros((MAX_NUM_OBJ, 3))
    for i in range(K):
        hcls[i], hres[i] = _angle2class(bbox[i, 6], num_heading_bin)
        c = int(bbox[i, 7])
        scls[i], sres[i] = c, bbox[i, 3:6] * 2 - mean_size_arr[c]
        l, w, h = bbox[i, 3:6]
        corners = _rotz(-1 * bbox[i, 6]) @ np.array([[-l, l, l, -l, -l, l, l, -l], [w, w, -w, -w, w, w, -w, -w],
                                                     [h, h, h, h, -h, -h, -h, -h]])
        corners += bbox[i, 0:3, None]
        centers[i] = (corners.min(1) + corners.max(1)) / 2
    ch = _choice(draws, pc.shape[0], num_points)
    mask = np.zeros(MAX_NUM_OBJ)
    mask[:K] = 1
    sem = np.zeros(MAX_NUM_OBJ)
    sem[:K] = bbox[:, 7]
    maxb = np.zeros((MAX_NUM_OBJ, 8))
    maxb[:K] = bbox
    return {"point_clouds": pc[ch].astype(np.float32), "center_label": centers.astype(np.float32),
            "heading_class_label": hcls.astype(np.int64), "heading_residual_label": hres.astype(np.float32),
            "size_class_label": scls.astype(np.int64), "size_residual_label": sres.astype(np.float32),
            "sem_cls_label": sem.astype(np.int64), "box_label_mask": mask.astype(np.float32),
            "vote_label": votes[ch, 1:].astype(np.float32), "vote_label_mask": votes[ch, 0].astype(np.int64),
            "scan_idx": np.array(idx, np.int64), "max_gt_bboxes": maxb}
