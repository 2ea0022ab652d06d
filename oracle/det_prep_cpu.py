"""numpy restatement of VoteNet's detection preprocessing (`downstream/votenet_det_new/lib/datasets/scannet/{batch_load_scannet_data.py,
load_scannet_data.py, scannet_utils.py}` and `sunrgbd/sunrgbd_data.py` `extract_sunrgbd_data` with `--gen_v1_data` / `--gen_v2_data`'s
arguments): the checker of pointcontrast_b200/det_prep.py, and the host route of profiles/bench_det_prep.py.  Nothing under
pointcontrast_b200/ imports this.

Where it departs from the original it follows the documented rules of the GPU route (DESIGN.md section 5): the alignment is
((x M0 + y M1) + z M2) + M3 per row, each operation rounded once; a bound meeting both zeros is -0.0 (minimum) / +0.0 (maximum); the
inside-box test is analytic.  Everything else is the original's expression.
"""
import csv
import json
import os

import numpy as np

OBJ_CLASS_IDS = np.array([3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39])
MAX_NUM_POINT = 50000
TYPE2CLASS = {'bed': 0, 'table': 1, 'sofa': 2, 'chair': 3, 'toilet': 4, 'desk': 5, 'dresser': 6, 'night_stand': 7, 'bookshelf': 8,
              'bathtub': 9}
NUM_POINT = 50000


def read_ply_vertices(path):
    """x y z red green blue of a binary little-endian PLY's vertex element as fp32 [V, 6] (`scannet_utils.read_mesh_vertices_rgb`)."""
    types = {'float': '<f4', 'float32': '<f4', 'double': '<f8', 'uchar': 'u1', 'uint8': 'u1', 'ushort': '<u2', 'short': '<i2',
             'int': '<i4', 'uint': '<u4'}
    with open(path, 'rb') as f:
        fields, n, elem = [], 0, None
        while True:
            w = f.readline().decode('ascii').split()
            if w and w[0] == 'end_header':
                break
            if w and w[0] == 'element':
                elem = w[1]
                if elem == 'vertex':
                    n = int(w[2])
            elif w and w[0] == 'property' and elem == 'vertex':
                fields.append((w[2], types[w[1]]))
        v = np.frombuffer(f.read(n * np.dtype(fields).itemsize), dtype=fields, count=n)
    out = np.zeros((n, 6), np.float32)
    for k, c in enumerate(('x', 'y', 'z', 'red', 'green', 'blue')):
        out[:, k] = v[c]
    return out


def read_label_mapping(path):
    mapping = {}
    with open(path) as f:
        for row in csv.DictReader(f, delimiter='\t'):
            mapping[row['raw_category']] = int(row['nyu40id'])
    try:
        int(list(mapping.keys())[0])
        return {int(k): v for k, v in mapping.items()}
    except ValueError:
        return mapping


def align(xyz, m):
    """[x y z 1] . M^T per row, fp64, in a fixed order; then fp32."""
    p = xyz.astype(np.float64)
    out = np.empty_like(xyz)
    for r in range(3):
        out[:, r] = ((p[:, 0] * m[r, 0] + p[:, 1] * m[r, 1]) + p[:, 2] * m[r, 2]) + m[r, 3]
    return out


def _bound(a, fn, zero_sign):
    v = fn(a)
    if np.isnan(v):
        return np.float32(np.nan)
    if v == 0 and (np.signbit(a[a == 0]) == zero_sign).any():
        return np.float32(-0.0 if zero_sign else 0.0)
    return v


def export(mesh_file, agg_file, seg_file, meta_file, label_map):
    """`load_scannet_data.export` (no output file): (vertices fp32 [V, 6], label_ids uint32, instance_ids uint32, boxes fp64 [n, 7]).
    Raises where the original raises."""
    mesh_vertices = read_ply_vertices(mesh_file)
    for line in open(meta_file).readlines():
        if 'axisAlignment' in line:
            axis_align_matrix = [float(x) for x in line.rstrip().strip('axisAlignment = ').split(' ')]
            break
    axis_align_matrix = np.array(axis_align_matrix).reshape((4, 4))
    mesh_vertices[:, 0:3] = align(mesh_vertices[:, 0:3], axis_align_matrix)
    object_id_to_segs, label_to_segs = {}, {}
    data = json.load(open(agg_file))
    for g in data['segGroups']:
        object_id, label, segs = g['objectId'] + 1, g['label'], g['segments']
        object_id_to_segs[object_id] = segs
        if label in label_to_segs:
            label_to_segs[label].extend(segs)
        else:
            label_to_segs[label] = segs
    seg_ids = np.array(json.load(open(seg_file))['segIndices'], np.int64)
    num_verts = len(seg_ids)
    order = np.argsort(seg_ids, kind='stable')
    uniq, start = np.unique(seg_ids[order], return_index=True)
    bounds = dict(zip(uniq.tolist(), zip(start.tolist(), np.append(start[1:], num_verts).tolist())))
    seg_to_verts = {s: order[a:b] for s, (a, b) in bounds.items()}
    label_ids = np.zeros(num_verts, np.uint32)
    for label, segs in label_to_segs.items():
        label_id = label_map[label]
        for seg in segs:
            label_ids[seg_to_verts[seg]] = label_id
    instance_ids = np.zeros(num_verts, np.uint32)
    object_id_to_label_id = {}
    for object_id, segs in object_id_to_segs.items():
        for seg in segs:
            verts = seg_to_verts[seg]
            instance_ids[verts] = object_id
            if object_id not in object_id_to_label_id:
                object_id_to_label_id[object_id] = label_ids[verts][0]
    instance_bboxes = np.zeros((len(object_id_to_segs), 7))
    for obj_id in object_id_to_segs:
        label_id = object_id_to_label_id[obj_id]
        obj_pc = mesh_vertices[instance_ids == obj_id, 0:3]
        if len(obj_pc) == 0:
            continue
        mn = [_bound(obj_pc[:, c], np.min, True) for c in range(3)]
        mx = [_bound(obj_pc[:, c], np.max, False) for c in range(3)]
        instance_bboxes[obj_id - 1, :] = np.array([(mn[0] + mx[0]) / 2, (mn[1] + mx[1]) / 2, (mn[2] + mx[2]) / 2,
                                                   mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2], label_id])
    return mesh_vertices, label_ids, instance_ids, instance_bboxes


def export_one_scan(scans_root, scan_name, label_map):
    """`batch_load_scannet_data.export_one_scan` without the writes: the four arrays it saves."""
    d = os.path.join(scans_root, scan_name)
    v, sem, ins, boxes = export(os.path.join(d, scan_name + '_vh_clean_2.ply'), os.path.join(d, scan_name + '.aggregation.json'),
                                os.path.join(d, scan_name + '_vh_clean_2.0.010000.segs.json'), os.path.join(d, scan_name + '.txt'), label_map)
    mask = np.ones(len(sem), bool)                      # DONOTCARE_CLASS_IDS is empty
    v, sem, ins = v[mask, :], sem[mask], ins[mask]
    boxes = boxes[np.isin(boxes[:, -1], OBJ_CLASS_IDS), :]
    if v.shape[0] > MAX_NUM_POINT:
        choices = np.random.choice(v.shape[0], MAX_NUM_POINT, replace=False)
        v, sem, ins = v[choices, :], sem[choices], ins[choices]
    return v, sem, ins, boxes


def convert_scannet(scans_root, out_dir, label_map_file, scan_names):
    """`batch_export` over `scan_names`; returns the names that failed."""
    label_map = read_label_mapping(label_map_file)
    os.makedirs(out_dir, exist_ok=True)
    failed = []
    for name in scan_names:
        prefix = os.path.join(out_dir, name)
        if os.path.isfile(prefix + '_vert.npy'):
            continue
        try:
            arrays = export_one_scan(scans_root, name, label_map)
        except Exception:
            failed.append(name)
            continue
        for suffix, a in zip(('_vert.npy', '_sem_label.npy', '_ins_label.npy', '_bbox.npy'), arrays):
            np.save(prefix + suffix, a)
    return failed


# ---------------------------------------------------------------------------------------------------------------- SUN RGB-D

def read_objects(path):
    """`read_sunrgbd_label`: [(classname, centroid, l, w, h, heading)]."""
    objs = []
    for line in [ln.rstrip() for ln in open(path)]:
        data = line.split(' ')
        data[1:] = [float(x) for x in data[1:]]
        o = np.zeros((3,))
        o[0], o[1] = data[11], data[12]
        objs.append((data[0], np.array([data[5], data[6], data[7]]), data[9], data[8], data[10], -1 * np.arctan2(o[1], o[0])))
    return objs


def inside(pts, centroid, l, w, h, heading):
    """The analytic inside test: |u| <= (l, w, h) for u = rotz(-heading)^T (p - centroid), each operation rounded once; False for every
    point of a box with l, w or h not > 0 or a non-finite value."""
    c, s = np.cos(-1 * np.array([heading]))[0], np.sin(-1 * np.array([heading]))[0]
    vals = np.array([*centroid, l, w, h, c, s])
    if not (l > 0 and w > 0 and h > 0 and np.isfinite(vals).all()):
        return np.zeros(len(pts), bool)
    dx, dy, dz = pts[:, 0] - centroid[0], pts[:, 1] - centroid[1], pts[:, 2] - centroid[2]
    ux = c * dx + s * dy
    uy = c * dy - s * dx
    return (np.abs(ux) <= l) & (np.abs(uy) <= w) & (np.abs(dz) <= h)


def votes(pc, objs):
    """`point_votes` of `extract_sunrgbd_data` for the whitelisted objects `objs` of `read_objects`, file order."""
    N = pc.shape[0]
    point_votes = np.zeros((N, 10))
    idx = np.zeros(N, np.int64)
    for cls, centroid, l, w, h, heading in objs:
        if cls not in TYPE2CLASS:
            continue
        m = inside(pc, centroid, l, w, h, heading)
        v = np.expand_dims(centroid, 0) - pc[m, 0:3]
        point_votes[m, 0] = 1
        k = idx[m]
        rows = np.flatnonzero(m)
        for slot in range(3):
            sel = (k == slot) | (k == 0)
            point_votes[rows[sel], 1 + 3 * slot:4 + 3 * slot] = v[sel]
        idx[m] = np.minimum(2, idx[m] + 1)
    return point_votes


def boxes(objs):
    rows = [np.array([*c, l, w, h, heading, TYPE2CLASS[cls]]) for cls, c, l, w, h, heading in objs if cls in TYPE2CLASS]
    return np.vstack(rows) if rows else np.zeros((0, 8))


def convert_sunrgbd(trainval_root, out_dir, v1=True, splits=('train', 'val')):
    """`extract_sunrgbd_data` per split as `--gen_v1_data` (v1) / `--gen_v2_data` call it."""
    import scipy.io as sio
    for split in splits:
        folder = os.path.join(out_dir, f"sunrgbd_pc_bbox_votes_50k_{'v1' if v1 else 'v2'}_{split}")
        os.makedirs(folder, exist_ok=True)
        for idx in [int(line.rstrip()) for line in open(os.path.join(trainval_root, f'{split}_data_idx.txt'))]:
            objs = read_objects(os.path.join(trainval_root, 'label_v1' if v1 else 'label', '%06d.txt' % idx))
            pc = sio.loadmat(os.path.join(trainval_root, 'depth', '%06d.mat' % idx))['instance']
            pc = pc[np.random.choice(pc.shape[0], NUM_POINT, replace=pc.shape[0] < NUM_POINT)]
            np.savez_compressed(os.path.join(folder, '%06d_pc.npz' % idx), pc=pc)
            np.save(os.path.join(folder, '%06d_bbox.npy' % idx), boxes(objs))
            np.savez_compressed(os.path.join(folder, '%06d_votes.npz' % idx), point_votes=votes(pc, objs))
