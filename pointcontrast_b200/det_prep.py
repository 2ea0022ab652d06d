"""VoteNet's detection training files from the released datasets (DESIGN.md 8f-15): the reference's
`downstream/votenet_det_new/lib/datasets/scannet/batch_load_scannet_data.py` (ScanNet) and `sunrgbd/sunrgbd_data.py --gen_v1_data` /
`--gen_v2_data` (SUN RGB-D), whose files this writes -- the folders `det_data.ScannetDetectionDataset` and
`SunrgbdDetectionVotesDataset` read.

    convert_scannet("ScanNet/scans", "scannet_train_detection_data", "scannetv2-labels.combined.tsv")    # <out>/<scene>_*.npy
    convert_sunrgbd("sunrgbd_trainval", "sunrgbd")      # <out>/sunrgbd_pc_bbox_votes_50k_v1_{train,val}/%06d_{pc.npz,bbox.npy,votes.npz}

    python -m pointcontrast_b200.det_prep scannet --scans <scans> --label_map <tsv> [--scan_list <txt>] --output <dir>
    python -m pointcontrast_b200.det_prep sunrgbd --input <sunrgbd_trainval> --output <dir> [--v2]

ScanNet, one scene at a time: a reader thread parses the next scene's JSON, PLY and meta line and restates `read_aggregation` as two
ordered write lists (label and instance), while the device maps the segment ids, resolves the last write per segment, aligns the vertices
and computes every instance's box (pcb_scannet_annotate); a writer thread writes the files.  SUN RGB-D: `.mat` files are read on a pool,
the ground-truth votes of several scenes are one pcb_sunrgbd_votes launch, and `savez_compressed` runs on a small pool.  The
`np.random.choice` draws stay on the calling thread in the original's order, so a process seeded with `np.random.seed(s)` writes what a
seeded original writes.

Deliberate differences from the reference (DESIGN.md section 5): the alignment is computed in a fixed order (the original's BLAS order is
unknown; the two agree after the fp32 store on everything tested), a box whose bounds meet both -0.0 and +0.0 takes -0.0 as its minimum
and +0.0 as its maximum, and the inside-box test is analytic instead of a Qhull Delaunay triangulation (they agree outside a 1e-9 band
around the faces).
"""
import argparse
import csv
import io
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from ._lib import check, lib, ptr, stream, workspace
from .pair_list import _read_ahead
from .semseg_data import read_ply
from .semseg_prep import _FileWriter

# `batch_load_scannet_data.py:18-24`
OBJ_CLASS_IDS = np.array([3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39])
MAX_NUM_POINT = 50000
# `sunrgbd_data.py:29`, `sunrgbd_utils.py:20`
TYPE_WHITELIST = ('bed', 'table', 'sofa', 'chair', 'toilet', 'desk', 'dresser', 'night_stand', 'bookshelf', 'bathtub')
TYPE2CLASS = {c: i for i, c in enumerate(TYPE_WHITELIST)}
SUNRGBD_NUM_POINT = 50000
_NONE = 0x7f7f7f7f
_I64_MAX = (1 << 63) - 1


class SceneError(ValueError):
    """A scene the original's `batch_export` reports as failed (its bare `except`) and writes nothing for."""


# ---------------------------------------------------------------------------------------------------------------- ScanNet host side

def read_label_map(path):
    """`scannet_utils.read_label_mapping(path, 'raw_category', 'nyu40id')`: a dict, with int keys when the first key reads as an int."""
    with open(path) as f:
        mapping = {row['raw_category']: int(row['nyu40id']) for row in csv.DictReader(f, delimiter='\t')}
    try:
        int(next(iter(mapping)))
    except ValueError:
        return mapping
    return {int(k): v for k, v in mapping.items()}


def read_axis_alignment(meta_path):
    """`load_scannet_data.py:71-77`: the first line holding 'axisAlignment', parsed with the original's expression (its `strip` strips
    characters, not a prefix), as fp64 [4, 4]."""
    with open(meta_path) as f:
        for line in f.readlines():
            if 'axisAlignment' in line:
                m = [float(x) for x in line.rstrip().strip('axisAlignment = ').split(' ')]
                return np.array(m).reshape((4, 4))
    raise SceneError(f"{meta_path}: no axisAlignment line")


def read_aggregation(path):
    """`load_scannet_data.read_aggregation`, quirks included: both dicts hold the same list objects, so the first object of a label also
    carries every later same-label object's segments, and a repeated objectId keeps its first position but takes the later list."""
    object_id_to_segs, label_to_segs = {}, {}
    with open(path) as f:
        data = json.load(f)
    for g in data['segGroups']:
        object_id, label, segs = g['objectId'] + 1, g['label'], g['segments']
        object_id_to_segs[object_id] = segs
        if label in label_to_segs:
            label_to_segs[label].extend(segs)
        else:
            label_to_segs[label] = segs
    return object_id_to_segs, label_to_segs


def _int_ids(values, what):
    if not all(type(v) is int for v in values):
        raise SceneError(f"{what}: a non-integer id")
    if values and (min(values) < -(1 << 63) or max(values) >= _I64_MAX):
        raise SceneError(f"{what}: an id outside int64")
    return np.array(values, dtype=np.int64)


def write_lists(object_id_to_segs, label_to_segs, label_map):
    """The label and instance passes of `export` (`load_scannet_data.py:86-100`) as ordered write lists, and per object (dict order) its
    id, first segment and box row.  Raises SceneError where the original raises without looking at a vertex: a label missing from the
    map, an id numpy cannot store as uint32, an object without segments (the box loop's KeyError)."""
    lab_seg, lab_val = [], []
    for label, segs in label_to_segs.items():
        if label not in label_map:
            raise SceneError(f"label {label!r} is not in the label map")
        v = label_map[label]
        if segs and not 0 <= v < 1 << 32:
            raise SceneError(f"label id {v} does not fit uint32")
        lab_seg += segs
        lab_val += [v] * len(segs)
    ins_seg, ins_obj, obj_id, first_seg = [], [], [], []
    n = len(object_id_to_segs)
    for d, (oid, segs) in enumerate(object_id_to_segs.items()):
        if not segs:
            raise SceneError(f"object {oid - 1} has no segments")
        if type(oid) is not int or not 0 <= oid < 1 << 32:
            raise SceneError(f"instance id {oid} does not fit uint32")
        ins_seg += segs
        ins_obj += [d] * len(segs)
        obj_id.append(oid)
        first_seg.append(segs[0])
    rows = np.array([o - 1 if o >= 1 else o - 1 + n for o in obj_id], np.int64)
    return dict(lab_seg=_int_ids(lab_seg, "segments"), lab_val=np.array(lab_val, np.uint32), ins_seg=_int_ids(ins_seg, "segments"),
                ins_obj=np.array(ins_obj, np.int32), obj_id=np.array(obj_id, np.uint32), first_seg=_int_ids(first_seg, "segments"),
                obj_row=np.where(rows < n, rows, -1).astype(np.int32), n_rows=n)


def scene_files(scans_root, name):
    d = os.path.join(scans_root, name)
    return dict(mesh=os.path.join(d, name + '_vh_clean_2.ply'), agg=os.path.join(d, name + '.aggregation.json'),
                seg=os.path.join(d, name + '_vh_clean_2.0.010000.segs.json'), meta=os.path.join(d, name + '.txt'))


def load_scene(scans_root, name, label_map):
    """Everything of one scene the host reads and decides: vertices fp32 [V, 6] (`read_mesh_vertices_rgb`), the alignment, the segment ids
    and the write lists.  Raises SceneError (or the reader's own error) where the original raises before the per-vertex work."""
    f = scene_files(scans_root, name)
    v = read_ply(f['mesh'])
    vert = np.zeros((len(v), 6), np.float32)
    for k, c in enumerate(('x', 'y', 'z', 'red', 'green', 'blue')):
        vert[:, k] = v[c]
    align = read_axis_alignment(f['meta'])
    lists = write_lists(*read_aggregation(f['agg']), label_map)
    with open(f['seg']) as fh:
        seg = _int_ids(json.load(fh)['segIndices'], f['seg'])
    if len(seg) != len(vert):
        raise SceneError(f"{f['seg']}: {len(seg)} vertices, the mesh has {len(vert)}")
    return dict(vert=vert, align=align, seg=seg, **lists)


def annotate(scene, device):
    """pcb_scannet_annotate on a scene of `load_scene`: the aligned vertices fp32 [V, 6] and the uint32 bits of sem and ins (int32 [V]) on
    the device, and the boxes fp64 [num_instances, 7] on the host.  Synchronises; raises SceneError where the original raises on the
    vertices."""
    V, n_obj, n_rows = len(scene['vert']), len(scene['obj_id']), scene['n_rows']
    if V == 0:                                          # no vertex: every segment is unknown, so only a scene without objects gets here
        if n_obj:
            raise SceneError("an object's segment is not in the mesh")
        return (torch.zeros(0, 6, device=device), torch.zeros(0, dtype=torch.int32, device=device),
                torch.zeros(0, dtype=torch.int32, device=device), np.zeros((0, 7)))
    t = {k: torch.from_numpy(np.ascontiguousarray(scene[k]).view(np.int32) if scene[k].dtype == np.uint32 else
                             np.ascontiguousarray(scene[k])).to(device, non_blocking=True)
         for k in ('vert', 'align', 'seg', 'lab_seg', 'lab_val', 'ins_seg', 'ins_obj', 'obj_id', 'first_seg', 'obj_row')}
    vout = torch.empty(V, 6, dtype=torch.float32, device=device)
    sem = torch.empty(V, dtype=torch.int32, device=device)
    ins = torch.empty(V, dtype=torch.int32, device=device)
    bbox = torch.empty(n_rows, 7, dtype=torch.float64, device=device)
    status = torch.empty(2, dtype=torch.int32, device=device)
    wsb = lib.pcb_scannet_annotate_ws_bytes(V, n_obj, n_rows)
    ws = workspace(wsb, device)
    check(lib.pcb_scannet_annotate(ptr(t['vert']), ptr(t['align']), V, ptr(t['seg']), ptr(t['lab_seg']), ptr(t['lab_val']),
                                   len(scene['lab_seg']), ptr(t['ins_seg']), ptr(t['ins_obj']), len(scene['ins_seg']), ptr(t['obj_id']),
                                   ptr(t['first_seg']), ptr(t['obj_row']), n_obj, n_rows, ptr(vout), ptr(sem), ptr(ins), ptr(bbox),
                                   ptr(status), ptr(ws), wsb, stream()))
    st = status.cpu().numpy()
    if st[0] != _NONE:
        raise SceneError(f"segment write {st[0]}: a segment no vertex has")
    if st[1] != _NONE:
        raise SceneError(f"object {int(scene['obj_id'][st[1]]) - 1}: its id is outside the {n_rows} box rows")
    return vout, sem, ins, bbox.cpu().numpy()


def _npy_header(a):
    """The header `np.save` writes before the bytes of a C-contiguous array (format 1.0)."""
    b = io.BytesIO()
    np.lib.format.write_array_header_1_0(b, np.lib.format.header_data_from_array_1_0(a))
    return b.getvalue()


def scannet_scenes(scans_root, scan_list=None):
    if scan_list is None:
        return sorted(d for d in os.listdir(scans_root) if d.startswith('scene') and os.path.isdir(os.path.join(scans_root, d)))
    with open(scan_list) as f:
        return [line.rstrip() for line in f]


def convert_scannet(scans_root, out_dir, label_map, scan_list=None, device=None, log=print):
    """`batch_load_scannet_data.batch_export` over `scan_list` (a file of scene names; default: every `scene*` directory of `scans_root`,
    sorted) with its roots as arguments.  A scene whose `_vert.npy` exists is skipped; a scene on which the original raises is reported and
    skipped, nothing written.  Returns the wall seconds of reading (reader thread), of the device work (with the draws and the copies
    back) and of writing (writer thread), and the scenes failed.  Every thread has ended when this returns or raises."""
    device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
    lmap = read_label_map(label_map) if isinstance(label_map, (str, os.PathLike)) else label_map
    os.makedirs(out_dir, exist_ok=True)
    secs = dict(read=0.0, device=0.0, write=0.0)
    todo = []
    for name in scannet_scenes(scans_root, scan_list):
        if os.path.isfile(os.path.join(out_dir, name) + '_vert.npy'):
            if log:
                log(f"{name}: File already exists. skipping.")
            continue
        todo.append(name)

    def load(name):
        t = time.perf_counter()
        try:
            return load_scene(scans_root, name, lmap)
        except Exception as e:                          # the original's bare except: reported when the scene is reached
            return e
        finally:
            secs['read'] += time.perf_counter() - t

    failed = []
    writer = _FileWriter(8)
    try:
        with torch.cuda.device(device), _read_ahead(todo, load) as scenes:
            for name, scene in scenes:
                t = time.perf_counter()
                try:
                    if isinstance(scene, Exception):
                        raise scene
                    vert, sem, ins, bbox = annotate(scene, device)
                except Exception as e:
                    failed.append(name)
                    if log:
                        log(f"Failed export scan: {name} ({e})")
                    secs['device'] += time.perf_counter() - t
                    continue
                bbox = np.ascontiguousarray(bbox[np.isin(bbox[:, -1], OBJ_CLASS_IDS)])
                if len(vert) > MAX_NUM_POINT:
                    choices = torch.from_numpy(np.random.choice(len(vert), MAX_NUM_POINT, replace=False)).to(device)
                    vert, sem, ins = (x.index_select(0, choices) for x in (vert, sem, ins))
                outs = []
                for x in (vert, sem, ins):
                    h = torch.empty(x.shape, dtype=x.dtype, pin_memory=True)
                    h.copy_(x, non_blocking=True)
                    outs.append(h)
                torch.cuda.current_stream(device).synchronize()
                secs['device'] += time.perf_counter() - t
                vert_h, sem_h, ins_h = outs[0].numpy(), outs[1].numpy().view(np.uint32), outs[2].numpy().view(np.uint32)
                prefix = os.path.join(out_dir, name)
                for suffix, a in (('_vert.npy', vert_h), ('_sem_label.npy', sem_h), ('_ins_label.npy', ins_h), ('_bbox.npy', bbox)):
                    writer.put(prefix + suffix, _npy_header(a), a)
                if log:
                    log(f"{name}: {len(scene['vert'])} vertices, {len(bbox)} boxes -> {prefix}_*.npy")
    finally:
        writer.close()
    writer.check()
    secs['write'] = writer.busy_s
    secs['failed'] = failed
    return secs


# ---------------------------------------------------------------------------------------------------------------- SUN RGB-D

def read_sunrgbd_label(path):
    """`sunrgbd_utils.read_sunrgbd_label` restricted to what the export uses: [(classname, centroid fp64 [3], l, w, h, heading)], with
    `SUNObject3d`'s own expressions (`l = data[9]`, `w = data[8]`, `h = data[10]`, `heading = -arctan2(o1, o0)`)."""
    objs = []
    with open(path) as f:
        for line in [ln.rstrip() for ln in f]:
            data = line.split(' ')
            data[1:] = [float(x) for x in data[1:]]
            orientation = np.zeros((3,))
            orientation[0], orientation[1] = data[11], data[12]
            objs.append((data[0], np.array([data[5], data[6], data[7]]), data[9], data[8], data[10],
                         -1 * np.arctan2(orientation[1], orientation[0])))
    return objs


def sunrgbd_boxes(objs):
    """The whitelisted objects in file order: `_bbox.npy` rows fp64 [K, 8] (centroid, l, w, h, heading, class) and the kernel's box rows
    [K, 8] (centroid, l, w, h, cos(-heading), sin(-heading) -- numpy's, so that the device and the numpy restatement decide alike)."""
    kept = [o for o in objs if o[0] in TYPE2CLASS]
    obbs = np.zeros((len(kept), 8))
    for k, (cls, c, l, w, h, heading) in enumerate(kept):
        obbs[k, 0:3] = c
        obbs[k, 3:6] = np.array([l, w, h])
        obbs[k, 6] = heading
        obbs[k, 7] = TYPE2CLASS[cls]
    rows = obbs.copy()
    for k in range(len(kept)):                          # one box at a time, as the numpy restatement computes them
        t = -1 * obbs[k:k + 1, 6]
        rows[k, 6], rows[k, 7] = np.cos(t)[0], np.sin(t)[0]
    return obbs, rows


def sunrgbd_votes(pcs, box_rows, device):
    """pcb_sunrgbd_votes over a batch of scenes: pcs [points [n_b, C >= 3]], box_rows [[K_b, 8] of `sunrgbd_boxes`] -> [votes fp64 [n_b, 10]]
    (host).  Synchronises."""
    pt_off = np.zeros(len(pcs) + 1, np.int64)
    pt_off[1:] = np.cumsum([len(p) for p in pcs])
    box_off = np.zeros(len(pcs) + 1, np.int64)
    box_off[1:] = np.cumsum([len(b) for b in box_rows])
    N = int(pt_off[-1])
    pts_h = torch.empty(N, 3, dtype=torch.float64, pin_memory=True)
    if N:
        np.concatenate([np.asarray(p)[:, :3] for p in pcs], out=pts_h.numpy())
    pts = pts_h.to(device, non_blocking=True)
    boxes = torch.from_numpy(np.concatenate(box_rows).reshape(-1, 8)).to(device)
    pt_off_d, box_off_d = torch.from_numpy(pt_off).to(device), torch.from_numpy(box_off).to(device)     # held until the launch is queued
    votes = torch.empty(N, 10, dtype=torch.float64, device=device)
    check(lib.pcb_sunrgbd_votes(ptr(pts), 3, pt_off.ctypes.data, ptr(pt_off_d), ptr(boxes) if len(boxes) else None, box_off.ctypes.data,
                                ptr(box_off_d), len(pcs), ptr(votes), stream()))
    out = torch.empty(votes.shape, dtype=torch.float64, pin_memory=True)
    out.copy_(votes, non_blocking=True)
    torch.cuda.current_stream(device).synchronize()
    out = out.numpy()
    return [out[a:b] for a, b in zip(pt_off[:-1], pt_off[1:])]


def _load_sunrgbd(root, label_dir, idx):
    import scipy.io as sio
    objs = read_sunrgbd_label(os.path.join(root, label_dir, '%06d.txt' % idx))
    return objs, sio.loadmat(os.path.join(root, 'depth', '%06d.mat' % idx))['instance']


def convert_sunrgbd(trainval_root, out_dir, v1=True, splits=("train", "val"), device=None, log=print, batch=8, read_threads=8,
                    write_threads=4):
    """`extract_sunrgbd_data(<split>_data_idx.txt, 'training', <out_dir>/sunrgbd_pc_bbox_votes_50k_<v>_<split>, num_point=50000,
    save_votes=True, use_v1=v1, skip_empty_scene=False)` for each split, as `--gen_v1_data` (`v1`) or `--gen_v2_data` calls it.  Labels and
    `.mat` files are read on a pool, `batch` scenes per device launch; the draws are `np.random.choice` in index order on this thread.
    Returns the wall seconds of reading (summed over the pool), of the device work and of writing (summed over the pool)."""
    device = torch.device(device or f"cuda:{torch.cuda.current_device()}")
    label_dir = 'label_v1' if v1 else 'label'
    secs = dict(read=0.0, device=0.0, write=0.0)

    def load(idx):
        t = time.perf_counter()
        try:
            return _load_sunrgbd(trainval_root, label_dir, idx)
        finally:
            secs['read'] += time.perf_counter() - t

    def save(path, fn, **arrays):
        t = time.perf_counter()
        fn(path, *arrays.values()) if fn is np.save else fn(path, **arrays)
        secs['write'] += time.perf_counter() - t

    with ThreadPoolExecutor(read_threads) as readers, ThreadPoolExecutor(write_threads) as writers, torch.cuda.device(device):
        pending = []
        try:
            for split in splits:
                with open(os.path.join(trainval_root, f'{split}_data_idx.txt')) as f:
                    idxs = [int(line.rstrip()) for line in f]
                folder = os.path.join(out_dir, f"sunrgbd_pc_bbox_votes_50k_{'v1' if v1 else 'v2'}_{split}")
                os.makedirs(folder, exist_ok=True)
                chunks = [idxs[i:i + batch] for i in range(0, len(idxs), batch)]
                ahead = [readers.submit(load, i) for i in chunks[0]] if chunks else []
                for k, chunk in enumerate(chunks):
                    loaded = [fu.result() for fu in ahead]
                    ahead = [readers.submit(load, i) for i in chunks[k + 1]] if k + 1 < len(chunks) else []
                    t = time.perf_counter()
                    pcs, obbs, rows = [], [], []
                    for objs, pc in loaded:
                        o, r = sunrgbd_boxes(objs)
                        choices = np.random.choice(pc.shape[0], SUNRGBD_NUM_POINT, replace=pc.shape[0] < SUNRGBD_NUM_POINT)
                        pcs.append(pc[choices])
                        obbs.append(o)
                        rows.append(r)
                    votes = sunrgbd_votes(pcs, rows, device)
                    secs['device'] += time.perf_counter() - t
                    for idx, pc, o, v in zip(chunk, pcs, obbs, votes):
                        p = os.path.join(folder, '%06d' % idx)
                        pending.append(writers.submit(save, p + '_pc.npz', np.savez_compressed, pc=pc))
                        pending.append(writers.submit(save, p + '_bbox.npy', np.save, arr=o))
                        pending.append(writers.submit(save, p + '_votes.npz', np.savez_compressed, point_votes=v))
                        if log:
                            log(f"{idx}: {len(o)} boxes -> {p}_*")
                    while len(pending) > 12 * batch:
                        pending.pop(0).result()
        finally:
            for fu in pending:
                fu.result()
    return secs


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m pointcontrast_b200.det_prep", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="dataset", required=True)
    s = sub.add_parser("scannet", help="ScanNet scans -> <output>/<scene>_{vert,sem_label,ins_label,bbox}.npy (on the GPU)")
    s.add_argument("--scans", required=True, help="the ScanNet scans/ folder")
    s.add_argument("--label_map", required=True, help="scannetv2-labels.combined.tsv")
    s.add_argument("--scan_list", default=None, help="a file of scene names (default: every scene* folder, sorted)")
    s.add_argument("--output", required=True)
    s.add_argument("--seed", type=int, default=None, help="np.random.seed before the draws")
    u = sub.add_parser("sunrgbd", help="sunrgbd_trainval -> <output>/sunrgbd_pc_bbox_votes_50k_v{1,2}_{train,val}/ (on the GPU)")
    u.add_argument("--input", required=True, help="the sunrgbd_trainval folder (depth/, label/, label_v1/, *_data_idx.txt)")
    u.add_argument("--output", required=True)
    u.add_argument("--v2", action="store_true", help="the v2 labels (label/) instead of v1 (label_v1/)")
    u.add_argument("--seed", type=int, default=None, help="np.random.seed before the draws")
    args = ap.parse_args(argv)
    if args.seed is not None:
        np.random.seed(args.seed)
    if args.dataset == "scannet":
        convert_scannet(args.scans, args.output, args.label_map, args.scan_list)
    else:
        convert_sunrgbd(args.input, args.output, v1=not args.v2)


if __name__ == "__main__":
    main()
