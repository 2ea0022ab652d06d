"""Synthetic ScanNet-pair-shaped voxel clouds (SURVEY.md section 8d).

Produces the batch dictionary the reference's collate function yields
(`pretrain/pointcontrast/lib/ddp_data_loaders.py:52-112`): batch-index-first int32
coordinates, fp32 3-channel features (ones + jitter, `:248-249`), and int32
correspondences indexing rows of the *batched* feature matrices (`:85-91`).

Host-side numpy/scipy only; no CUDA and no oracle involved.
"""
import numpy as np
from scipy.spatial import cKDTree

# 9 rectangles: floor, two walls, two boxes (3 visible faces each). (origin, edge_u, edge_v)
_W, _L, _H = 3.2, 3.0, 2.4


def _rects():
    r = [((0, 0, 0), (_W, 0, 0), (0, _L, 0)),            # floor
         ((0, 0, 0), (_W, 0, 0), (0, 0, _H)),            # wall y=0
         ((0, 0, 0), (0, _L, 0), (0, 0, _H))]            # wall x=0
    for (ox, oy, sx, sy, sz) in ((1.0, 1.2, 1.2, 0.7, 0.75), (2.2, 0.4, 0.8, 0.5, 1.6)):
        r.append(((ox, oy, sz), (sx, 0, 0), (0, sy, 0)))            # top
        r.append(((ox, oy + sy, 0), (sx, 0, 0), (0, 0, sz)))        # front (y+)
        r.append(((ox + sx, oy, 0), (0, sy, 0), (0, 0, sz)))        # side (x+)
    return [tuple(np.asarray(a, dtype=np.float64) for a in t) for t in r]


def synth_room(seed, scale=0.751, n_raw=300_000):
    """Area-weighted uniform samples on the room surfaces, + N(0, 5 mm) noise. [n_raw, 3] float64."""
    rng = np.random.default_rng(seed)
    rects = _rects()
    areas = np.array([np.linalg.norm(np.cross(u, v)) for _, u, v in rects])
    which = rng.choice(len(rects), size=n_raw, p=areas / areas.sum())
    a = rng.random(n_raw)[:, None]
    b = rng.random(n_raw)[:, None]
    o = np.stack([rects[i][0] for i in range(len(rects))])[which]
    u = np.stack([rects[i][1] for i in range(len(rects))])[which]
    v = np.stack([rects[i][2] for i in range(len(rects))])[which]
    pts = (o + a * u + b * v) * scale
    pts += rng.normal(0.0, 0.005, size=pts.shape)
    return pts


def synth_labelled_room(seed, n_raw, scale=1.0, labels=(1, 2, 3, 4, 5, 6, 7, 8, 9), label_noise=0.1, num_labels=41):
    """A labelled, coloured room as the semseg `.ply` files hold it: float32 xyz [n_raw, 3], uint8 rgb [n_raw, 3], uint8 labels [n_raw].
    Each surface of `synth_room` has one label of `labels` and a base colour; a `label_noise` share of the points gets a uniformly random
    label in [0, num_labels), so voxels on surface boundaries and noisy points mix labels."""
    rng = np.random.default_rng(seed)
    rects = _rects()
    areas = np.array([np.linalg.norm(np.cross(u, v)) for _, u, v in rects])
    which = rng.choice(len(rects), size=n_raw, p=areas / areas.sum())
    a, b = rng.random(n_raw)[:, None], rng.random(n_raw)[:, None]
    o, u, v = (np.stack([r[k] for r in rects])[which] for k in range(3))
    pts = (o + a * u + b * v) * scale + rng.normal(0.0, 0.005, size=(n_raw, 3))
    base = rng.integers(30, 226, size=(len(rects), 3))
    rgb = np.clip(base[which] + rng.normal(0, 12, size=(n_raw, 3)), 0, 255).astype(np.uint8)
    lab = np.asarray(labels, np.int64)[which % len(labels)]
    noisy = rng.random(n_raw) < label_noise
    lab[noisy] = rng.integers(0, num_labels, noisy.sum())
    return pts.astype(np.float32), rgb, lab.astype(np.uint8)


def write_ply(path, xyz, rgb, labels=None):
    """A binary little-endian PLY with the vertex layout of the semseg preprocessing (`downstream/semseg/lib/pc_utils.py:41-70`)."""
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")]
    if labels is not None:
        fields.append(("label", "u1"))
    v = np.empty(len(xyz), dtype=fields)
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"], v["green"], v["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    if labels is not None:
        v["label"] = labels
    types = {"<f4": "float", "u1": "uchar"}
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"] + [f"property {types[t]} {n}" for n, t in fields]
    with open(path, "wb") as f:
        f.write(("\n".join(head + ["end_header"]) + "\n").encode("ascii"))
        f.write(v.tobytes())


def _rot(rng):
    """Random rotation, same law as `sample_random_trans` (`ddp_data_loaders.py:137-142`)."""
    axis = rng.random(3) - 0.5
    theta = (rng.random() * 2.0 - 1.0) * np.pi
    axis = axis / np.linalg.norm(axis) * theta
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    th = np.linalg.norm(axis)
    if th < 1e-12:
        return np.eye(3)
    Kn = K / th
    return np.eye(3) + np.sin(th) * Kn + (1 - np.cos(th)) * (Kn @ Kn)      # Rodrigues == expm(K)


def _voxelize(xyz, voxel):
    """First point of every occupied voxel, rows sorted by (x, y, z) voxel key. Returns (coords int32, sel)."""
    c = np.floor(xyz / voxel).astype(np.int64)
    key = ((c[:, 0] + (1 << 20)) << 42) | ((c[:, 1] + (1 << 20)) << 21) | (c[:, 2] + (1 << 20))
    _, sel = np.unique(key, return_index=True)
    return c[sel].astype(np.int32), sel


def synth_pair_raw(seed, scale=0.9, n_raw=300_000):
    """The two raw (un-voxelised) views of `synth_pair(seed, scale)` as float32 point clouds in their own frames, and the
    ground-truth transform T01 [4,4] taking view-0 coordinates to view-1 coordinates -- the inputs of the reference loader's
    per-sample work (`ddp_data_loaders.py:196-245`), for `pointcontrast_b200.voxel.make_pair`."""
    rng = np.random.default_rng(seed + 7_000_003)
    world = synth_room(seed, scale, n_raw)
    Wd = _W * scale
    v0 = world[world[:, 0] < 0.65 * Wd]
    v1 = world[world[:, 0] > 0.25 * Wd]
    R0, R1 = _rot(rng), _rot(rng)
    m0, m1 = v0.mean(0), v1.mean(0)
    T = np.eye(4)
    T[:3, :3] = R1 @ R0.T
    T[:3, 3] = R1 @ (m0 - m1)
    return {"p0": ((v0 - m0) @ R0.T).astype(np.float32), "p1": ((v1 - m1) @ R1.T).astype(np.float32), "T01": T}


def synth_pair(seed, scale=0.9, voxel=0.025, n_raw=300_000, search_mult=1.5):
    """One scene pair: two overlapping, independently rotated, voxelised views + correspondences."""
    rng = np.random.default_rng(seed + 7_000_003)
    world = synth_room(seed, scale, n_raw)
    Wd = _W * scale
    v0 = world[world[:, 0] < 0.65 * Wd]
    v1 = world[world[:, 0] > 0.25 * Wd]
    R0, R1 = _rot(rng), _rot(rng)
    m0, m1 = v0.mean(0), v1.mean(0)
    p0 = (v0 - m0) @ R0.T                     # view frames (mean-centred then rotated)
    p1 = (v1 - m1) @ R1.T
    c0, s0 = _voxelize(p0, voxel)
    c1, s1 = _voxelize(p1, voxel)
    # matches between the selected points, measured in the common world frame
    tree = cKDTree(v1[s1])
    nb = tree.query_ball_point(v0[s0], r=search_mult * voxel)
    cnt = np.fromiter((len(x) for x in nb), dtype=np.int64, count=len(nb))
    i0 = np.repeat(np.arange(len(nb)), cnt)
    i1 = np.fromiter((j for x in nb for j in sorted(x)), dtype=np.int64, count=int(cnt.sum()))
    corr = np.stack([i0, i1], 1).astype(np.int32)
    if corr.shape[0] == 0:
        corr = np.zeros((1, 2), np.int32)
    frng = np.random.default_rng(seed + 13)

    def feats(n):
        f = np.ones((n, 3), np.float32)
        if frng.random() < 0.95:
            f += frng.normal(0.0, 0.01, size=f.shape).astype(np.float32)
        return f
    return {"coords0": c0, "coords1": c1, "feats0": feats(len(c0)), "feats1": feats(len(c1)),
            "xyz0": p0[s0].astype(np.float32), "xyz1": p1[s1].astype(np.float32), "corr": corr}


def collate_pairs(pairs):
    """Batch dict in the reference's layout (`ddp_data_loaders.py:52-112`), as numpy arrays."""
    C0, C1, F0, F1, M, X0, X1, lens = [], [], [], [], [], [], [], []
    o0 = o1 = 0
    for b, p in enumerate(pairs):
        n0, n1 = len(p["coords0"]), len(p["coords1"])
        C0.append(np.concatenate([np.full((n0, 1), b, np.int32), p["coords0"]], 1))
        C1.append(np.concatenate([np.full((n1, 1), b, np.int32), p["coords1"]], 1))
        F0.append(p["feats0"]); F1.append(p["feats1"])
        X0.append(p["xyz0"]); X1.append(p["xyz1"])
        M.append(p["corr"] + np.array([[o0, o1]], np.int32))
        lens.append([n0, n1])
        o0 += n0; o1 += n1
    return {"sinput0_C": np.concatenate(C0), "sinput1_C": np.concatenate(C1),
            "sinput0_F": np.concatenate(F0), "sinput1_F": np.concatenate(F1),
            "pcd0": np.concatenate(X0), "pcd1": np.concatenate(X1),
            "correspondences": np.concatenate(M).astype(np.int32), "len_batch": lens}


def synth_batch(step, batch_size, scale=0.9, voxel=0.025, n_raw=300_000):
    """Pair p of step s uses seed 1000*s + p (SURVEY.md section 8d)."""
    return collate_pairs([synth_pair(1000 * step + p, scale, voxel, n_raw) for p in range(batch_size)])


def synth_votenet_batch(seed, batch_size, num_points, scale=1.5):
    """VoteNet's collated `point_clouds` (`no_height=True`, `use_color=False`): float32 [batch_size, num_points, 3], scene b a room of
    about 4.8 m x 4.5 m x 3.6 m (at scale 1.5) sampled with seed 1000 * seed + b, centred in x and y, floor at z = 0."""
    out = np.empty((batch_size, num_points, 3), np.float32)
    for b in range(batch_size):
        pts = synth_room(1000 * seed + b, scale, num_points)
        pts[:, :2] -= pts[:, :2].mean(0)
        out[b] = pts
    return out


def synth_scene(seed, scale=2.5, voxel=0.05, n_raw=1_500_000):
    """S3DIS-shaped single room for the forward-only config (C4): coords [N,4], RGB/255-0.5 features."""
    rng = np.random.default_rng(seed + 99)
    pts = synth_room(seed, scale, n_raw)
    pts = (pts - pts.mean(0)) @ _rot(rng).T
    c, sel = _voxelize(pts, voxel)
    f = (rng.integers(0, 256, size=(len(c), 3)).astype(np.float32) / 255.0 - 0.5)
    C = np.concatenate([np.zeros((len(c), 1), np.int32), c], 1)
    return {"coords": C, "feats": f}
