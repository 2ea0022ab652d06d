"""Synthetic ScanNet-pair-shaped voxel clouds (SURVEY.md section 8d).

Produces the batch dictionary the reference's collate function yields
(`pretrain/pointcontrast/lib/ddp_data_loaders.py:52-112`): batch-index-first int32
coordinates, fp32 3-channel features (ones + jitter, `:248-249`), and int32
correspondences indexing rows of the *batched* feature matrices (`:85-91`).

Host-side numpy/scipy only; no CUDA and no oracle involved.
"""
import struct
import zlib

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


def synth_votenet_loss_batch(seed, batch_size, num_points, num_seed, num_proposal, vote_factor, num_heading_bin, mean_size, num_class,
                             max_obj=64, scale=1.5):
    """A seeded labelled VoteNet batch with predictions: every `end_points` array `loss_helper.get_loss` reads, as numpy.

    Labels follow `scannet_detection_dataset.py`: scene b is the room of `synth_votenet_batch(seed, ...)` with 3 to 12 random axis-aligned
    boxes standing on its floor in the first slots of `max_obj`, the rest zero with box_label_mask 0; a point inside
    a box votes for its centre (vote_label = centre - point, the 3 slots for the first 3 boxes that hold it, the first repeated) with
    vote_label_mask 1.  Predictions stand in for the network: seeds a random subset (int32 seed_inds), votes near the true centres,
    proposals (aggregated_vote_xyz) at votes, centres and scores with noise, half of the proposals near a box."""
    rng = np.random.default_rng(seed)
    B, N, S, K, V, NH, NS, C = batch_size, num_points, num_seed, num_proposal, vote_factor, num_heading_bin, len(mean_size), num_class
    pc = synth_votenet_batch(seed, B, N, scale)
    ep = {k: np.zeros(s, d) for k, s, d in (
        ("vote_label", (B, N, 9), np.float32), ("vote_label_mask", (B, N), np.int64), ("center_label", (B, max_obj, 3), np.float32),
        ("heading_class_label", (B, max_obj), np.int64), ("heading_residual_label", (B, max_obj), np.float32),
        ("size_class_label", (B, max_obj), np.int64), ("size_residual_label", (B, max_obj, 3), np.float32),
        ("sem_cls_label", (B, max_obj), np.int64), ("box_label_mask", (B, max_obj), np.float32))}
    ep["point_clouds"] = pc
    for b in range(B):
        lo, hi = pc[b].min(0), pc[b].max(0)
        boxes = []
        for _ in range(rng.integers(3, 13)):
            size = rng.uniform(0.3, 1.5, 3)
            c = rng.uniform(lo + size / 2, hi - size / 2)
            c[2] = lo[2] + size[2] / 2                                  # standing on the floor
            boxes.append((c, size))
        votes = [[] for _ in range(N)]
        for j, (c, s) in enumerate(boxes):
            sc = rng.integers(NS)
            ep["center_label"][b, j] = c
            ep["size_class_label"][b, j] = sc
            ep["size_residual_label"][b, j] = s - np.asarray(mean_size, np.float32)[sc]
            ep["heading_class_label"][b, j] = rng.integers(NH)
            ep["heading_residual_label"][b, j] = rng.uniform(-np.pi / NH, np.pi / NH)
            ep["sem_cls_label"][b, j] = rng.integers(C)
            ep["box_label_mask"][b, j] = 1
            for i in np.flatnonzero((np.abs(pc[b] - c) <= s / 2).all(1)):
                votes[i].append(c - pc[b, i])
        for i, v in enumerate(votes):
            if v:
                v = (v + [v[0]] * 3)[:3]
                ep["vote_label"][b, i] = np.concatenate(v)
                ep["vote_label_mask"][b, i] = 1
    inds = np.stack([rng.choice(N, S, replace=False) for _ in range(B)]).astype(np.int32)
    seed_xyz = np.take_along_axis(pc, inds[..., None].astype(np.int64), 1)
    gt_vote = np.take_along_axis(ep["vote_label"], inds[..., None].astype(np.int64), 1)[:, :, :3]
    vote_xyz = seed_xyz[:, :, None, :] + gt_vote[:, :, None, :] + rng.normal(0, 0.15, (B, S, V, 3))
    agg = vote_xyz.reshape(B, S * V, 3)[np.arange(B)[:, None], np.stack([rng.choice(S * V, K, replace=K > S * V) for _ in range(B)])]
    near = rng.random((B, K)) < 0.5
    slot = np.stack([rng.integers(0, int(ep["box_label_mask"][b].sum()), K) for b in range(B)])
    agg = np.where(near[..., None], ep["center_label"][np.arange(B)[:, None], slot] + rng.normal(0, 0.15, (B, K, 3)), agg)
    ep.update(seed_inds=inds, seed_xyz=seed_xyz.astype(np.float32), vote_xyz=vote_xyz.reshape(B, S * V, 3).astype(np.float32),
              aggregated_vote_xyz=agg.astype(np.float32), center=(agg + rng.normal(0, 0.1, (B, K, 3))).astype(np.float32))
    for k, n in (("objectness_scores", (2,)), ("heading_scores", (NH,)), ("heading_residuals_normalized", (NH,)), ("size_scores", (NS,)),
                 ("size_residuals_normalized", (NS, 3)), ("sem_cls_scores", (C,))):
        ep[k] = rng.normal(0, 1.0 if k.endswith("scores") else 0.5, (B, K) + n).astype(np.float32)
    return ep


def _scan_rects(scale):
    """The closed room of the scan walks (the `synth_room` surfaces and the two other walls), as plane arrays O, U, V, N at `scale`."""
    rects = _rects() + [tuple(np.asarray(a, np.float64) for a in r) for r in (((_W, 0, 0), (0, _L, 0), (0, 0, _H)),      # wall x=W
                                                                            ((0, _L, 0), (_W, 0, 0), (0, 0, _H)))]     # wall y=L
    O, U, V = (np.stack([r[k] for r in rects]) * scale for k in range(3))
    return O, U, V, np.cross(U, V)


def _walk_pose(yaw, phase, scale):
    """The camera of the scan walks: on a circle around the room centre at 60 % of the wall height, looking 20 degrees down in
    direction `yaw`.  Returns (position, look, side, up)."""
    centre = np.array([_W / 2, _L / 2, 0.6 * _H]) * scale
    pos = centre + np.array([0.2 * _W * np.cos(phase), 0.2 * _L * np.sin(phase), 0.0]) * scale
    look = np.array([np.cos(yaw), np.sin(yaw), -np.tan(np.deg2rad(20.0))])
    look /= np.linalg.norm(look)
    side = np.cross(look, [0.0, 0.0, 1.0])
    side /= np.linalg.norm(side)
    return pos, look, side, np.cross(side, look)


def _first_hit(rays, pos, planes):
    """The ray parameter of the nearest surface each ray (rows of `rays`, from `pos`) hits, inf where it hits none."""
    O, U, V, N = planes
    uu, vv = np.einsum("ij,ij->i", U, U), np.einsum("ij,ij->i", V, V)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = ((O - pos) * N).sum(1) / (rays @ N.T)                       # [m, rects]: the ray's parameter at each plane
        a = (((pos - O) * U).sum(1) + t * (rays @ U.T)) / uu            # the hit point in the rectangle's (u, v) coordinates
        b = (((pos - O) * V).sum(1) + t * (rays @ V.T)) / vv
        t = np.where((t > 0) & (a >= 0) & (a <= 1) & (b >= 0) & (b <= 1), t, np.inf)
    return t.min(1)


def synth_scan_frames(seed, n_frames, points_per_frame=250_000, scale=2.0, half_angle_deg=30.0):
    """A depth-camera walk through a `synth_room`-style room (at `scale`): n_frames fp64 [points_per_frame, 3] world-frame clouds, the
    `pcd` of ScanNet's `<scene>/pcd/<frame>.npz` (about 250k points, like a 640x480 depth frame).  Frame k casts rays uniformly over a
    view cone of `half_angle_deg` from pose k and keeps the nearest surface each ray hits (the room closed by its two other walls, so
    every ray hits one), + N(0, 5 mm) noise.  The camera circles the room centre at 60 % of the wall height, looking 20 degrees down, and turns
    10-50 degrees between frames, so consecutive frames overlap by amounts on both sides of the pair list's 0.3 threshold."""
    rng = np.random.default_rng(seed)
    planes = _scan_rects(scale)
    cos_half = np.cos(np.deg2rad(half_angle_deg))
    yaw, phase = rng.random() * 2 * np.pi, rng.random() * 2 * np.pi
    frames = []
    for _ in range(n_frames):
        pos, look, side, up = _walk_pose(yaw, phase, scale)
        got, parts, frac = 0, [], 0.5
        while got < points_per_frame:
            m = int(1.2 * (points_per_frame - got) / frac) + 1024
            c = 1.0 - rng.random(m) * (1.0 - cos_half)                      # uniform over the cone's solid angle
            s, phi = np.sqrt(1.0 - c * c), rng.random(m) * 2 * np.pi
            d = c[:, None] * look + (s * np.cos(phi))[:, None] * side + (s * np.sin(phi))[:, None] * up
            tmin = _first_hit(d, pos, planes)
            keep = np.isfinite(tmin)
            frac = max(keep.mean(), 0.5)
            parts.append(pos + tmin[keep, None] * d[keep])
            got += int(keep.sum())
        pts = np.concatenate(parts)[:points_per_frame]
        frames.append(pts + rng.normal(0.0, 0.005, size=pts.shape))
        yaw += np.deg2rad(rng.uniform(10.0, 50.0))
        phase += np.deg2rad(rng.uniform(5.0, 20.0))
    return frames



# ScanNet's depth camera (640 x 480; `_info.txt` of a scan): non-integral principal point
SCANNET_DEPTH_INTRINSIC = np.array([[577.590698, 0.0, 318.905426, 0.0], [0.0, 578.729797, 242.683609, 0.0], [0.0, 0.0, 1.0, 0.0],
                                    [0.0, 0.0, 0.0, 1.0]])
SCANNET_COLOR_INTRINSIC = np.array([[1170.187988, 0.0, 647.75, 0.0], [0.0, 1170.187988, 483.75, 0.0], [0.0, 0.0, 1.0, 0.0],
                                    [0.0, 0.0, 0.0, 1.0]])


def write_sens(path, depth, poses, intrinsic_depth, seed=0, version=4, depth_compression=1, color_size=(1296, 968),
               color_bytes=(90_000, 160_000)):
    """A `.sens` file in the layout `SensorData.load` reads (`SensorData.py:57-79`): depth uint16 [F, H, W] zlib-compressed, poses
    [F, 4, 4] stored as float32, the depth intrinsics and ScanNet's colour intrinsics, identity extrinsics.  Each frame's colour
    payload is `color_bytes` random bytes (uniform in the range; a ScanNet JPEG is about that size), so that a loader that reads colour
    pays for it.  `version` and `depth_compression` are written as given."""
    depth = np.asarray(depth, np.uint16)
    F, H, W = depth.shape
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 256, color_bytes[1], dtype=np.uint8).tobytes()
    eye = np.eye(4, dtype=np.float32)
    with open(path, "wb") as f:
        name = b"StructureSensor"
        f.write(struct.pack("<IQ", version, len(name)) + name)
        for m in (SCANNET_COLOR_INTRINSIC, eye, intrinsic_depth, eye):
            f.write(np.asarray(m, "<f4").tobytes())
        f.write(struct.pack("<iiIIIIfQ", 2, depth_compression, color_size[0], color_size[1], W, H, 1000.0, F))
        for i in range(F):
            n = int(rng.integers(color_bytes[0], color_bytes[1] + 1))
            start = int(rng.integers(0, color_bytes[1] - n + 1))
            blob = zlib.compress(depth[i].astype("<u2").tobytes(), 1)
            f.write(np.asarray(poses[i], "<f4").tobytes() + struct.pack("<QQQQ", 33_333 * i, 33_333 * i + 1, n, len(blob)))
            f.write(pool[start:start + n])
            f.write(blob)


def synth_sens_scan(seed, n_frames, width=640, height=480, frames_per_view=1, render_every=1, holes=0.02, far=0.001, bad_poses=(),
                    scale=2.0):
    """A ScanNet-like depth scan for `write_sens`: (depth uint16 [n_frames, height, width] in millimetres, camera-to-world poses fp64
    [n_frames, 4, 4], the 4 x 4 depth intrinsics).  The camera walks as in `synth_scan_frames` (room, circle, look direction), turning
    1 / `frames_per_view` of that walk's step per frame; each frame renders the room through a pinhole with ScanNet's intrinsics
    scaled to width x height (non-integral cx, cy; camera x right, y down, z forward), depth along the optical axis + N(0, 5 mm),
    rounded to millimetres.  A `holes` share of the pixels is 0 (no reading) and a `far` share 65535 (the format's largest depth).
    Frames f with f % render_every != 0 repeat the depth of the last rendered frame (a cheaper long scan).  The frames of `bad_poses`
    get an all -inf pose, as ScanNet stores a frame without tracking."""
    rng = np.random.default_rng(seed)
    planes = _scan_rects(scale)
    K = SCANNET_DEPTH_INTRINSIC.copy()
    K[0] *= width / 640.0
    K[1] *= height / 480.0
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    v, u = np.divmod(np.arange(height * width, dtype=np.float64), width)
    cam = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], 1)          # the ray of each pixel in the camera frame, z = 1
    yaw, phase = rng.random() * 2 * np.pi, rng.random() * 2 * np.pi
    depth = np.empty((n_frames, height, width), np.uint16)
    poses = np.empty((n_frames, 4, 4))
    for i in range(n_frames):
        pos, look, side, up = _walk_pose(yaw, phase, scale)
        R = np.stack([side, -up, look], 1)
        poses[i] = np.eye(4)
        poses[i, :3, :3], poses[i, :3, 3] = R, pos
        if i % render_every == 0:
            z = _first_hit(cam @ R.T, pos, planes) + rng.normal(0.0, 0.005, height * width)
            mm = np.where(np.isfinite(z), np.clip(np.rint(z * 1000.0), 0, 65535), 0)
            r = rng.random(height * width)
            mm[r < holes] = 0
            mm[r > 1.0 - far] = 65535
            depth[i] = mm.reshape(height, width)
        else:
            depth[i] = depth[i - 1]
        yaw += np.deg2rad(rng.uniform(10.0, 50.0)) / frames_per_view
        phase += np.deg2rad(rng.uniform(5.0, 20.0)) / frames_per_view
    for i in bad_poses:
        poses[i] = -np.inf
    return depth, poses, K


def synth_scene(seed, scale=2.5, voxel=0.05, n_raw=1_500_000):
    """S3DIS-shaped single room for the forward-only config (C4): coords [N,4], RGB/255-0.5 features."""
    rng = np.random.default_rng(seed + 99)
    pts = synth_room(seed, scale, n_raw)
    pts = (pts - pts.mean(0)) @ _rot(rng).T
    c, sel = _voxelize(pts, voxel)
    f = (rng.integers(0, 256, size=(len(c), 3)).astype(np.float32) / 255.0 - 0.5)
    C = np.concatenate([np.zeros((len(c), 1), np.int32), c], 1)
    return {"coords": C, "feats": f}


# ScanNet nyu40 ids of the detected classes (`model_util_scannet.py`), used when no config is given
SCANNET_NYU40IDS = (3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39)


def write_scannet_detection_scene(path, name, seed, n, n_boxes, n_inst=8, nyu40ids=SCANNET_NYU40IDS):
    """`<path>/<name>_{vert,sem_label,ins_label,bbox}.npy` in the format of the original preprocessing (`batch_load_scannet_data.py`):
    vert fp32 [n, 6] (xyz in a 6 x 5 x 3 m room, colour 0-255), sem / ins labels uint32 [n], bbox fp64 [n_boxes, 7] (centre, size,
    nyu40 id).  Instance ids are arbitrary uint32 values: 0 (unannotated) and ids near 2^32 are always present.  The last instance mixes
    object and non-object semantic labels row by row, so whether it gets votes depends on its first sampled row."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform((-3, -2.5, 0), (3, 2.5, 3), (n, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (n, 3)).astype(np.float32)
    ids = np.unique(np.concatenate([[0, 4294967295, 2147483648 + seed],
                                    rng.choice(4294967000, max(n_inst - 3, 0), replace=False)]).astype(np.uint32))
    ins = ids[rng.integers(0, len(ids), n)].astype(np.uint32)
    sem_of = {int(i): (int(rng.choice(nyu40ids)) if rng.random() < 0.8 else int(rng.choice([1, 2, 22, 40]))) for i in ids}
    sem = np.array([sem_of[int(i)] for i in ins], np.uint32)
    mixed = ins == ids[-1]
    sem[mixed] = np.where(rng.random(int(mixed.sum())) < 0.5, nyu40ids[0], 1).astype(np.uint32)
    bbox = np.zeros((n_boxes, 7))
    bbox[:, 0:3] = rng.uniform((-2.5, -2, 0.2), (2.5, 2, 2.5), (n_boxes, 3))
    bbox[:, 3:6] = rng.uniform(0.2, 2.0, (n_boxes, 3))
    bbox[:, 6] = rng.choice(nyu40ids, n_boxes)
    np.save(f"{path}/{name}_vert.npy", np.concatenate([xyz, rgb], 1))
    np.save(f"{path}/{name}_sem_label.npy", sem)
    np.save(f"{path}/{name}_ins_label.npy", ins)
    np.save(f"{path}/{name}_bbox.npy", bbox)


def write_sunrgbd_detection_scene(path, name, seed, n, n_boxes, n_class=10):
    """`<path>/<name>_pc.npz` (pc fp64 [n, 6], colour in 0-1), `<name>_bbox.npy` fp64 [n_boxes, 8] (centre, half sizes, heading, class)
    and `<name>_votes.npz` (point_votes fp64 [n, 10]: mask, then three votes; a point inside fewer than three boxes repeats its first
    vote, as the original's `sunrgbd_data.py` export does), compressed like the original's."""
    rng = np.random.default_rng(seed)
    pc = np.concatenate([rng.uniform((-3, 0.5, -1.2), (3, 6, 1.5), (n, 3)), rng.random((n, 3))], 1)
    bbox = np.zeros((n_boxes, 8))
    bbox[:, 0:3] = rng.uniform((-2.5, 1, -1), (2.5, 5.5, 1), (n_boxes, 3))
    bbox[:, 3:6] = rng.uniform(0.1, 1.2, (n_boxes, 3))
    bbox[:, 6] = rng.uniform(-np.pi, np.pi, n_boxes)
    bbox[:, 7] = rng.integers(0, n_class, n_boxes)
    votes = np.zeros((n, 10))
    nv = rng.integers(0, 4, n) * (rng.random(n) < 0.6)
    for j in range(3):
        v = rng.uniform(-1, 1, (n, 3))
        votes[:, 1 + 3 * j:4 + 3 * j] = np.where((nv > j)[:, None], v, votes[:, 1:4])
    votes[:, 0] = nv > 0
    np.savez_compressed(f"{path}/{name}_pc.npz", pc=pc)
    np.savez_compressed(f"{path}/{name}_votes.npz", point_votes=votes)
    np.save(f"{path}/{name}_bbox.npy", bbox)
