"""numpy / scipy restatement of the semantic-segmentation training data path (`downstream/semseg/lib/transforms.py`,
`lib/voxelizer.py`, `lib/dataset.py:275-309`), the checker of pointcontrast_b200/semseg_data.py.

Every function takes its random draws as arguments, so a run of the reference with recorded draws
(`tests/golden/make_semseg_golden.py`) replays here exactly.  The arithmetic follows the reference's dtypes step by step:

* elastic distortion: `scipy.ndimage.convolve` on float32 noise accumulates each 3-tap sum in float64 in footprint order
  (`0 + w x[i-1] + w x[i] + w x[i+1]`, `w = float64(float32(1/3))`, out-of-grid taps read 0) and rounds the sum to float32;
  `RegularGridInterpolator` (linear) works in float64: per axis the interval `g[i] <= x < g[i+1]` (clamped to the last one),
  `t = (x - g[i]) / (g[i+1] - g[i])`, the 8 corners in `itertools.product` order (last axis fastest) with weight `((1 * w0) * w1) * w2`,
  summed from 0 in that order; points outside `[g[0], g[-1]]` on any axis get 0.  `coords += interp * magnitude` rounds to float32.
* voxelisation: `floor(homo(xyz) @ T.T[:, :3])` in float64 (`voxelizer.py:134-135`), minus its per-axis minimum (`:138-142`),
  then `sparse_quantize` with labels (ME 0.4.3 `quantize_label`): one row per voxel in ascending (x, y, z) order, the first point of
  the voxel, its common label or `ignore_label`.
* colour: auto-contrast in float32 (`transforms.py:45-61`), translation and jitter in float64 clipped to [0, 255] and stored in
  float32 (`:32-36`, `:69-74`).
"""
import itertools

import numpy as np

F32 = np.float32


# ---------------------------------------------------------------- elastic distortion (`transforms.py:187-217`)

def noise_shape(coords, granularity):
    """`transforms.py:197-200`: the noise grid's spatial shape and the float32 per-axis minimum."""
    coords_min = coords.min(0)
    noise_dim = ((coords - coords_min).max(0) // granularity).astype(int) + 3
    return noise_dim, coords_min


def grid_axes(coords_min, granularity, noise_dim):
    """`transforms.py:210-214`: float64 axes `linspace(min - g, min + g (dim - 2), dim)` (float32 min, as the reference has it)."""
    return [np.linspace(d_min, d_max, d) for d_min, d_max, d in
            zip(coords_min - granularity, coords_min + granularity * (noise_dim - 2), noise_dim)]


def blur3(noise, axis):
    """`scipy.ndimage.convolve(noise, ones(3)/3 along `axis`, mode='constant', cval=0)` on float32 noise."""
    w = np.float64(np.float32(1.0) / np.float32(3.0))
    x = noise.astype(np.float64)
    pad = [(0, 0)] * x.ndim
    pad[axis] = (1, 1)
    xp = np.pad(x, pad)
    n = x.shape[axis]
    sl = lambda a, b: tuple(slice(a, b) if d == axis else slice(None) for d in range(x.ndim))
    acc = np.zeros_like(x)
    for k in range(3):                                   # footprint order: x[i-1], x[i], x[i+1]
        acc = acc + w * xp[sl(k, k + n)]
    return acc.astype(F32)


def smooth_noise(noise):
    """`transforms.py:204-207`: two rounds of the x, y, z box filters."""
    for _ in range(2):
        for ax in range(3):
            noise = blur3(noise, ax)
    return noise


def interpolate(axes, values, xyz):
    """`RegularGridInterpolator(axes, values, bounds_error=0, fill_value=0)(xyz)`, linear, values float32 [gx, gy, gz, 3]."""
    x = np.asarray(xyz, np.float64)
    idx, t = [], []
    oob = np.zeros(len(x), bool)
    for d, g in enumerate(axes):
        v = x[:, d]
        i = np.clip(np.searchsorted(g, v, side="right") - 1, 0, len(g) - 2)
        idx.append(i)
        t.append((v - g[i]) / (g[i + 1] - g[i]))
        oob |= (v < g[0]) | (v > g[-1])
    value = np.zeros((len(x), values.shape[-1]))
    for corner in itertools.product((0, 1), repeat=3):
        weight = np.ones(len(x))
        for d, c in enumerate(corner):
            weight = weight * (t[d] if c else 1 - t[d])
        term = values[idx[0] + corner[0], idx[1] + corner[1], idx[2] + corner[2]].astype(np.float64) * weight[:, None]
        value = value + term
    value[oob] = 0
    return value


def elastic_distortion(coords, granularity, magnitude, noise):
    """`transforms.py:187-217` with the drawn float32 noise grid `noise` [*noise_dim, 3].  Returns (new coords, blurred grid)."""
    noise_dim, coords_min = noise_shape(coords, granularity)
    assert tuple(noise.shape) == tuple(noise_dim) + (3,)
    blurred = smooth_noise(noise.astype(F32))
    out = coords.copy()
    out += interpolate(grid_axes(coords_min, granularity, noise_dim), blurred, coords) * magnitude
    return out, blurred


# ---------------------------------------------------------------- voxelisation (`voxelizer.py:49-148`)

def rotation(axis, theta):
    """`voxelizer.py:14-15`."""
    from scipy.linalg import expm, norm
    return expm(np.cross(np.eye(3), axis / norm(axis) * theta))


def transformation_matrix(voxel_size, thetas, order, scale_draw):
    """`voxelizer.py:49-79` with the drawn angles (x, y, z), the `np.random.shuffle` permutation `order` of the three rotations and the
    scale draw (None: no scale augmentation).  Returns (M_v, M_r)."""
    M_v, M_r = np.eye(4), np.eye(4)
    mats = []
    for ax, th in enumerate(thetas):
        a = np.zeros(3)
        a[ax] = 1
        mats.append(rotation(a, th))
    mats = [mats[i] for i in order]
    M_r[:3, :3] = mats[0] @ mats[1] @ mats[2]
    scale = 1 / voxel_size
    if scale_draw is not None:
        scale *= scale_draw
    np.fill_diagonal(M_v[:3, :3], scale)
    return M_v, M_r


def clip_mask(coords, clip_bound, trans_aug_ratio):
    """`voxelizer.py:81-111` for a scalar bound (S3DIS `CLIP_BOUND = 4`), centre = the bounding-box centre.  None: room too small."""
    bound_min = np.min(coords, 0).astype(float)
    bound_max = np.max(coords, 0).astype(float)
    bound_size = bound_max - bound_min
    center = bound_min + bound_size * 0.5
    center += np.multiply(trans_aug_ratio, bound_size)
    lim = clip_bound
    if bound_size.max() < lim:
        return None
    return ((coords[:, 0] >= (-lim + center[0])) & (coords[:, 0] < (lim + center[0])) & (coords[:, 1] >= (-lim + center[1])) &
            (coords[:, 1] < (lim + center[1])) & (coords[:, 2] >= (-lim + center[2])) & (coords[:, 2] < (lim + center[2])))


def affine_floor(coords, T):
    """`voxelizer.py:134-142`: (floor(homo @ T.T[:, :3]) - min) as int32, the per-axis minimum, and the float64 pre-floor values."""
    homo = np.hstack((coords, np.ones((coords.shape[0], 1), dtype=coords.dtype))).astype(np.float64)
    pre = ((homo[:, :1] * T[None, :3, 0] + homo[:, 1:2] * T[None, :3, 1]) + homo[:, 2:3] * T[None, :3, 2]) + homo[:, 3:4] * T[None, :3, 3]
    c = np.floor(pre)
    mn = c.min(0)
    return (c - mn).astype(np.int32), mn.astype(np.int64), pre


def sparse_quantize(coords, feats=None, labels=None, ignore_label=255, return_index=False):
    """`ME.utils.sparse_quantize` (0.4.3) on integer coordinates, rows in ascending (x, y, z) order.  With labels: each voxel's
    first point and its label if all of the voxel's points agree, else `ignore_label` (`quantize_label`)."""
    c = np.asarray(coords).astype(np.int64)
    key = ((c[:, 0] + (1 << 20)) << 42) | ((c[:, 1] + (1 << 20)) << 21) | (c[:, 2] + (1 << 20))
    order = np.argsort(key, kind="stable")
    sk = key[order]
    head = np.ones(len(sk), bool)
    head[1:] = sk[1:] != sk[:-1]
    sel = order[head]
    if labels is None:
        if return_index or feats is None:
            return sel
        return c[sel].astype(np.int32), feats[sel]
    lab = np.asarray(labels)[order].astype(np.int64)
    starts = np.flatnonzero(head)
    lo = np.minimum.reduceat(lab, starts)
    hi = np.maximum.reduceat(lab, starts)
    colabels = np.where(lo == hi, lo, ignore_label).astype(np.int32)
    if return_index:
        return sel, colabels
    if feats is None:
        return c[sel].astype(np.int32), colabels
    return c[sel].astype(np.int32), feats[sel], colabels


# ---------------------------------------------------------------- input transforms (`transforms.py:23-179`)

def dropout(coords, feats, labels, inds):
    """`transforms.py:153-158` with the drawn index set."""
    return coords[inds], feats[inds], labels[inds]


def horizontal_flip(coords, axes):
    """`transforms.py:173-179` for the flipped axes."""
    coords = coords.copy()
    for ax in axes:
        coords[:, ax] = np.max(coords[:, ax]) - coords[:, ax]
    return coords


def auto_contrast(feats, blend_factor):
    """`transforms.py:45-61` (the blend reads `feats`, all columns, as the reference does)."""
    feats = feats.copy()
    lo = feats[:, :3].min(0, keepdims=True)
    hi = feats[:, :3].max(0, keepdims=True)
    assert hi.max() > 1
    scale = 255 / (hi - lo)
    contrast_feats = (feats[:, :3] - lo) * scale
    feats[:, :3] = (1 - blend_factor) * feats + blend_factor * contrast_feats
    return feats


def translation_offset(rand13, trans_range_ratio):
    """`transforms.py:34`: float64 [1, 3] from the `np.random.rand(1, 3)` draw."""
    return (rand13 - 0.5) * 255 * 2 * trans_range_ratio


def translate(feats, tr):
    """`transforms.py:35`."""
    feats = feats.copy()
    feats[:, :3] = np.clip(tr + feats[:, :3], 0, 255)
    return feats


def jitter(feats, randn, std):
    """`transforms.py:71-73` with the drawn standard-normal float64 array `randn` [N, 3]."""
    feats = feats.copy()
    noise = randn.copy()
    noise *= std * 255
    feats[:, :3] = np.clip(noise + feats[:, :3], 0, 255)
    return feats


def label_map(num_labels, ignore_labels, ignore_label=255):
    """`dataset.py:249-260`: a lookup table [max(num_labels, ignore_label + 1)] (unused entries -1)."""
    lut = -np.ones(max(num_labels, ignore_label + 1), np.int64)
    n_used = 0
    for l in range(num_labels):
        if l in ignore_labels:
            lut[l] = ignore_label
        else:
            lut[l] = n_used
            n_used += 1
    lut[ignore_label] = ignore_label
    return lut


def collate(list_data, limit_numpoints):
    """`transforms.py:251-283` (numpy in, numpy out): batch column first, truncation at `limit_numpoints`."""
    C, F, L = [], [], []
    total = 0
    for b, (c, f, l) in enumerate(list_data):
        total += len(c)
        if limit_numpoints and total > limit_numpoints:
            break
        C.append(np.concatenate([np.full((len(c), 1), b, np.int32), c.astype(np.int32)], 1))
        F.append(f)
        L.append(l.astype(np.int32))
    return np.concatenate(C), np.concatenate(F).astype(F32), np.concatenate(L)


# ---------------------------------------------------------------- one scene (`dataset.py:275-309`) with recorded draws

# class constants of the reference's datasets (`lib/datasets/scannet.py:64-82,175-176`, `lib/datasets/stanford.py:19-107`) and the
# colour settings of `config/default.yaml:88-89`
SCANNET_2CM = dict(voxel_size=0.02, clip_bound=None, scale_bound=(0.9, 1.1),
                   rotation_bound=((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi)),
                   translation_ratio_bound=((-0.2, 0.2), (-0.2, 0.2), (0, 0)), elastic=((0.2, 0.4), (0.8, 1.6)), num_labels=41,
                   ignore_labels=tuple(set(range(41)) - {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39}),
                   trans_ratio=0.10, jitter_std=0.05)
STANFORD = dict(voxel_size=0.05, clip_bound=4, scale_bound=(0.9, 1.1),
                rotation_bound=((-np.pi / 32, np.pi / 32), (-np.pi / 32, np.pi / 32), (-np.pi, np.pi)),
                translation_ratio_bound=((-0.2, 0.2), (-0.2, 0.2), (-0.05, 0.05)), elastic=None, num_labels=14, ignore_labels=(10,),
                trans_ratio=0.10, jitter_std=0.05)


class Replay:
    """Hands out a recorded sequence of draws [(kind, value), ...] in order, checking each kind."""

    def __init__(self, record):
        self.record, self.pos = list(record), 0

    def __call__(self, kind):
        k, v = self.record[self.pos]
        assert k == kind, (self.pos, k, kind)
        self.pos += 1
        return v


def read_draws(z, prefix):
    """The draws of one scene of tests/golden/semseg_augment.npz: `<prefix>kinds` and `<prefix>d<i>` (scalars and arrays)."""
    return [(str(k), z[f"{prefix}d{i}"]) for i, k in enumerate(z[f"{prefix}kinds"])]


def run_scene(coords, feats, labels, p, draw, ignore_label=255):
    """The training item of `VoxelizationDataset.__getitem__` (`dataset.py:275-309`) with `augment_data=True` and the transforms of
    `dataset.py:330-351`, every random value taken from `draw(kind)`.  coords float32 [N,3], feats float32 [N,3], labels int [N].
    Returns a dict of the intermediate and final arrays."""
    out = {}
    coords, feats, labels = coords.copy(), feats.copy(), labels.copy()
    if p["elastic"] is not None and float(draw("random")) < 0.95:                        # `transforms.py:219-225`
        for g, m in p["elastic"]:
            coords, blurred = elastic_distortion(coords, g, m, np.asarray(draw("randn")).astype(F32))
    out["elastic"] = coords.copy()
    if p["clip_bound"] is not None:                                                      # `voxelizer.py:115-125`
        ratio = np.array([float(draw("uniform")) for _ in range(3)])
        keep = clip_mask(coords, p["clip_bound"], ratio)
        if keep is not None:
            coords, feats, labels = coords[keep], feats[keep], labels[keep]
    thetas = [float(draw("uniform")) for _ in range(3)]                                  # `voxelizer.py:57-79`
    order = [int(i) for i in draw("shuffle")]
    scale = float(draw("uniform"))
    M_v, M_r = transformation_matrix(p["voxel_size"], thetas, order, scale)
    T = M_r @ M_v
    c, mn, _ = affine_floor(coords, T)
    M_t = np.eye(4)
    M_t[:3, -1] = -mn
    out["transformation"] = (M_t @ T).flatten()
    coords, feats, labels = sparse_quantize(c, feats, labels=labels, ignore_label=ignore_label)
    out["vox_coords"], out["vox_feats"], out["vox_labels"] = coords.copy(), feats.copy(), labels.copy()
    if float(draw("random")) < 0.2:                                                      # RandomDropout(0.2)
        coords, feats, labels = dropout(coords, feats, labels, np.asarray(draw("choice")))
    if float(draw("random")) < 0.95:                                                     # RandomHorizontalFlip('z')
        coords = horizontal_flip(coords, [ax for ax in (0, 1) if float(draw("random")) < 0.5])
    if float(draw("random")) < 0.2:                                                      # ChromaticAutoContrast()
        feats = auto_contrast(feats, float(draw("random")))
    if float(draw("random")) < 0.95:                                                     # ChromaticTranslation(0.1)
        feats = translate(feats, translation_offset(np.asarray(draw("rand")), p["trans_ratio"]))
    if float(draw("random")) < 0.95:                                                     # ChromaticJitter(0.05)
        feats = jitter(feats, np.asarray(draw("randn"), np.float64), p["jitter_std"])
    lut = label_map(p["num_labels"], p["ignore_labels"], ignore_label)
    out["coords"], out["feats"], out["labels"] = coords, feats, lut[labels]
    return out
