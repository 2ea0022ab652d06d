"""Semantic-segmentation finetune data path on the GPU (SURVEY.md 8f-6): a mirror of the reference's training loader
(`downstream/semseg/lib/dataset.py:194-385`, `lib/voxelizer.py`, `lib/transforms.py`) whose per-scene work -- elastic distortion,
rotation / scale / floor, label-aware voxelisation, dropout, flip and the colour augmentation -- runs on libpcb200 instead of one
CPU worker per loader.

    ds = ScannetVoxelization2cmDataset(config, augment_data=True, ...)     # or initialize_data_loader(...) for the reference's wiring
    loader = initialize_data_loader(ScannetVoxelization2cmDataset, config, "train", shuffle=True, augment_data=True, batch_size=6,
                                    limit_numpoints=0, iter_size=2, normalize_color=True)
    trainer.train_step(next(iter(loader)))                                  # `semseg.SegmentationTrainer`

Randomness: scalar decisions (gates, angles, scale, blend factor, translation) come from Python `random` / `np.random` in the
reference's call order; arrays (the elastic noise grid, the jitter noise, the dropout index set) from a `torch.Generator` on the
device.  Both go through a `Draws` object, so a `ReplayDraws` of a recorded sequence reproduces a scene exactly, and every
transform's `apply` also takes its draws as arguments.  `det_data` (the VoteNet detection loader) draws through the same objects.
"""
import ctypes
import logging
import os
import random

import numpy as np
import torch

from . import _lib, voxel
from ._lib import check, lib, ptr, stream, workspace

# ---------------------------------------------------------------------------------------------------------------- PLY

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
              "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4", "float": "<f4", "float32": "<f4", "double": "<f8",
              "float64": "<f8"}


def read_ply(path):
    """The `vertex` element of a binary little-endian PLY file as a numpy structured array (what `PlyData.read(path).elements[0].data`
    gives for the files `lib/pc_utils.py:41-70` writes: x, y, z f4, red, green, blue u1, optionally label u1)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fields, n, fmt, in_vertex, seen_vertex = [], None, None, False, False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: no end_header")
            words = line.decode("ascii").split()
            if not words or words[0] in ("comment", "obj_info"):
                continue
            if words[0] == "end_header":
                break
            if words[0] == "format":
                fmt = words[1]
            elif words[0] == "element":
                in_vertex = words[1] == "vertex"
                if in_vertex:
                    if seen_vertex or fields:
                        raise ValueError(f"{path}: the vertex element must come first")
                    n, seen_vertex = int(words[2]), True
            elif words[0] == "property":
                if words[1] == "list":
                    if in_vertex:
                        raise ValueError(f"{path}: list properties in the vertex element are not supported")
                    continue
                if in_vertex:
                    fields.append((words[2], _PLY_TYPES[words[1]]))
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: format {fmt} (only binary_little_endian is read)")
        if n is None:
            raise ValueError(f"{path}: no vertex element")
        data = np.fromfile(f, dtype=np.dtype(fields), count=n)
    if len(data) != n:
        raise ValueError(f"{path}: {len(data)} of {n} vertices")
    return data


def read_txt(path):
    """`lib/utils.py` `read_txt`: the non-empty lines of a split file."""
    with open(path) as f:
        return [x.strip() for x in f if x.strip()]


# ---------------------------------------------------------------------------------------------------------------- randomness

class Draws:
    """The reference's random sources: `random.random()` and `np.random.*` for scalars on the host, in the reference's call order;
    `generator` (a CUDA `torch.Generator`) for the array draws on the device."""

    def __init__(self, device="cuda", generator=None):
        self.device = torch.device(device)
        self.generator = generator if generator is not None else torch.Generator(device=self.device)

    def random(self):
        return random.random()

    def uniform(self, lo, hi):
        return np.random.uniform(lo, hi)

    def rand(self, *shape):
        return np.random.rand(*shape)

    def shuffle(self, x):
        np.random.shuffle(x)

    def randn(self, shape, dtype):
        return torch.randn(tuple(int(s) for s in shape), generator=self.generator, device=self.device, dtype=dtype)

    def choice(self, n, k):
        """`np.random.choice(n, k, replace=False)`: k distinct indices in random order (int64, device)."""
        return torch.randperm(n, generator=self.generator, device=self.device)[:k]

    def rand_device(self, n):
        """`np.random.random(n)` on the device: fp64 uniform [0, 1) [n]."""
        return torch.rand(int(n), generator=self.generator, device=self.device, dtype=torch.float64)

    def choices(self, ns, k):
        """`np.random.choice(n, k, replace=n < k)` for every scene size n in `ns`, in one call: int64 [len(ns), k] scene-local indices on
        the device.  A scene with n >= k gets a uniformly random ordered k-subset (no repeats), a smaller one k iid indices.  The sets
        come from `pcb_det_choices`, a Philox stream keyed by the generator's seed and offset, which the call advances: equal generator
        states give equal sets."""
        off = np.zeros(len(ns) + 1, np.int64)
        off[1:] = np.cumsum(np.asarray(ns, np.int64))
        if len(ns) == 0 or int(k) < 1 or (np.diff(off) < 1).any():
            raise ValueError(f"choices: every scene needs a point and k >= 1 (sizes {list(ns)}, k {k})")
        seed, offset = self.generator.initial_seed(), self.generator.get_offset()
        self.generator.set_offset(offset + 4)
        out = torch.empty(len(ns), int(k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            d_off = torch.from_numpy(off).to(self.device)
            wsb = lib.pcb_det_choices_ws_bytes(int(off[-1]))
            ws = workspace(wsb, self.device)
            check(lib.pcb_det_choices(off.ctypes.data, ptr(d_off), len(ns), int(k), seed & (2 ** 64 - 1), offset, ptr(out), ptr(ws), wsb,
                                      stream()))
        return out


class ReplayDraws:
    """Replays a recorded sequence of draws [(kind, value), ...] (kinds: random, uniform, rand, shuffle (the permutation), randn,
    choice, rand_device, choices (one index array per scene)), checking that the calls come in the recorded order."""

    def __init__(self, record, device="cuda"):
        self.record, self.pos, self.device = list(record), 0, torch.device(device)

    def _next(self, kind):
        if self.pos >= len(self.record):
            raise IndexError(f"replay: no draw left for {kind}")
        k, v = self.record[self.pos]
        if k != kind:
            raise ValueError(f"replay: draw {self.pos} is {k}, the transform asked for {kind}")
        self.pos += 1
        return v

    def random(self):
        return float(self._next("random"))

    def uniform(self, lo, hi):
        return float(self._next("uniform"))

    def rand(self, *shape):
        v = np.asarray(self._next("rand"), np.float64)
        assert v.shape == shape
        return v

    def shuffle(self, x):
        perm = [int(i) for i in self._next("shuffle")]
        x[:] = [x[i] for i in perm]

    def randn(self, shape, dtype):
        v = torch.as_tensor(np.asarray(self._next("randn")))
        assert tuple(v.shape) == tuple(int(s) for s in shape), (tuple(v.shape), shape)
        return v.to(self.device, dtype)

    def choice(self, n, k):
        v = torch.as_tensor(np.asarray(self._next("choice"), np.int64))
        assert len(v) == k
        return v.to(self.device)

    def rand_device(self, n):
        v = torch.as_tensor(np.asarray(self._next("rand_device"), np.float64))
        assert tuple(v.shape) == (int(n),)
        return v.to(self.device)

    def choices(self, ns, k):
        v = [np.asarray(c, np.int64) for c in self._next("choices")]
        assert len(v) == len(ns) and all(c.shape == (int(k),) for c in v)
        if any(len(c) and (c.min() < 0 or c.max() >= n) for c, n in zip(v, ns)):
            raise ValueError("replay: a recorded choice set is outside its scene")
        return torch.from_numpy(np.stack(v)).to(self.device)


_DEFAULT = {}


def _draws(d):
    if d is not None:
        return d
    dev = torch.cuda.current_device()
    if dev not in _DEFAULT:
        _DEFAULT[dev] = Draws(torch.device("cuda", dev))
    return _DEFAULT[dev]


# ---------------------------------------------------------------------------------------------------------------- kernels

def point_bounds(xyz):
    """Per-axis (min, max) of float32 CUDA points [N,3], N >= 1, as numpy float32 [3] arrays (synchronises)."""
    _lib.require_cuda(xyz)
    xyz = xyz.contiguous()
    lo, hi = (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_point_bounds_ws_bytes()
        ws = workspace(wsb, xyz.device)
        check(lib.pcb_point_bounds(ptr(xyz), xyz.shape[0], lo, hi, ptr(ws), wsb, stream()))
    return np.array(lo[:], np.float32), np.array(hi[:], np.float32)


def elastic_distort(xyz, noise, axes, magnitude):
    """In place: blur `noise` (float32 CUDA [gx,gy,gz,3]) with the two rounds of box filters, then xyz += interp(xyz) * magnitude.
    axes: three float64 numpy arrays (the grid positions)."""
    _lib.require_cuda(xyz); _lib.require_cuda(noise)
    assert xyz.dtype == torch.float32 and xyz.is_contiguous() and noise.dtype == torch.float32 and noise.is_contiguous()
    gx, gy, gz = (int(s) for s in noise.shape[:3])
    assert tuple(noise.shape) == (gx, gy, gz, 3) and [len(a) for a in axes] == [gx, gy, gz]
    ax = torch.from_numpy(np.concatenate([np.asarray(a, np.float64) for a in axes])).to(xyz.device)
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_elastic_distort_ws_bytes(gx, gy, gz)
        ws = workspace(wsb, xyz.device)
        check(lib.pcb_elastic_distort(ptr(xyz), xyz.shape[0], ptr(noise), gx, gy, gz, ptr(ax), float(magnitude), ptr(ws), wsb, stream()))
    return xyz


def affine_floor(xyz, T):
    """(floor(homo(xyz) @ T[:3].T) - its per-axis minimum as int32 CUDA [N,3], the minimum as numpy int64 [3]); T: float64 4x4."""
    _lib.require_cuda(xyz)
    xyz = xyz.contiguous()
    assert xyz.dtype == torch.float32
    Tc = np.ascontiguousarray(T, np.float64).reshape(16)
    out = torch.empty(xyz.shape[0], 3, dtype=torch.int32, device=xyz.device)
    mn = (ctypes.c_int32 * 3)()
    with torch.cuda.device(xyz.device):
        wsb = lib.pcb_affine_floor_ws_bytes()
        ws = workspace(wsb, xyz.device)
        check(lib.pcb_affine_floor(ptr(xyz), xyz.shape[0], Tc.ctypes.data, ptr(out), mn, ptr(ws), wsb, stream()))
    return out, np.array(mn[:], np.int64)


def voxelize_labels(coords, labels, ignore_label):
    """int32 CUDA coords [N,3] + labels [N] -> (voxel coords int32 [M,3] in (x,y,z) order, sel int64 [M] (first point), labels int32 [M]:
    the voxel's common label, else ignore_label)."""
    _lib.require_cuda(coords)
    coords = coords.contiguous().int()
    labels = labels.to(coords.device).contiguous().int()
    n = coords.shape[0]
    out = torch.empty(n, 3, dtype=torch.int32, device=coords.device)
    sel = torch.empty(n, dtype=torch.int32, device=coords.device)
    lab = torch.empty(n, dtype=torch.int32, device=coords.device)
    m = ctypes.c_int64(0)
    with torch.cuda.device(coords.device):
        wsb = lib.pcb_voxelize_labels_ws_bytes(n)
        ws = workspace(wsb, coords.device)
        check(lib.pcb_voxelize_labels(ptr(coords), ptr(labels), n, int(ignore_label), ptr(out), ptr(sel), ptr(lab), ctypes.byref(m), ptr(ws),
                                      wsb, stream()))
    return out[:m.value], sel[:m.value].long(), lab[:m.value]


def input_transform(coords, feats, flip_mask=0, contrast=False, blend=0.0, translation=None, jitter_noise=None, jitter_scale=0.0,
                    normalize=False):
    """In place, one pass: flip (bit k of flip_mask: axis k) -> auto-contrast (blend factor `blend`) -> colour translation (float64 [3]) ->
    colour jitter (standard-normal float64 CUDA [N,3] times `jitter_scale`) -> optional colour / 255 - 0.5.  coords may be None when
    nothing is flipped."""
    _lib.require_cuda(feats)
    assert feats.dtype == torch.float32 and feats.is_contiguous() and feats.shape[1] == 3
    assert (coords is None and not flip_mask) or (coords.dtype == torch.int32 and coords.is_contiguous() and coords.shape == feats.shape)
    n = feats.shape[0]
    if n == 0:
        return coords, feats
    tr = None
    if translation is not None:
        tr = (ctypes.c_double * 3)(*[float(v) for v in np.asarray(translation, np.float64).reshape(3)])
    if jitter_noise is not None:
        assert jitter_noise.dtype == torch.float64 and tuple(jitter_noise.shape) == (n, 3)
        jitter_noise = jitter_noise.contiguous()
    with torch.cuda.device(feats.device):
        wsb = lib.pcb_semseg_input_transform_ws_bytes()
        ws = workspace(wsb, feats.device)
        check(lib.pcb_semseg_input_transform(ptr(coords), ptr(feats), n, int(flip_mask), int(bool(contrast)), float(blend), tr, ptr(jitter_noise),
                                             float(jitter_scale), int(bool(normalize)), ptr(ws), wsb, stream()))
    return coords, feats


# ---------------------------------------------------------------------------------------------------------------- transforms

class _InputTransform:
    """A transform of the one-pass input kernel: `draw(n)` returns its kernel arguments; `Compose` fuses consecutive ones."""

    def draw(self, n):
        raise NotImplementedError

    def apply(self, coords, feats, labels, **args):
        input_transform(coords, feats, **args)
        return coords, feats, labels

    def __call__(self, coords, feats, labels):
        return self.apply(coords, feats, labels, **self.draw(len(coords)))


class ChromaticTranslation(_InputTransform):
    """`transforms.py:23-36`."""

    def __init__(self, trans_range_ratio=1e-1, draws=None):
        self.trans_range_ratio, self.draws = trans_range_ratio, draws

    def draw(self, n):
        d = _draws(self.draws)
        if d.random() < 0.95:
            return {"translation": ((d.rand(1, 3) - 0.5) * 255 * 2 * self.trans_range_ratio)[0]}
        return {}


class ChromaticAutoContrast(_InputTransform):
    """`transforms.py:39-61`."""

    def __init__(self, randomize_blend_factor=True, blend_factor=0.5, draws=None):
        self.randomize_blend_factor, self.blend_factor, self.draws = randomize_blend_factor, blend_factor, draws

    def draw(self, n):
        d = _draws(self.draws)
        if d.random() < 0.2:
            return {"contrast": True, "blend": d.random() if self.randomize_blend_factor else self.blend_factor}
        return {}


class ChromaticJitter(_InputTransform):
    """`transforms.py:64-74`."""

    def __init__(self, std=0.01, draws=None):
        self.std, self.draws = std, draws

    def draw(self, n):
        d = _draws(self.draws)
        if d.random() < 0.95:
            return {"jitter_noise": d.randn((n, 3), torch.float64), "jitter_scale": self.std * 255}
        return {}


class RandomHorizontalFlip(_InputTransform):
    """`transforms.py:161-179` (3-D coordinates)."""

    def __init__(self, upright_axis, is_temporal, draws=None):
        if is_temporal:
            raise NotImplementedError("temporal (4-D) coordinates are not supported")
        self.is_temporal, self.D, self.draws = is_temporal, 3, draws
        self.upright_axis = {"x": 0, "y": 1, "z": 2}[upright_axis.lower()]
        self.horz_axes = set(range(self.D)) - set([self.upright_axis])

    def draw(self, n):
        d = _draws(self.draws)
        mask = 0
        if d.random() < 0.95:
            for ax in self.horz_axes:
                if d.random() < 0.5:
                    mask |= 1 << ax
        return {"flip_mask": mask} if mask else {}


class RandomDropout:
    """`transforms.py:144-158`: a row gather with the drawn index set."""

    def __init__(self, dropout_ratio=0.2, dropout_application_ratio=0.5, draws=None):
        self.dropout_ratio, self.dropout_application_ratio, self.draws = dropout_ratio, dropout_application_ratio, draws

    def apply(self, coords, feats, labels, inds):
        return coords[inds].contiguous(), feats[inds].contiguous(), labels[inds].contiguous()

    def __call__(self, coords, feats, labels):
        d = _draws(self.draws)
        if d.random() < self.dropout_ratio:
            N = len(coords)
            return self.apply(coords, feats, labels, d.choice(N, int(N * (1 - self.dropout_ratio))))
        return coords, feats, labels


class ElasticDistortion:
    """`transforms.py:182-225` on float32 CUDA points (in place, as the reference)."""

    def __init__(self, distortion_params, draws=None):
        self.distortion_params, self.draws = distortion_params, draws

    @staticmethod
    def grid(coords, granularity):
        """The noise grid's shape and float64 axes (`transforms.py:197-200,210-214`) from the points' float32 bounds."""
        coords_min, coords_max = point_bounds(coords)
        noise_dim = ((coords_max - coords_min) // granularity).astype(int) + 3       # == (coords - coords_min).max(0) // granularity
        axes = [np.linspace(d_min, d_max, d) for d_min, d_max, d in
                zip(coords_min - granularity, coords_min + granularity * (noise_dim - 2), noise_dim)]
        return noise_dim, axes

    def elastic_distortion(self, coords, feats, labels, granularity, magnitude, noise=None):
        """noise: the float32 CUDA grid [*noise_dim, 3] (drawn when None); on return it holds the blurred grid."""
        noise_dim, axes = self.grid(coords, granularity)
        if noise is None:
            noise = _draws(self.draws).randn((*noise_dim, 3), torch.float32)
        elastic_distort(coords, noise, axes, magnitude)
        return coords, feats, labels

    def __call__(self, coords, feats, labels):
        if self.distortion_params is not None:
            if _draws(self.draws).random() < 0.95:
                for granularity, magnitude in self.distortion_params:
                    coords, feats, labels = self.elastic_distortion(coords, feats, labels, granularity, magnitude)
        return coords, feats, labels


class Compose:
    """`transforms.py:228-237`; consecutive flip / colour transforms run as one pass of the input kernel (their draws are taken
    in order first: none of them depends on the data the others change)."""

    def __init__(self, transforms):
        self.transforms = transforms

    def __call__(self, *args):
        pending = {}
        for t in self.transforms:
            if isinstance(t, _InputTransform):
                d = t.draw(len(args[0]))
                if pending.keys() & d.keys():
                    input_transform(args[0], args[1], **pending)
                    pending = {}
                pending.update(d)
                continue
            if pending:
                input_transform(args[0], args[1], **pending)
                pending = {}
            args = t(*args)
        if pending:
            input_transform(args[0], args[1], **pending)
        return args


# ---------------------------------------------------------------------------------------------------------------- voxelizer

def M(axis, theta):
    """`voxelizer.py:14-15`: rotation by `theta` about `axis`."""
    from scipy.linalg import expm, norm
    return expm(np.cross(np.eye(3), axis / norm(axis) * theta))


class Voxelizer:
    """`voxelizer.py:18-148` on CUDA tensors.  `voxelize` returns (coords int32 [M,3] in ascending (x,y,z) order, feats [M,3],
    labels int32 [M], the flattened float64 transformation)."""

    def __init__(self, voxel_size=1, clip_bound=None, use_augmentation=False, scale_augmentation_bound=None, rotation_augmentation_bound=None,
                 translation_augmentation_ratio_bound=None, ignore_label=255, draws=None):
        self.voxel_size, self.clip_bound, self.ignore_label = voxel_size, clip_bound, ignore_label
        self.use_augmentation = use_augmentation
        self.scale_augmentation_bound = scale_augmentation_bound
        self.rotation_augmentation_bound = rotation_augmentation_bound
        self.translation_augmentation_ratio_bound = translation_augmentation_ratio_bound
        self.draws = draws

    def get_transformation_matrix(self):
        d = _draws(self.draws)
        voxelization_matrix, rotation_matrix = np.eye(4), np.eye(4)
        rot_mat = np.eye(3)
        if self.use_augmentation and self.rotation_augmentation_bound is not None:
            rot_mats = []
            for axis_ind, rot_bound in enumerate(self.rotation_augmentation_bound):
                theta = 0
                axis = np.zeros(3)
                axis[axis_ind] = 1
                if rot_bound is not None:
                    theta = d.uniform(*rot_bound)
                rot_mats.append(M(axis, theta))
            d.shuffle(rot_mats)
            rot_mat = rot_mats[0] @ rot_mats[1] @ rot_mats[2]
        rotation_matrix[:3, :3] = rot_mat
        scale = 1 / self.voxel_size
        if self.use_augmentation and self.scale_augmentation_bound is not None:
            scale *= d.uniform(*self.scale_augmentation_bound)
        np.fill_diagonal(voxelization_matrix[:3, :3], scale)
        return voxelization_matrix, rotation_matrix

    def clip(self, coords, center=None, trans_aug_ratio=None):
        """`voxelizer.py:81-111` for a scalar bound: a boolean CUDA mask, or None when the scene is smaller than the bound."""
        if not isinstance(self.clip_bound, (int, float)):
            raise NotImplementedError("only a scalar clip bound is supported")
        lo, hi = point_bounds(coords)
        bound_min, bound_max = lo.astype(float), hi.astype(float)
        bound_size = bound_max - bound_min
        if center is None:
            center = bound_min + bound_size * 0.5
        if trans_aug_ratio is not None:
            center += np.multiply(trans_aug_ratio, bound_size)
        lim = self.clip_bound
        if bound_size.max() < lim:
            return None
        c = coords.double()                 # float32 points against float64 bounds: compared in float64
        mask = torch.ones(len(c), dtype=torch.bool, device=c.device)
        for k in range(3):
            mask &= (c[:, k] >= float(-lim + center[k])) & (c[:, k] < float(lim + center[k]))
        return mask

    def voxelize(self, coords, feats, labels, center=None):
        assert coords.shape[1] == 3 and coords.shape[0] == feats.shape[0] and coords.shape[0]
        if labels is None:
            raise ValueError("Voxelizer.voxelize needs labels")
        if self.clip_bound is not None:
            trans_aug_ratio = np.zeros(3)
            if self.use_augmentation and self.translation_augmentation_ratio_bound is not None:
                for axis_ind, trans_ratio_bound in enumerate(self.translation_augmentation_ratio_bound):
                    trans_aug_ratio[axis_ind] = _draws(self.draws).uniform(*trans_ratio_bound)
            clip_inds = self.clip(coords, center, trans_aug_ratio)
            if clip_inds is not None:
                coords, feats, labels = coords[clip_inds].contiguous(), feats[clip_inds], labels[clip_inds]
        M_v, M_r = self.get_transformation_matrix()
        rigid_transformation = M_v
        if self.use_augmentation:
            rigid_transformation = M_r @ rigid_transformation
        coords_aug, min_coords = affine_floor(coords, rigid_transformation)
        M_t = np.eye(4)
        M_t[:3, -1] = -min_coords
        rigid_transformation = M_t @ rigid_transformation
        vc, sel, vl = voxelize_labels(coords_aug, labels, self.ignore_label)
        return vc, feats[sel].contiguous(), vl, rigid_transformation.flatten()


# ---------------------------------------------------------------------------------------------------------------- datasets

class VoxelizationDataset:
    """`dataset.py:144-308`: PLY scenes -> prevoxel transform -> voxelizer -> input transform -> label map, on `device`.
    Items are (coords int32 [M,3], feats float32 [M,3], labels int32 [M]) CUDA tensors (+ the float32 transformation)."""
    IS_TEMPORAL = False
    CLIP_BOUND = (-1000, -1000, -1000, 1000, 1000, 1000)
    ROTATION_AXIS = None
    NUM_IN_CHANNEL = None
    NUM_LABELS = -1
    IGNORE_LABELS = None
    VOXEL_SIZE = 0.05
    SCALE_AUGMENTATION_BOUND = (0.9, 1.1)
    ROTATION_AUGMENTATION_BOUND = ((-np.pi / 6, np.pi / 6), (-np.pi, np.pi), (-np.pi / 6, np.pi / 6))
    TRANSLATION_AUGMENTATION_RATIO_BOUND = ((-0.2, 0.2), (-0.05, 0.05), (-0.2, 0.2))
    ELASTIC_DISTORT_PARAMS = None
    PREVOXELIZATION_VOXEL_SIZE = None
    AUGMENT_COORDS_TO_FEATS = False

    def __init__(self, data_paths, prevoxel_transform=None, input_transform=None, target_transform=None, data_root="/", ignore_label=255,
                 return_transformation=False, augment_data=False, config=None, device="cuda", draws=None, **kwargs):
        if self.AUGMENT_COORDS_TO_FEATS:
            raise NotImplementedError("AUGMENT_COORDS_TO_FEATS")
        self.augment_data, self.config = augment_data, config
        self.data_root = str(data_root)
        self.data_paths = sorted(data_paths)
        self.prevoxel_transform, self.input_transform, self.target_transform = prevoxel_transform, input_transform, target_transform
        self.ignore_mask = ignore_label
        self.return_transformation = return_transformation
        self.device = torch.device(device)
        self.voxelizer = Voxelizer(voxel_size=self.VOXEL_SIZE, clip_bound=self.CLIP_BOUND, use_augmentation=augment_data,
                                   scale_augmentation_bound=self.SCALE_AUGMENTATION_BOUND, rotation_augmentation_bound=self.ROTATION_AUGMENTATION_BOUND,
                                   translation_augmentation_ratio_bound=self.TRANSLATION_AUGMENTATION_RATIO_BOUND, ignore_label=ignore_label,
                                   draws=draws)
        label_map = {}
        n_used = 0
        for l in range(self.NUM_LABELS):
            if l in self.IGNORE_LABELS:
                label_map[l] = self.ignore_mask
            else:
                label_map[l] = n_used
                n_used += 1
        label_map[self.ignore_mask] = self.ignore_mask
        self.label_map = label_map
        self.NUM_LABELS -= len(self.IGNORE_LABELS)
        lut = np.full(max(label_map) + 1, -1, np.int32)
        for k, v in label_map.items():
            lut[k] = v
        self._lut = torch.from_numpy(lut).to(self.device)

    def load_ply(self, index):
        """`dataset.py:180-187`: float32 xyz, float32 rgb, int32 labels (numpy).  A scene without a `label` property (the ScanNet
        test split) gets the ignore label everywhere."""
        data = read_ply(os.path.join(self.data_root, self.data_paths[index]))
        coords = np.array([data["x"], data["y"], data["z"]], dtype=np.float32).T
        feats = np.array([data["red"], data["green"], data["blue"]], dtype=np.float32).T
        if "label" in data.dtype.names:
            labels = np.array(data["label"], dtype=np.int32)
        else:
            labels = np.full(len(data), self.ignore_mask, np.int32)
        return coords, feats, labels, None

    def map_labels(self, labels):
        """`dataset.py:297-298` through a lookup table on the device."""
        if len(labels) and (int(labels.min()) < 0 or int(labels.max()) >= len(self._lut)):
            raise KeyError("label outside the dataset's label map")
        out = self._lut[labels.long()]
        if len(out) and int(out.min()) < 0:
            raise KeyError("label outside the dataset's label map")
        return out

    def __getitem__(self, index):
        coords, feats, labels, center = self.load_ply(index)
        coords, feats, labels = (torch.from_numpy(np.ascontiguousarray(a)).to(self.device) for a in (coords, feats, labels))
        if self.PREVOXELIZATION_VOXEL_SIZE is not None:
            _, inds = voxel.voxelize(coords, self.PREVOXELIZATION_VOXEL_SIZE)
            coords, feats, labels = coords[inds].contiguous(), feats[inds], labels[inds]
        if self.prevoxel_transform is not None:
            coords, feats, labels = self.prevoxel_transform(coords, feats, labels)
        coords, feats, labels, transformation = self.voxelizer.voxelize(coords, feats, labels, center=center)
        if self.input_transform is not None:
            coords, feats, labels = self.input_transform(coords, feats, labels)
        if self.target_transform is not None:
            coords, feats, labels = self.target_transform(coords, feats, labels)
        if self.IGNORE_LABELS is not None:
            labels = self.map_labels(labels)
        out = [coords, feats, labels]
        if self.return_transformation:
            out.append(transformation.astype(np.float32))
        return tuple(out)

    def __len__(self):
        return len(self.data_paths)


# `lib/datasets/scannet.py:20-21`
VALID_CLASS_IDS = (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39)
_PHASES = {"train": "Train", "val": "Val", "trainval": "TrainVal", "test": "Test"}


class ScannetVoxelizationDataset(VoxelizationDataset):
    """`lib/datasets/scannet.py:64-117`.  The split file is read from `split_dir` (the reference: `./splits/scannet`)."""
    CLIP_BOUND = None
    TEST_CLIP_BOUND = None
    VOXEL_SIZE = 0.05
    ROTATION_AUGMENTATION_BOUND = ((-np.pi / 64, np.pi / 64), (-np.pi / 64, np.pi / 64), (-np.pi, np.pi))
    TRANSLATION_AUGMENTATION_RATIO_BOUND = ((-0.2, 0.2), (-0.2, 0.2), (0, 0))
    ELASTIC_DISTORT_PARAMS = ((0.2, 0.4), (0.8, 1.6))
    ROTATION_AXIS = "z"
    LOCFEAT_IDX = 2
    NUM_LABELS = 41
    IGNORE_LABELS = tuple(set(range(41)) - set(VALID_CLASS_IDS))
    IS_FULL_POINTCLOUD_EVAL = True
    DATA_PATH_FILE = {"Train": "scannetv2_train.txt", "Val": "scannetv2_val.txt", "TrainVal": "scannetv2_trainval.txt",
                      "Test": "scannetv2_test.txt"}

    def __init__(self, config, prevoxel_transform=None, input_transform=None, target_transform=None, augment_data=True,
                 elastic_distortion=False, cache=False, phase="train", split_dir="./splits/scannet", device="cuda", draws=None):
        phase = _PHASES[phase.lower()]
        if phase not in ("Train", "TrainVal"):
            self.CLIP_BOUND = self.TEST_CLIP_BOUND
        data_paths = read_txt(os.path.join(split_dir, self.DATA_PATH_FILE[phase]))
        logging.info("Loading {}: {}".format(self.__class__.__name__, self.DATA_PATH_FILE[phase]))
        super().__init__(data_paths, data_root=config.data.scannet_path, prevoxel_transform=prevoxel_transform, input_transform=input_transform,
                         target_transform=target_transform, ignore_label=config.data.ignore_label,
                         return_transformation=config.data.return_transformation, augment_data=augment_data, config=config, device=device,
                         draws=draws)


class ScannetVoxelization2cmDataset(ScannetVoxelizationDataset):
    """`lib/datasets/scannet.py:175-176`."""
    VOXEL_SIZE = 0.02


class StanfordDataset(VoxelizationDataset):
    """`lib/datasets/stanford.py:19-162` (S3DIS, 5 cm, clipped to 8 m cubes).  Split files under `<stanford3d_path>/splits/`."""
    CLIP_SIZE = None
    LOCFEAT_IDX = 2
    ROTATION_AXIS = "z"
    NUM_LABELS = 14
    IGNORE_LABELS = (10,)
    IS_FULL_POINTCLOUD_EVAL = True
    DATA_PATH_FILE = {"Train": "train.txt", "Val": "val.txt", "TrainVal": "trainval.txt", "Test": "test.txt"}
    VOXEL_SIZE = 0.05
    CLIP_BOUND = 4
    TEST_CLIP_BOUND = None
    ROTATION_AUGMENTATION_BOUND = ((-np.pi / 32, np.pi / 32), (-np.pi / 32, np.pi / 32), (-np.pi, np.pi))
    TRANSLATION_AUGMENTATION_RATIO_BOUND = ((-0.2, 0.2), (-0.2, 0.2), (-0.05, 0.05))
    AUGMENT_COORDS_TO_FEATS = False
    NUM_IN_CHANNEL = 3

    def __init__(self, config, prevoxel_transform=None, input_transform=None, target_transform=None, cache=False, augment_data=True,
                 elastic_distortion=False, phase="train", device="cuda", draws=None):
        phase = _PHASES[phase.lower()]
        if phase not in ("Train", "TrainVal"):
            self.CLIP_BOUND = self.TEST_CLIP_BOUND
        data_root = config.data.stanford3d_path
        files = self.DATA_PATH_FILE[phase]
        data_paths = []
        for split in (files if isinstance(files, (list, tuple)) else [files]):
            data_paths += read_txt(os.path.join(data_root, "splits", split))
        if config.data.get("voxel_size"):
            self.VOXEL_SIZE = config.data.voxel_size
        super().__init__(data_paths, data_root=data_root, prevoxel_transform=prevoxel_transform, input_transform=input_transform,
                         target_transform=target_transform, ignore_label=config.data.ignore_label,
                         return_transformation=config.data.return_transformation, augment_data=augment_data, config=config, device=device,
                         draws=draws)



class StanfordArea5Dataset(StanfordDataset):
    """`lib/datasets/stanford.py:165-171`: Areas 1-4 and 6 train, Area 5 is validation and test (no TrainVal split), from the split files
    `semseg_prep.generate_splits` writes."""
    DATA_PATH_FILE = {"Train": ["area1.txt", "area2.txt", "area3.txt", "area4.txt", "area6.txt"], "Val": "area5.txt", "Test": "area5.txt"}


class StanfordArea53cmDataset(StanfordArea5Dataset):
    """`lib/datasets/stanford.py:174-176`."""
    CLIP_BOUND = 3.2
    VOXEL_SIZE = 0.03


class StanfordArea57d5cmDataset(StanfordArea5Dataset):
    """`lib/datasets/stanford.py:179-180`."""
    VOXEL_SIZE = 0.075


class StanfordArea510cmDataset(StanfordArea5Dataset):
    """`lib/datasets/stanford.py:183-184`."""
    VOXEL_SIZE = 0.1

# ---------------------------------------------------------------------------------------------------------------- collate / loader

class cfl_collate_fn_factory:
    """`transforms.py:240-283` on CUDA tensors: batch column first, the batch truncated before the scene that would exceed
    `limit_numpoints` (0 / False: no limit)."""

    def __init__(self, limit_numpoints):
        self.limit_numpoints = limit_numpoints

    def __call__(self, list_data):
        coords, feats, labels = list(zip(*list_data))[:3]
        coords_batch, feats_batch, labels_batch = [], [], []
        batch_num_points = 0
        for batch_id, _ in enumerate(coords):
            num_points = coords[batch_id].shape[0]
            batch_num_points += num_points
            if self.limit_numpoints and batch_num_points > self.limit_numpoints:
                num_full_points = sum(len(c) for c in coords)
                logging.warning(f"\t\tCannot fit {num_full_points} points into {self.limit_numpoints} points limit. Truncating batch size at "
                                f"{batch_id} out of {len(coords)} with {batch_num_points - num_points}.")
                break
            c = coords[batch_id]
            coords_batch.append(torch.cat((torch.full((num_points, 1), batch_id, dtype=torch.int32, device=c.device), c.int()), 1))
            feats_batch.append(feats[batch_id])
            labels_batch.append(labels[batch_id].int())
        return torch.cat(coords_batch, 0).int(), torch.cat(feats_batch, 0).float(), torch.cat(labels_batch, 0).int()


class cflt_collate_fn_factory:
    """`transforms.py:286-316`: the `cfl` collate plus the items' transformations as float32 CPU rows [B, 17] -- the 16 entries of the
    4x4, then the batch index -- for the scenes the `limit_numpoints` truncation keeps.  (The reference concatenates a 1-D matrix with
    a 2-D column and an empty point-cloud list; this is what it means to build, DESIGN.md section 5.)"""

    def __init__(self, limit_numpoints):
        self.limit_numpoints = limit_numpoints

    def __call__(self, list_data):
        coords, feats, labels, transformations = list(zip(*list_data))[:4]
        coords_batch, feats_batch, labels_batch = cfl_collate_fn_factory(self.limit_numpoints)(list(zip(coords, feats, labels)))
        kept, total = len(coords), 0
        for b, c in enumerate(coords):               # the scenes cfl keeps: those before the one that would exceed the limit
            total += len(c)
            if self.limit_numpoints and total > self.limit_numpoints:
                kept = b
                break
        rows = [np.concatenate([np.asarray(t, np.float32).reshape(16), np.float32([b])]) for b, t in enumerate(transformations[:kept])]
        return coords_batch, feats_batch, labels_batch, torch.from_numpy(np.stack(rows).astype(np.float32))


def _rank_world(rank, world):
    from .trainer import get_rank, get_world_size
    rank = get_rank() if rank is None else int(rank)
    world = get_world_size() if world is None else int(world)
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"rank {rank} of world {world}")
    return rank, world


class VoxelizationLoader:
    """The training loader (`dataset.py:311-385` with `repeat=True`): endless; each item is a list of `iter_size` collated sub-batches
    (coords, feats, target) -- what `semseg.SegmentationTrainer.train_step` takes.  `normalize_color` applies `lib/train.py:114`
    (colour / 255 - 0.5) to each sub-batch.

    Data parallel (`dataset.py:374-376`): rank `rank` of `world` (default: torch.distributed's, else 0 of 1) takes every world-th
    entry of the shared endless permutation, `batch_size` scenes per sub-batch on each rank (the global batch is batch_size * world),
    `ceil(n / world) // batch_size` items per epoch.  `seed`: the permutations come from their own generator (`shared_randperm`),
    which the ranks need to draw the same ones; None draws them from the global torch RNG."""

    def __init__(self, dataset, batch_size, collate_fn, iter_size=1, shuffle=True, normalize_color=False, rank=None, world=None, seed=None):
        from .scannet_pairs import DistributedInfSampler
        self.dataset, self.batch_size, self.collate_fn = dataset, batch_size, collate_fn
        self.iter_size, self.normalize_color = iter_size, normalize_color
        self.rank, self.world = _rank_world(rank, world)
        if self.world > 1 and shuffle and seed is None:
            raise ValueError("a shuffled loader on several ranks needs a seed shared by the ranks")
        self.sampler = DistributedInfSampler(len(dataset), self.world, self.rank, shuffle, seed=seed)

    def __len__(self):
        return len(self.sampler) // self.batch_size

    def _sub_batch(self):
        coords, feats, target = self.collate_fn([self.dataset[next(self.sampler)] for _ in range(self.batch_size)])
        if self.normalize_color:
            input_transform(None, feats, normalize=True)
        return coords, feats, target

    def __iter__(self):
        while True:
            yield [self._sub_batch() for _ in range(self.iter_size)]


class VoxelizationPassLoader:
    """The evaluation loader (`dataset.py:311-385` with `repeat=False`): one pass over the dataset in sampler order (a fresh permutation
    per pass when `shuffle`), `ceil(n / batch_size)` items, the last one possibly short.  Each item is one collated (coords, feats,
    target), colours normalised once when `normalize_color` -- what `semseg.test` takes.  With `cflt_collate_fn_factory` the items are
    (coords, feats, target, transformation).

    Sharded (`rank` / `world`, default 0 of 1): rank r gets batches b = r, r + world, ... of the batch sequence one process makes --
    the same order and batch composition, so the per-batch AP means are the same numbers -- possibly none.  `seed`: each pass's
    permutation comes from its own generator (`shared_randperm`, seeded by (seed, pass count)), which shuffled shards need; None
    draws it from the global torch RNG."""

    def __init__(self, dataset, batch_size, collate_fn, shuffle=False, normalize_color=False, rank=0, world=1, seed=None):
        self.dataset, self.batch_size, self.collate_fn = dataset, batch_size, collate_fn
        self.shuffle, self.normalize_color = shuffle, normalize_color
        self.rank, self.world = _rank_world(rank, world)
        if self.world > 1 and shuffle and seed is None:
            raise ValueError("a shuffled sharded pass needs a seed shared by the ranks")
        self.seed, self.passes = seed, 0

    def num_batches(self):
        """The number of batches of the whole pass (all ranks)."""
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def __len__(self):
        return len(range(self.rank, self.num_batches(), self.world))

    def __iter__(self):
        from .scannet_pairs import shared_randperm
        order = shared_randperm(len(self.dataset), self.seed, self.passes).tolist() if self.shuffle else list(range(len(self.dataset)))
        self.passes += 1
        for b in range(self.rank, self.num_batches(), self.world):
            item = self.collate_fn([self.dataset[i] for i in order[b * self.batch_size:(b + 1) * self.batch_size]])
            if self.normalize_color:
                input_transform(None, item[1], normalize=True)
            yield tuple(item)


def initialize_data_loader(DatasetClass, config, phase, shuffle, augment_data, batch_size, limit_numpoints, iter_size=1, normalize_color=True,
                           input_transform=None, target_transform=None, device="cuda", draws=None, repeat=True, rank=None, world=None,
                           **dataset_kwargs):
    """`dataset.py:311-385`: elastic distortion before voxelisation, then dropout, flip, auto-contrast, colour translation and jitter
    (`config.augmentation.data_aug_color_trans_ratio` / `data_aug_color_jitter_std`).  `repeat=True`: the endless training loader;
    `repeat=False`: one pass (`VoxelizationPassLoader`, `iter_size` unused), whose items carry the transformations
    (`cflt_collate_fn_factory`) when `config.data.return_transformation` is set.

    `rank` / `world`: the training loader's shard (default: torch.distributed's); the pass loader is sharded only when they are given.
    On several ranks the permutations come from a generator seeded by `config.misc.seed`; on one, from the global torch RNG."""
    prevoxel = [ElasticDistortion(DatasetClass.ELASTIC_DISTORT_PARAMS, draws=draws)] if augment_data else []
    transforms = list(input_transform or [])
    if augment_data:
        transforms += [RandomDropout(0.2, draws=draws), RandomHorizontalFlip(DatasetClass.ROTATION_AXIS, DatasetClass.IS_TEMPORAL, draws=draws),
                       ChromaticAutoContrast(draws=draws), ChromaticTranslation(config.augmentation.data_aug_color_trans_ratio, draws=draws),
                       ChromaticJitter(config.augmentation.data_aug_color_jitter_std, draws=draws)]
    dataset = DatasetClass(config, prevoxel_transform=Compose(prevoxel) if prevoxel else None,
                           input_transform=Compose(transforms) if transforms else None, target_transform=target_transform,
                           augment_data=augment_data, phase=phase, device=device, draws=draws, **dataset_kwargs)
    if not repeat:
        collate = cflt_collate_fn_factory if config.data.get("return_transformation") else cfl_collate_fn_factory
        rank, world = _rank_world(rank or 0, world or 1)
        return VoxelizationPassLoader(dataset, batch_size, collate(limit_numpoints), shuffle=shuffle, normalize_color=normalize_color,
                                      rank=rank, world=world, seed=config.misc.seed if world > 1 else None)
    rank, world = _rank_world(rank, world)
    return VoxelizationLoader(dataset, batch_size, cfl_collate_fn_factory(limit_numpoints), iter_size=iter_size, shuffle=shuffle,
                              normalize_color=normalize_color, rank=rank, world=world, seed=config.misc.seed if world > 1 else None)
