"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the MinkowskiEngine operator surface.

A CPU restatement (numpy for the integer coordinate work, torch CPU tensors + autograd for the
floating-point work) of the MinkowskiEngine v0.4.3 semantics that PointContrast's hot path
exercises (the original repository's `README.md:24,34` pins the version; the library itself is not part of that
repository, and not installable offline -- SURVEY.md section 8c).

PARITY UNPINNED at the ME boundary: the reference holds no golden vectors for this path and
MinkowskiEngine cannot be run here.  What *is* pinned (tests/test_oracle_*.py):
  * the operator (stride-1 k3, stride-2 k2, transposed k2 s2) against dense
    torch.nn.functional.conv3d / conv_transpose3d in fp64;
  * the model wiring, by running the reference's own `model/res16unet.py` on top of this module;
  * the hardest-contrastive loss, by running the reference's own function (`lib/ddp_trainer.py:186-238`).
Residual unpinned items: the weight-index <-> kernel-offset enumeration order (single tables below)
and the default parameter init.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.  The product path (pointcontrast_b200/) never does.

Semantics restated (numbers refer to SURVEY.md section 8c):
 (1) coords int32 [b, x, y, z], batch first   (`lib/ddp_data_loaders.py:68-70`)
 (2) stride: floor(c / (s*ts)) * (s*ts), true floor on negatives
 (3) odd kernel: offsets centred; even kernel: offsets {0..k-1} * ts
 (4) stride-1 conv output coords == input coords
 (5) correlation: Y[u] = sum_k W[k]^T X[u + o_k]
 (6) HYPERCUBE enumeration: first spatial axis fastest
 (7) HYBRID with all-HYPERCUBE axes: origin first, then axis by axis (`model/modules/common.py:107-114`)
 (8) transposed conv: forward map of the strided pair with in/out swapped, output on the cached finer map
 (9) BatchNorm = torch.nn.BatchNorm1d on .F  (`model/modules/common.py:21`, `model/resnet.py:95-97`)
"""
import math
import sys
import types
from enum import Enum

import numpy as np
import torch
import torch.nn as nn


class RegionType(Enum):
    HYPERCUBE = 0
    HYPERCROSS = 1
    CUSTOM = 2
    HYBRID = 3


def _as_list(v, D):
    if isinstance(v, (list, tuple, np.ndarray, torch.Tensor)):
        v = [int(x) for x in v]
        assert len(v) == D
        return v
    return [int(v)] * D


def hypercube_offsets(kernel_size):
    """(6): x fastest.  Odd sizes centred, even sizes start at 0 (3).  Returns int64 [K, D] in units of ts."""
    D = len(kernel_size)
    K = int(np.prod(kernel_size))
    out = np.zeros((K, D), np.int64)
    for k in range(K):
        r = k
        for d in range(D):
            idx = r % kernel_size[d]
            r //= kernel_size[d]
            out[k, d] = idx - (kernel_size[d] // 2 if kernel_size[d] % 2 == 1 else 0)
    return out


def hybrid_offsets(kernel_size, axis_types):
    """(7): ME builds a CUSTOM list: start at the origin; per axis, append every existing offset shifted by
    each non-centre step of that axis (HYPERCUBE axes), then HYPERCROSS axes add +-steps from the origin only."""
    D = len(kernel_size)
    offs = [[0] * D]
    for ax, (t, ks) in enumerate(zip(axis_types, kernel_size)):
        if t != RegionType.HYPERCUBE:
            continue
        c = (ks - 1) // 2
        new = []
        for o in offs:
            for cur in range(ks):
                if cur == c:
                    continue
                o2 = list(o)
                o2[ax] = cur - c
                new.append(o2)
        offs.extend(new)
    for ax, (t, ks) in enumerate(zip(axis_types, kernel_size)):
        if t != RegionType.HYPERCROSS:
            continue
        c = (ks - 1) // 2
        for cur in range(ks):
            if cur == c:
                continue
            o2 = [0] * D
            o2[ax] = cur - c
            offs.append(o2)
    return np.asarray(offs, np.int64)


class KernelGenerator:
    def __init__(self, kernel_size=-1, stride=1, dilation=1, is_sparse_region=False,
                 region_type=RegionType.HYPERCUBE, region_offsets=None, axis_types=None, dimension=-1):
        assert dimension > 0
        self.dimension = dimension
        self.kernel_size = _as_list(kernel_size, dimension)
        self.kernel_stride = _as_list(stride, dimension)
        self.kernel_dilation = _as_list(dilation, dimension)
        self.region_type = region_type
        self.axis_types = axis_types
        assert all(d == 1 for d in self.kernel_dilation), "oracle: dilation 1 only (all the hot path uses)"
        if region_type == RegionType.HYPERCUBE:
            self.offsets = hypercube_offsets(self.kernel_size)
        elif region_type == RegionType.HYBRID:
            self.offsets = hybrid_offsets(self.kernel_size, axis_types)
        else:
            raise NotImplementedError(region_type)
        self.kernel_volume = len(self.offsets)


# --------------------------------------------------------------------------- coordinates (integer, numpy)
_OFF = 1 << 15


def pack_keys(c):
    """(b, x, y, z) -> int64 key whose numeric order is lexicographic (b, x, y, z)."""
    c = np.asarray(c, np.int64)
    assert c.shape[1] == 4
    assert (c[:, 0] >= 0).all() and (c[:, 0] < 65535).all()
    assert (np.abs(c[:, 1:]) < _OFF).all()
    return (c[:, 0] << 48) | ((c[:, 1] + _OFF) << 32) | ((c[:, 2] + _OFF) << 16) | (c[:, 3] + _OFF)


def stride_coords(coords, new_ts):
    """(2) + canonical order: unique coarse coordinates sorted by packed key (SURVEY 8a row K1)."""
    c = np.asarray(coords, np.int64).copy()
    c[:, 1:] = np.floor_divide(c[:, 1:], new_ts) * new_ts
    keys = np.unique(pack_keys(c))
    out = np.stack([keys >> 48, ((keys >> 32) & 0xFFFF) - _OFF, ((keys >> 16) & 0xFFFF) - _OFF,
                    (keys & 0xFFFF) - _OFF], 1)
    return out.astype(np.int32)


def kernel_map(in_coords, out_coords, offsets):
    """Per offset k: (in_rows, out_rows) with C_in[i] == C_out[j] + o_k, sorted by out row.  `offsets` are
    absolute (already multiplied by the input tensor stride)."""
    kin = pack_keys(in_coords)
    order = np.argsort(kin, kind="stable")
    skin = kin[order]
    oc = np.asarray(out_coords, np.int64)
    maps = []
    for o in offsets:
        q = oc.copy()
        q[:, 1:] += o
        ok = (np.abs(q[:, 1:]) < _OFF).all(1)
        qk = pack_keys(np.where(ok[:, None], q, 0))
        pos = np.searchsorted(skin, qk)
        pos = np.minimum(pos, len(skin) - 1)
        hit = ok & (skin[pos] == qk)
        j = np.nonzero(hit)[0]
        maps.append((order[pos[j]].astype(np.int64), j.astype(np.int64)))
    return maps


class CoordsKey:
    def __init__(self, D, ts):
        self.D = D
        self.ts = tuple(ts)

    def getTensorStride(self):
        return list(self.ts)

    def __eq__(self, o):
        return isinstance(o, CoordsKey) and self.ts == o.ts and self.D == o.D

    def __hash__(self):
        return hash((self.D, self.ts))


class CoordsManager:
    def __init__(self, D=3):
        self.D = D
        self.levels = {}       # ts tuple -> int32 [N, 1+D]
        self.maps = {}

    def initialize(self, coords, ts):
        c = np.ascontiguousarray(coords.cpu().numpy() if isinstance(coords, torch.Tensor) else coords).astype(np.int32)
        assert len(np.unique(pack_keys(c))) == len(c), "duplicate coordinates"
        self.levels[tuple(ts)] = c
        return CoordsKey(self.D, ts)

    def get_coords(self, key):
        return torch.from_numpy(self.levels[key.ts])

    def stride(self, key, stride):
        new_ts = tuple(t * s for t, s in zip(key.ts, stride))
        if new_ts not in self.levels:
            assert len(set(new_ts)) == 1
            self.levels[new_ts] = stride_coords(self.levels[key.ts], new_ts[0])
        return CoordsKey(self.D, new_ts)

    def get_kernel_map(self, in_key, out_key, kgen, transpose):
        ck = (in_key.ts, out_key.ts, tuple(kgen.kernel_size), kgen.region_type, transpose)
        if ck not in self.maps:
            if not transpose:
                ts = in_key.ts[0]
                m = kernel_map(self.levels[in_key.ts], self.levels[out_key.ts], kgen.offsets * ts)
            else:   # (8): forward map of (fine -> coarse), swapped.  in_key is the coarse level.
                ts = out_key.ts[0]
                fwd = kernel_map(self.levels[out_key.ts], self.levels[in_key.ts], kgen.offsets * ts)
                m = [(j, i) for (i, j) in fwd]
            self.maps[ck] = [(torch.from_numpy(i), torch.from_numpy(j)) for i, j in m]
        return self.maps[ck]


class SparseTensor:
    def __init__(self, feats, coords=None, coords_key=None, coords_manager=None, force_creation=False,
                 allow_duplicate_coords=False, tensor_stride=1):
        assert isinstance(feats, torch.Tensor)
        if coords_manager is None:
            assert coords is not None
            D = coords.shape[1] - 1
            coords_manager = CoordsManager(D)
            coords_key = coords_manager.initialize(coords, _as_list(tensor_stride, D))
        self._F = feats
        self.coords_key = coords_key
        self.coords_man = coords_manager

    @property
    def F(self):
        return self._F

    @property
    def feats(self):
        return self._F

    @property
    def C(self):
        return self.coords_man.get_coords(self.coords_key)

    coords = C

    @property
    def tensor_stride(self):
        return list(self.coords_key.ts)

    @property
    def D(self):
        return self.coords_man.D

    def to(self, device):
        self._F = self._F.to(device)
        return self

    def __len__(self):
        return len(self._F)

    def size(self):
        return self._F.size()

    def __iadd__(self, other):
        assert self.coords_key == other.coords_key
        self._F = self._F + other.F
        return self

    def __add__(self, other):
        assert self.coords_key == other.coords_key
        return SparseTensor(self._F + other.F, coords_key=self.coords_key, coords_manager=self.coords_man)


def sparse_conv(x, W, maps, n_out):
    """ME 0.4.3 ConvolutionForwardKernelCPU algorithm: per offset gather -> GEMM -> scatter-add."""
    out = x.new_zeros((n_out, W.shape[2]))
    for k, (i, j) in enumerate(maps):
        if len(i):
            out = out.index_add(0, j, x.index_select(0, i) @ W[k])
    return out


class MinkowskiNetwork(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.D = D


class _ConvBase(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, is_transpose=False, dimension=-1):
        super().__init__()
        assert dimension > 0
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size, stride, dilation, dimension=dimension)
        self.kernel_generator = kernel_generator
        self.in_channels, self.out_channels = in_channels, out_channels
        self.stride = _as_list(stride, dimension)
        self.is_transpose = is_transpose
        self.dimension = dimension
        self.kernel_volume = kernel_generator.kernel_volume
        self.kernel = nn.Parameter(torch.empty(self.kernel_volume, in_channels, out_channels))
        self.bias = nn.Parameter(torch.empty(1, out_channels)) if has_bias else None
        self.has_bias = has_bias
        n = (out_channels if is_transpose else in_channels) * self.kernel_volume
        stdv = 1.0 / math.sqrt(n)
        with torch.no_grad():
            self.kernel.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.uniform_(-stdv, stdv)

    def forward(self, x):
        cm = x.coords_man
        if not self.is_transpose:
            out_key = cm.stride(x.coords_key, self.stride)
        else:
            ts = tuple(t // s for t, s in zip(x.coords_key.ts, self.stride))
            assert ts in cm.levels, "transposed conv needs the cached finer coordinate map"
            out_key = CoordsKey(cm.D, ts)
        maps = cm.get_kernel_map(x.coords_key, out_key, self.kernel_generator, self.is_transpose)
        y = sparse_conv(x.F, self.kernel, maps, len(cm.levels[out_key.ts]))
        if self.bias is not None:
            y = y + self.bias
        return SparseTensor(y, coords_key=out_key, coords_manager=cm)


class MinkowskiConvolution(_ConvBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, dimension=-1):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, has_bias, kernel_generator,
                         False, dimension)


class MinkowskiConvolutionTranspose(_ConvBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, generate_new_coords=False, dimension=-1):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, has_bias, kernel_generator,
                         True, dimension)


class MinkowskiBatchNorm(nn.Module):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def forward(self, x):
        return SparseTensor(self.bn(x.F), coords_key=x.coords_key, coords_manager=x.coords_man)


class MinkowskiReLU(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, x):
        return SparseTensor(torch.relu(x.F), coords_key=x.coords_key, coords_manager=x.coords_man)


# Pooling layers of the sibling models (SURVEY.md 8f-4; `model/resnet.py:63`, `model/modules/common.py:170-214`), restated with the
# same kernel maps: sum pooling = the convolution of (5) with every W[k] = identity; average pooling divides by the number of inputs
# present; the transposed / unpooling variants use the swapped map of (8).
class _PoolBase(nn.Module):
    AVERAGE, TRANSPOSE = False, False

    def __init__(self, kernel_size=-1, stride=1, dilation=1, kernel_generator=None, dimension=-1):
        super().__init__()
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size, stride, dilation, dimension=dimension)
        self.kernel_generator = kernel_generator
        self.stride = _as_list(stride, dimension)

    def forward(self, x):
        cm = x.coords_man
        if not self.TRANSPOSE:
            out_key = cm.stride(x.coords_key, self.stride)
        else:
            out_key = CoordsKey(cm.D, tuple(t // s for t, s in zip(x.coords_key.ts, self.stride)))
        maps = cm.get_kernel_map(x.coords_key, out_key, self.kernel_generator, self.TRANSPOSE)
        n_out = len(cm.levels[out_key.ts])
        y = x.F.new_zeros((n_out, x.F.shape[1]))
        cnt = x.F.new_zeros((n_out, 1))
        for i, j in maps:
            if len(i):
                y = y.index_add(0, j, x.F.index_select(0, i))
                cnt = cnt.index_add(0, j, x.F.new_ones((len(j), 1)))
        if self.AVERAGE:
            y = y / cnt.clamp(min=1)
        return SparseTensor(y, coords_key=out_key, coords_manager=cm)


class MinkowskiSumPooling(_PoolBase):
    pass


class MinkowskiAvgPooling(_PoolBase):
    AVERAGE = True


class MinkowskiPoolingTranspose(_PoolBase):
    TRANSPOSE = True


class MinkowskiAvgUnpooling(_PoolBase):
    AVERAGE, TRANSPOSE = True, True


class _Unsupported(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError(f"oracle: {type(self).__name__} is restated by plain torch in the tests that need it")


class MinkowskiGlobalPooling(_Unsupported):
    pass


class MinkowskiInstanceNorm(_Unsupported):
    pass


def cat(*tensors):
    k = tensors[0].coords_key
    for t in tensors:
        assert t.coords_key == k, "cat: coords_key mismatch"
    return SparseTensor(torch.cat([t.F for t in tensors], 1), coords_key=k, coords_manager=tensors[0].coords_man)


def install(name="MinkowskiEngine"):
    """Register this module as `MinkowskiEngine` (+ `.MinkowskiOps`) so the reference's model files import on it."""
    me = sys.modules[__name__]
    ops = types.ModuleType(name + ".MinkowskiOps")
    ops.cat = cat
    me.MinkowskiOps = ops
    sys.modules[name] = me
    sys.modules[name + ".MinkowskiOps"] = ops
    import collections
    import collections.abc
    if not hasattr(collections, "Sequence"):       # `model/modules/common.py:78,93` uses the removed alias
        collections.Sequence = collections.abc.Sequence
    return me
