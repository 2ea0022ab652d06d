"""MinkowskiEngine-compatible operator surface backed by libpcb200 (hand-written sm_90a CUDA, include/pcb200.h).

This module provides the names PointContrast's hot path imports from `MinkowskiEngine` v0.4.3
(`pretrain/pointcontrast/model/res16unet.py:10-12`, `model/resnet.py:8-9`, `model/modules/common.py:9,21,53-62,
127-167`, `model/modules/resnet_block.py:10`, `lib/ddp_trainer.py:26,290-297`), with the same constructor
arguments, attributes and state_dict keys, so that the reference's model and trainer files run on it unchanged
after `pointcontrast_b200.me.install()` (which registers it as `MinkowskiEngine`).

Differences from ME 0.4.3, by design:
  * the coordinate manager lives on the GPU (hash table + dense neighbour tables), not in a CPU hash map;
  * rows of strided levels are in canonical packed-key order (ME's is hash-iteration order, i.e. unspecified);
  * there is no CPU execution path: every op raises on CPU tensors.
"""
import ctypes
import math
import sys
import types
from enum import Enum

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import check, lib, ptr, stream, workspace


class RegionType(Enum):
    HYPERCUBE = 0
    HYPERCROSS = 1
    CUSTOM = 2
    HYBRID = 3


def _listify(v, D):
    if isinstance(v, (list, tuple, np.ndarray, torch.Tensor)):
        v = [int(a) for a in v]
        if len(v) != D:
            raise ValueError(f"expected {D} values, got {v}")
        return v
    return [int(v)] * D


def _cube_offsets(ks):
    """First spatial axis fastest; odd sizes centred, even sizes anchored at 0 (SURVEY.md 8c items 3, 6)."""
    grids = np.meshgrid(*[np.arange(k) - (k // 2 if k % 2 else 0) for k in reversed(ks)], indexing="ij")
    return np.stack([g.reshape(-1) for g in reversed(grids)], 1).astype(np.int64)


def _hybrid_offsets(ks, axis_types):
    """ME's HYBRID -> CUSTOM expansion: origin, then per HYPERCUBE axis every existing offset shifted by each
    non-centre step, then HYPERCROSS axes from the origin (SURVEY.md 8c item 7)."""
    D = len(ks)
    offs = [tuple([0] * D)]
    for ax in range(D):
        if axis_types[ax] != RegionType.HYPERCUBE:
            continue
        c = (ks[ax] - 1) // 2
        steps = [s - c for s in range(ks[ax]) if s != c]
        offs += [tuple(o[:ax]) + (s,) + tuple(o[ax + 1:]) for o in list(offs) for s in steps]
    for ax in range(D):
        if axis_types[ax] != RegionType.HYPERCROSS:
            continue
        c = (ks[ax] - 1) // 2
        offs += [tuple([0] * ax + [s - c] + [0] * (D - ax - 1)) for s in range(ks[ax]) if s != c]
    return np.asarray(offs, np.int64)


class KernelGenerator:
    def __init__(self, kernel_size=-1, stride=1, dilation=1, is_sparse_region=False,
                 region_type=RegionType.HYPERCUBE, region_offsets=None, axis_types=None, dimension=-1):
        if dimension != 3:
            raise NotImplementedError("pointcontrast_b200 implements D=3 (the PointContrast hot path)")
        self.dimension = dimension
        self.kernel_size = _listify(kernel_size, dimension)
        self.kernel_stride = _listify(stride, dimension)
        self.kernel_dilation = _listify(dilation, dimension)
        if any(d != 1 for d in self.kernel_dilation):
            raise NotImplementedError("dilation != 1 is not on the hot path")
        self.region_type = region_type
        self.axis_types = axis_types
        if region_type == RegionType.HYPERCUBE:
            self.offsets = _cube_offsets(self.kernel_size)
        elif region_type == RegionType.HYBRID:
            self.offsets = _hybrid_offsets(self.kernel_size, axis_types)
        else:
            raise NotImplementedError(f"{region_type} is not on the hot path")
        self.kernel_volume = len(self.offsets)
        if self.kernel_volume > _lib.MAX_KERNEL_VOLUME:
            raise NotImplementedError("kernel volume > 27")
        self.cache_key = (tuple(self.kernel_size), tuple(map(tuple, self.offsets.tolist())))


class CoordsKey:
    def __init__(self, D, ts):
        self.D = D
        self.ts = tuple(int(t) for t in ts)

    def getTensorStride(self):
        return list(self.ts)

    def getKey(self):
        return self.ts

    def __eq__(self, o):
        return isinstance(o, CoordsKey) and self.D == o.D and self.ts == o.ts

    def __hash__(self):
        return hash((self.D, self.ts))

    def __repr__(self):
        return f"CoordsKey(ts={self.ts})"


class _Level:
    __slots__ = ("keys", "n", "ts", "tkeys", "tvals", "cap", "_coords")

    def __init__(self, keys, n, ts):
        self.keys, self.n, self.ts = keys, n, ts
        self.tkeys = self.tvals = None
        self.cap = 0
        self._coords = None


class ConvPlan:
    """Neighbour tables for one (input level, output level, kernel) triple -- ME's cached kernel map.
    fwd:   Y[j]  = sum_k X[fwd_tbl[fwd_kmap[k]][j]] W[k]
    dgrad: dX[i] = sum_k dY[dg_tbl[dg_kmap[k]][i]] W[k]^T
    wgrad: dW[k] = sum_r A[wg_tbl[k][r]]^T B[r], (A,B) = (X,dY) if wg_gather_x else (dY,X) with transposed output.
    fwd_perm: the tile order (pcb_conv_tile_order) of fwd_tbl for the tensor-core kernel, or None (identity)."""
    __slots__ = ("K", "n_in", "n_out", "fwd_tbl", "fwd_kmap", "dg_tbl", "dg_kmap", "wg_tbl", "wg_gather_x", "fwd_perm", "_counts",
                 "_c_kmaps")

    def pair_counts(self):
        """|M_k| per kernel offset (host list) -- the ME per-offset map sizes."""
        if self._counts is None:
            cnt = torch.zeros(self.K, dtype=torch.int64, device=self.fwd_tbl.device)
            check(lib.pcb_kernel_map_count(ptr(self.fwd_tbl), self.K, self.fwd_tbl.shape[1], ptr(cnt), stream()))
            self._counts = cnt.cpu().tolist()
        return self._counts

    def c_kmap(self, which):
        """HOST int32 array of the kernel-offset permutation `which` ("fwd_kmap" / "dg_kmap"), cached on the plan, or None."""
        if which not in self._c_kmaps:
            vals = getattr(self, which)
            self._c_kmaps[which] = _c_int_array(vals) if vals is not None else None
        return self._c_kmaps[which]


# Rows per window of the tile order: a tile's rows, sorted by neighbour mask, all come from one window of this many consecutive output
# rows, so the input rows its gathers read stay close together (L2-resident) while the window still holds enough rows of each mask
# class to fill whole tiles.  Chosen by the sweep of profiles/bench_conv_order.py (DESIGN.md section 7).
TILE_ORDER_WINDOW = 16384


def _c_int_array(vals):
    return (ctypes.c_int32 * len(vals))(*[int(v) for v in vals])


class CoordsManager:
    """GPU coordinate manager: one hashed level per tensor stride + cached neighbour tables."""

    def __init__(self, D=3):
        if D != 3:
            raise NotImplementedError("D=3 only")
        self.D = D
        self.levels = {}
        self.plans = {}
        self._pending = None          # (cpu coords, ts) until a device is known
        self.device = None

    # -- construction
    def initialize(self, coords, ts):
        if coords.dim() != 2 or coords.shape[1] != self.D + 1:
            raise ValueError("coords must be [N, 1+D] = (batch, x, y, z)")
        ts = tuple(ts)
        if coords.is_cuda:
            self._init_device(coords, ts)
        else:
            self._pending = (coords, ts)
        return CoordsKey(self.D, ts)

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.PcbError("the coordinate manager lives on a CUDA device (no CPU path)")
        if self._pending is not None:
            coords, ts = self._pending
            self._pending = None
            self._init_device(coords.to(device, non_blocking=True), ts)
        elif self.device is not None and self.device != device:
            raise _lib.PcbError("moving a built coordinate manager across devices is not supported")

    def _init_device(self, coords, ts):
        self.device = coords.device
        c = coords.to(torch.int32).contiguous()
        n = c.shape[0]
        with torch.cuda.device(self.device):
            keys = torch.empty(n, dtype=torch.int64, device=self.device)
            status = torch.zeros(1, dtype=torch.int32, device=self.device)
            check(lib.pcb_coords_pack(ptr(c), n, ptr(keys), ptr(status), stream()))
            lvl = _Level(keys, n, ts)
            lvl._coords = c
            self._hash(lvl, status)
            st = int(status.item())
        if st & _lib.ERR_RANGE:
            raise _lib.PcbError("coordinate out of the packable range (batch < 65535, |x|,|y|,|z| < 32768)")
        if st & _lib.ERR_DUPLICATE:
            raise _lib.PcbError("duplicate coordinates in SparseTensor")
        self.levels[ts] = lvl

    def _hash(self, lvl, status=None):
        cap = 1 << max(4, int(math.ceil(math.log2(max(2 * lvl.n, 2)))))
        lvl.cap = cap
        lvl.tkeys = torch.empty(cap, dtype=torch.int64, device=self.device)
        lvl.tvals = torch.empty(cap, dtype=torch.int32, device=self.device)
        if status is None:
            status = torch.zeros(1, dtype=torch.int32, device=self.device)
        check(lib.pcb_hash_build(ptr(lvl.keys), lvl.n, ptr(lvl.tkeys), ptr(lvl.tvals), cap, ptr(status), stream()))

    def _require_ready(self):
        if self._pending is not None or self.device is None:
            raise _lib.PcbError("SparseTensor is still on the CPU: call .to(cuda_device) first (no CPU path)")

    # -- queries
    def get_coords(self, key):
        self._require_ready()
        lvl = self.levels[key.ts]
        if lvl._coords is None:
            with torch.cuda.device(self.device):
                c = torch.empty(lvl.n, 4, dtype=torch.int32, device=self.device)
                check(lib.pcb_coords_unpack(ptr(lvl.keys), lvl.n, ptr(c), stream()))
            lvl._coords = c
        return lvl._coords

    def num_rows(self, key):
        return self.levels[key.ts].n

    def stride(self, key, stride):
        self._require_ready()
        stride = _listify(stride, self.D)
        new_ts = tuple(t * s for t, s in zip(key.ts, stride))
        if new_ts == key.ts:
            return key
        if new_ts not in self.levels:
            if len(set(new_ts)) != 1:
                raise NotImplementedError("anisotropic tensor strides are not on the hot path")
            src = self.levels[key.ts]
            with torch.cuda.device(self.device):
                out_keys = torch.empty(src.n, dtype=torch.int64, device=self.device)
                wsb = lib.pcb_coords_stride_ws_bytes(src.n)
                ws = workspace(wsb, self.device)
                n_out = ctypes.c_int64(0)
                check(lib.pcb_coords_stride(ptr(src.keys), src.n, new_ts[0], ptr(out_keys), None, ctypes.byref(n_out),
                                            ptr(ws), wsb, stream()))
                lvl = _Level(out_keys[:n_out.value].clone(), n_out.value, new_ts)
                self._hash(lvl)
            self.levels[new_ts] = lvl
        return CoordsKey(self.D, new_ts)

    def _table(self, out_lvl, in_lvl, offsets):
        K = len(offsets)
        tbl = torch.empty(K, out_lvl.n, dtype=torch.int32, device=self.device)
        offs = _c_int_array(np.asarray(offsets, np.int64).reshape(-1).tolist())
        check(lib.pcb_kernel_map(ptr(out_lvl.keys), out_lvl.n, ptr(in_lvl.tkeys), ptr(in_lvl.tvals), in_lvl.cap, offs, K,
                                 ptr(tbl), stream()))
        return tbl

    def _tile_order(self, tbl):
        n = tbl.shape[1]
        perm = torch.empty(n, dtype=torch.int32, device=self.device)
        wsb = lib.pcb_conv_tile_order_ws_bytes(n)
        ws = workspace(wsb, self.device)
        check(lib.pcb_conv_tile_order(ptr(tbl), n, tbl.shape[0], n, TILE_ORDER_WINDOW, ptr(perm), ptr(ws), wsb, stream()))
        return perm

    def conv_plan(self, in_key, out_key, kgen, transpose, tile_order=False):
        """Cached per (levels, kernel) like ME's kernel-map cache; strided conv and its transpose share tables.  tile_order: the plan
        also carries the tile order of its forward table, built once per table (a 1-offset kernel has nothing to reorder)."""
        self._require_ready()
        fine, coarse = (out_key, in_key) if transpose else (in_key, out_key)
        ck = (fine.ts, coarse.ts, kgen.cache_key)
        ent = self.plans.get(ck)
        with torch.cuda.device(self.device):
            if ent is None:
                ent = {}
                offs = kgen.offsets * fine.ts[0]
                if fine.ts == coarse.ts:
                    lvl = self.levels[fine.ts]
                    ent["same"] = self._table(lvl, lvl, offs)
                    lookup = {tuple(o): i for i, o in enumerate(kgen.offsets.tolist())}
                    ent["opp"] = [lookup[tuple(-a for a in o)] for o in kgen.offsets.tolist()] \
                        if all(tuple(-a for a in o) in lookup for o in kgen.offsets.tolist()) else None
                else:
                    lf, lc = self.levels[fine.ts], self.levels[coarse.ts]
                    ent["down"] = self._table(lc, lf, offs)        # rows: coarse, entries: fine rows
                    ent["up"] = self._table(lf, lc, -offs)         # rows: fine, entries: the (single) coarse parent
                self.plans[ck] = ent
        p = ConvPlan()
        p._counts = None
        p._c_kmaps = {}
        p.K = kgen.kernel_volume
        p.n_in, p.n_out = self.levels[in_key.ts].n, self.levels[out_key.ts].n
        if "same" in ent:
            if ent["opp"] is None:
                raise NotImplementedError("asymmetric stride-1 kernels are not on the hot path")
            fwd, dg = "same", "same"
            p.fwd_kmap, p.dg_kmap = None, ent["opp"]
            p.wg_tbl, p.wg_gather_x = ent["same"], True
        else:
            fwd, dg = ("up", "down") if transpose else ("down", "up")
            p.fwd_kmap = p.dg_kmap = None
            p.wg_tbl, p.wg_gather_x = ent["down"], not transpose
        p.fwd_tbl, p.dg_tbl = ent[fwd], ent[dg]
        p.fwd_perm = None
        if tile_order and p.K > 1:
            if ("perm", fwd) not in ent:
                with torch.cuda.device(self.device):
                    ent[("perm", fwd)] = self._tile_order(ent[fwd])
            p.fwd_perm = ent[("perm", fwd)]
        return p


# ------------------------------------------------------------------------------------------------ tensor
class SparseTensor:
    def __init__(self, feats, coords=None, coords_key=None, coords_manager=None, force_creation=False,
                 allow_duplicate_coords=False, tensor_stride=1):
        if not isinstance(feats, torch.Tensor):
            raise TypeError("feats must be a torch.Tensor")
        if allow_duplicate_coords or force_creation:
            raise NotImplementedError("allow_duplicate_coords / force_creation are not supported: coordinates must be unique "
                                      "(the reference voxelises before building the tensor, `lib/ddp_data_loaders.py:228-241`)")
        if coords_manager is None:
            if coords is None:
                raise ValueError("either coords or (coords_key, coords_manager) is required")
            D = coords.shape[1] - 1
            coords_manager = CoordsManager(D)
            coords_key = coords_manager.initialize(coords, _listify(tensor_stride, D))
            if feats.is_cuda:
                coords_manager.to(feats.device)
        elif coords_key is None:
            raise ValueError("coords_key is required with coords_manager")
        self._F = feats
        self.coords_key = coords_key
        self.coords_man = coords_manager

    @property
    def F(self):
        return self._F

    feats = F

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

    @property
    def device(self):
        return self._F.device

    def to(self, device):
        self._F = self._F.to(device)
        self.coords_man.to(self._F.device)
        return self

    def __len__(self):
        return self._F.shape[0]

    def size(self):
        return self._F.size()

    def __iadd__(self, other):
        if self.coords_key != other.coords_key:
            raise ValueError("coords_key mismatch in +=")
        self._F += other.F
        return self

    def __add__(self, other):
        if self.coords_key != other.coords_key:
            raise ValueError("coords_key mismatch in +")
        return SparseTensor(self._F + other.F, coords_key=self.coords_key, coords_manager=self.coords_man)

    def __repr__(self):
        return f"SparseTensor(F={tuple(self._F.shape)}, ts={self.tensor_stride})"


# ------------------------------------------------------------------------------------------------ convolution
FORCE_SIMT = False      # tests flip this to run the exact fp32 kernels
SIMT_OPS = set()        # diagnostics: subset of {"fwd", "dgrad", "wgrad"} forced onto the exact fp32 kernels (modular path)
# bench.py sets this to a list: every convolution / weight-gradient entry-point call then appends its description here, in
# issue order -- the same order in which the library (pcb_profile_enable) brackets those calls with CUDA events.
PROFILE = None
# Fused executor: activations travel as fp16 hi/lo planes and the forward weight tiles are fp16 (22 mantissa bits per operand instead of
# bf16 hi/lo's 16): the forward pass is what sets the whole-network gradient error.  Test hook: False runs bf16 everywhere (the
# modular path's numerics), the reference side of tests/test_gpu_model.py and profiles/grad_precision_ab.py.
FWD_FP16 = True


def record_profile(kind, plan, K, Cin, Cout, tc):
    """The PROFILE record of one library call ("fwd" / "dgrad" / "wgrad" of the convolution [K][Cin][Cout] on `plan`)."""
    if PROFILE is not None:
        PROFILE.append(dict(kind=kind, K=K, Cin=Cin, Cout=Cout, n_in=plan.n_in, n_out=plan.n_out, plan=plan, tc=tc))


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def conv(kind, plan, Cin, Cout, x, ldx, y, ldy, tiles=None, w=None, bias=None, accumulate=False, fp16=False):
    """y (+)= one convolution of `plan` with the kernel [K][Cin][Cout]: kind "fwd" maps x [n_in, Cin] to y [n_out, Cout], kind "dgrad"
    (the data gradient: opposite roles) maps x [n_out, Cout] to y [n_in, Cin].  Arguments are device pointers, row strides in elements.
      tiles: this call's pre-tiled weights (`_PreparedWeights.tiles`) -> the split-operand tensor-core kernel; x = (hi, lo) plane
             pointers, bf16 unless `fp16` (fp16 planes and forward tiles);
      else : the exact fp32 kernel on x = fp32 rows and w = the fp32 weights in this call's [K][Cin][Cout] roles; it cannot accumulate."""
    K = plan.K
    record_profile(kind, plan, K, Cin, Cout, tiles is not None)
    if kind == "fwd":
        tbl, kmap, perm, n_out = plan.fwd_tbl, plan.c_kmap("fwd_kmap"), plan.fwd_perm, plan.n_out
    else:
        tbl, kmap, perm, n_out, Cin, Cout = plan.dg_tbl, plan.c_kmap("dg_kmap"), None, plan.n_in, Cout, Cin
    if tiles is not None:
        flags = (_lib.CONV_ACCUMULATE if accumulate else 0) | ((_lib.PLANES_A_FP16 | _lib.PLANES_B_FP16) if fp16 else 0)
        wsb = lib.pcb_conv_forward_split_ws_bytes(K, n_out, Cin, Cout)
        ws = workspace(wsb, _device())
        check(lib.pcb_conv_forward_split_ordered(x[0], x[1], ldx, ptr(tbl), tbl.shape[1], kmap, K, ptr(perm), n_out, Cin, Cout, tiles,
                                                 bias, y, ldy, ptr(ws), wsb, flags, stream()))
    else:
        if accumulate:
            raise _lib.PcbError("the exact fp32 convolution writes its output, it does not accumulate")
        check(lib.pcb_conv_forward(x, ldx, ptr(tbl), tbl.shape[1], kmap, K, n_out, Cin, Cout, w, bias, y, ldy, stream()))


def wgrad(plan, Cin, Cout, x, ldx, dy, lddy, dw, split, accumulate=False, force_simt=False):
    """dw (+)= the weight gradient [K][Cin][Cout] of `plan` from its input x [n_in, Cin] and output gradient dy [n_out, Cout] (device
    pointers, row strides in elements).  split: x, dy = (hi, lo) bf16 plane pointers -> the tensor-core kernel; else fp32 rows -> the
    exact kernel (force_simt: its generic kernel also for the stem layer)."""
    K = plan.K
    record_profile("wgrad", plan, K, Cin, Cout, split)
    if plan.wg_gather_x:
        A, lda, B, ldb, Ca, Cb, tr, rows = x, ldx, dy, lddy, Cin, Cout, 0, plan.n_out
    else:
        A, lda, B, ldb, Ca, Cb, tr, rows = dy, lddy, x, ldx, Cout, Cin, 1, plan.n_in
    flags = _lib.CONV_ACCUMULATE if accumulate else 0
    tbl = plan.wg_tbl
    if split:
        wsb = lib.pcb_conv_wgrad_split_ws_bytes(K, rows, Ca, Cb)
        ws = workspace(wsb, _device())
        check(lib.pcb_conv_wgrad_split(A[0], A[1], lda, B[0], B[1], ldb, ptr(tbl), tbl.shape[1], K, rows, Ca, Cb, dw, tr, ptr(ws), wsb,
                                       flags, stream()))
    else:
        wsb = lib.pcb_conv_wgrad_ws_bytes(K, rows, Ca, Cb)
        ws = workspace(wsb, _device())
        check(lib.pcb_conv_wgrad(A, lda, B, ldb, ptr(tbl), tbl.shape[1], K, rows, Ca, Cb, dw, tr, ptr(ws), wsb,
                                 flags | (_lib.CONV_FORCE_SIMT if force_simt else 0), stream()))


_WEIGHTS_EPOCH = [0]


def bump_weights_epoch():
    """Parameters were rewritten through raw pointers (the fused SGD kernel, a broadcast into the flat buffer): torch's
    per-tensor version counters do not see that, so every cached split / tiled copy of a kernel is invalidated here."""
    _WEIGHTS_EPOCH[0] += 1


class _PreparedWeights:
    """A kernel's weights pre-tiled for the split-operand conv kernel, refreshed when the parameter or the wanted format changes."""

    def __init__(self):
        self.tile_tag = None
        self._tiles = None

    @staticmethod
    def tag(kernel, fp16):
        return (kernel.data_ptr(), kernel._version, tuple(kernel.shape), _WEIGHTS_EPOCH[0], fp16)

    def tiles(self, kernel, fp16):
        """(forward, data-gradient) weights pre-tiled as shared-memory images for the split wgmma kernel (TMA bulk loads); the
        forward tiles are fp16 x 2^10 if `fp16`, else bf16 like the data-gradient ones."""
        tag = self.tag(kernel, fp16)
        if tag != self.tile_tag:
            K, Cin, Cout = kernel.shape
            f = torch.empty(lib.pcb_weight_tile_bytes(K, Cin, Cout, 0), dtype=torch.uint8, device=kernel.device)
            d = torch.empty(lib.pcb_weight_tile_bytes(K, Cin, Cout, 1), dtype=torch.uint8, device=kernel.device)
            check(lib.pcb_weight_tile(ptr(kernel.detach()), K, Cin, Cout, ptr(f), ptr(d), _lib.PLANES_B_FP16 if fp16 else 0, stream()))
            self._tiles, self.tile_tag = (f, d), tag
        return self._tiles


def _simt(op):
    return FORCE_SIMT or op in SIMT_OPS


def tensor_core_shape(Cin, Cout):
    """Widths the split-operand tensor-core kernels tile (both multiples of 32); other convolutions run the exact fp32 kernels."""
    return Cin % 32 == 0 and Cout % 32 == 0


def _use_tc(Cin, Cout, op="fwd"):
    return (not _simt(op)) and tensor_core_shape(Cin, Cout)


def _split_rows(t):
    """bf16 hi/lo planes of a contiguous fp32 matrix (the operand format of the tensor-core kernels): (storage, (hi, lo) pointers)."""
    n = t.shape[0] * t.shape[1]
    pl = torch.empty(2 * n, dtype=torch.bfloat16, device=t.device)
    hi = pl.data_ptr()
    check(lib.pcb_split_rows(ptr(t), t.shape[1], t.shape[0], t.shape[1], hi, hi + 2 * n, t.shape[1], 0, stream()))
    return pl, (hi, hi + 2 * n)


class _SparseConvFunction(torch.autograd.Function):
    """The modular surface's convolution: tensor-core shapes run the split-operand kernel on bf16 hi/lo planes and bf16 weight
    tiles; the 3-channel stem, widths that are not multiples of 32 and FORCE_SIMT / SIMT_OPS run the exact fp32 kernels."""

    @staticmethod
    def forward(ctx, x, kernel, bias, plan, prepared):
        _lib.require_cuda(x)
        x = x.contiguous()
        if x.dtype != torch.float32:
            raise _lib.PcbError("features must be float32")
        Cin, Cout = kernel.shape[1:]
        with torch.cuda.device(x.device):
            y = torch.empty(plan.n_out, Cout, dtype=torch.float32, device=x.device)
            b = bias.detach().reshape(-1) if bias is not None else None
            if _use_tc(Cin, Cout):
                xs, xp = _split_rows(x)
                conv("fwd", plan, Cin, Cout, xp, Cin, ptr(y), Cout, tiles=ptr(prepared.tiles(kernel, False)[0]), bias=ptr(b))
            else:
                w = kernel.detach().contiguous()
                conv("fwd", plan, Cin, Cout, ptr(x), Cin, ptr(y), Cout, w=ptr(w), bias=ptr(b))
        ctx.save_for_backward(x, kernel)
        ctx.plan, ctx.prepared, ctx.has_bias = plan, prepared, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, kernel = ctx.saved_tensors
        plan = ctx.plan
        Cin, Cout = kernel.shape[1:]
        dy = dy.contiguous()
        dx = dw = db = None
        with torch.cuda.device(dy.device):
            dgrad_tc = ctx.needs_input_grad[0] and _use_tc(Cin, Cout, "dgrad")
            wgrad_tc = ctx.needs_input_grad[1] and _use_tc(Cin, Cout, "wgrad")
            dys, dyp = _split_rows(dy) if dgrad_tc or wgrad_tc else (None, None)      # one split of dy serves both tensor-core calls
            if ctx.needs_input_grad[0]:
                dx = torch.empty(plan.n_in, Cin, dtype=torch.float32, device=dy.device)
                if dgrad_tc:
                    conv("dgrad", plan, Cin, Cout, dyp, Cout, ptr(dx), Cin, tiles=ptr(ctx.prepared.tiles(kernel, False)[1]))
                else:
                    wt = kernel.detach().transpose(1, 2).contiguous()      # the data-gradient roles' [K][Cout][Cin]
                    conv("dgrad", plan, Cin, Cout, ptr(dy), Cout, ptr(dx), Cin, w=ptr(wt))
            if ctx.needs_input_grad[1]:
                dw = torch.empty_like(kernel)
                if wgrad_tc:
                    xs, xp = _split_rows(x)
                    wgrad(plan, Cin, Cout, xp, Cin, dyp, Cout, ptr(dw), True)
                else:       # exact fp32 (stem layer, odd widths, FORCE_SIMT)
                    wgrad(plan, Cin, Cout, ptr(x), Cin, ptr(dy), Cout, ptr(dw), False, force_simt=_simt("wgrad"))
            if ctx.has_bias and ctx.needs_input_grad[2]:
                db = dy.sum(0, keepdim=True)
        return dx, dw, db, None, None


class MinkowskiNetwork(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.D = D

    def __call__(self, *args, **kwargs):
        """Training-mode calls of a network wired like Res16UNet (`model/res16unet.py:36-268`) run as ONE fused autograd
        node (`fused.py`) -- whichever file defines the class, so the reference's own `model/res16unet.py` gets the same
        kernels and schedule as this package's model.  Everything else goes through `forward` module by module."""
        if len(args) == 1 and not kwargs and isinstance(args[0], SparseTensor) and args[0].F.is_cuda:
            from . import fused
            if fused.applicable_eval(self, args[0]):
                x = args[0]
                return SparseTensor(fused._normalised(self, fused.run_eval(self, x)), coords_key=x.coords_key, coords_manager=x.coords_man)
            if fused.applicable(self, args[0]):
                x = args[0]
                F = fused._normalised(self, fused.run(self, x))      # `model/res16unet.py:262-266` (no epsilon)
                return SparseTensor(F, coords_key=x.coords_key, coords_manager=x.coords_man)
        return super().__call__(*args, **kwargs)


class _ConvolutionBase(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, is_transpose=False, dimension=-1):
        super().__init__()
        if dimension <= 0:
            raise ValueError("dimension must be positive")
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size, stride, dilation, dimension=dimension)
        self.kernel_generator = kernel_generator
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _listify(kernel_size, dimension)
        self.stride = _listify(stride, dimension)
        self.dilation = _listify(dilation, dimension)
        self.is_transpose = is_transpose
        self.has_bias = has_bias
        self.dimension = dimension
        self.kernel_volume = kernel_generator.kernel_volume
        self.kernel = nn.Parameter(torch.empty(self.kernel_volume, in_channels, out_channels))
        self.bias = nn.Parameter(torch.empty(1, out_channels)) if has_bias else None
        self._prepared = _PreparedWeights()
        self.reset_parameters(is_transpose)

    def reset_parameters(self, is_transpose=False):
        n = (self.out_channels if is_transpose else self.in_channels) * self.kernel_volume
        stdv = 1.0 / math.sqrt(n)
        with torch.no_grad():
            self.kernel.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.uniform_(-stdv, stdv)

    def forward(self, input):
        cm = input.coords_man
        if not self.is_transpose:
            out_key = cm.stride(input.coords_key, self.stride)
        else:
            ts = tuple(t // s for t, s in zip(input.coords_key.ts, self.stride))
            if ts not in cm.levels:
                raise _lib.PcbError("MinkowskiConvolutionTranspose needs the cached finer coordinate map")
            out_key = CoordsKey(cm.D, ts)
        plan = cm.conv_plan(input.coords_key, out_key, self.kernel_generator, self.is_transpose)
        y = _SparseConvFunction.apply(input.F, self.kernel, self.bias, plan, self._prepared)
        return SparseTensor(y, coords_key=out_key, coords_manager=cm)

    def extra_repr(self):
        return (f"in={self.in_channels}, out={self.out_channels}, kernel_size={self.kernel_size}, "
                f"stride={self.stride}, region={self.kernel_generator.region_type.name}")


class MinkowskiConvolution(_ConvolutionBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, dimension=-1):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, has_bias, kernel_generator, False,
                         dimension)


class MinkowskiConvolutionTranspose(_ConvolutionBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, has_bias=False,
                 kernel_generator=None, generate_new_coords=False, dimension=-1):
        if generate_new_coords:
            raise NotImplementedError("generate_new_coords is not on the hot path")
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, has_bias, kernel_generator, True,
                         dimension)


# ------------------------------------------------------------------------------------------------ batch norm
class _BatchNormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, eps, momentum, training):
        _lib.require_cuda(x)
        x = x.contiguous()
        n, C = x.shape
        y = torch.empty_like(x)
        with torch.cuda.device(x.device):
            if training:
                mean = torch.empty(C, dtype=torch.float32, device=x.device)
                invstd = torch.empty_like(mean)
                wsb = lib.pcb_bn_ws_bytes(n, C)
                ws = workspace(wsb, x.device)
                check(lib.pcb_bn_stats_seg(ptr(x), C, n, n, C, eps, momentum if momentum is not None else 0.0, ptr(mean),
                                           ptr(invstd), ptr(running_mean), ptr(running_var), ptr(ws), wsb, stream()))
            else:
                mean, invstd = running_mean, torch.rsqrt(running_var + eps)
            check(lib.pcb_bn_apply_seg(ptr(x), C, n, n, C, ptr(mean), ptr(invstd), ptr(gamma.detach()), ptr(beta.detach()), None, C,
                                       0, ptr(y), C, None, None, 0, None, None, stream()))
        ctx.save_for_backward(x, gamma, mean, invstd)
        ctx.training = training
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, mean, invstd = ctx.saved_tensors
        dy = dy.contiguous()
        n, C = x.shape
        if not ctx.training:
            scale = gamma * invstd
            xhat = (x - mean) * invstd
            return dy * scale, (dy * xhat).sum(0), dy.sum(0), None, None, None, None, None
        dx = torch.empty_like(x)
        dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
        dbeta = torch.empty_like(dgamma)
        with torch.cuda.device(x.device):
            wsb = lib.pcb_bn_ws_bytes(n, C)
            ws = workspace(wsb, x.device)
            check(lib.pcb_bn_backward_seg(ptr(dy), C, ptr(x), C, None, 0, n, n, C, ptr(mean), ptr(invstd), ptr(gamma.detach()), ptr(dx),
                                          C, ptr(dgamma), ptr(dbeta), 0, None, 0, 0, None, None, 0, ptr(ws), wsb, stream()))
        return dx, dgamma, dbeta, None, None, None, None, None


class MinkowskiBatchNorm(nn.Module):
    """BatchNorm1d over all rows of .F.  Holds a real `nn.BatchNorm1d` as `.bn` so that parameter names
    (`bn.weight`, `bn.running_mean`, ...) and `weight_initialization` (`model/resnet.py:93-97`) are unchanged."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        if not (affine and track_running_stats):
            raise NotImplementedError("only affine, running-stat-tracking BatchNorm is on the hot path")
        if momentum is None:
            raise NotImplementedError("momentum=None (cumulative moving average) is not on the hot path; pass a float")
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def forward(self, input):
        bn = self.bn
        training = bn.training
        if training:
            bn.num_batches_tracked += 1
        y = _BatchNormFunction.apply(input.F, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum,
                                     training)
        return SparseTensor(y, coords_key=input.coords_key, coords_manager=input.coords_man)


class MinkowskiReLU(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()
        self.inplace = inplace

    def forward(self, input):
        f = torch.relu_(input.F) if self.inplace else torch.relu(input.F)
        return SparseTensor(f, coords_key=input.coords_key, coords_manager=input.coords_man)


# ------------------------------------------------------------------------------------------------ pooling & per-instance ops
# The layers the sibling models use next to the hot path (SURVEY.md 8f-4: `model/resnet.py:63`, `model/modules/common.py:19-30,170-214`,
# `downstream/semseg/lib/layers.py:12-90`).  Pooling runs on the neighbour tables with one gather-sum kernel (`pcb_gather_sum`);
# the per-instance reductions (global pooling, broadcast, instance norm) are segment sums over the batch index.
def _gather_sum(x, tbl, kmap, K, n_out, want_count=False):
    x = x.contiguous()
    C = x.shape[1]
    pad = (-C) % 4
    if pad:
        x = torch.nn.functional.pad(x, (0, pad))
    y = torch.empty(n_out, C + pad, dtype=torch.float32, device=x.device)
    cnt = torch.empty(n_out, dtype=torch.float32, device=x.device) if want_count else None
    km = _c_int_array(kmap) if kmap is not None else None
    with torch.cuda.device(x.device):
        check(lib.pcb_gather_sum(ptr(x), C + pad, ptr(tbl), tbl.shape[1], km, K, n_out, C + pad, ptr(y), C + pad, ptr(cnt), stream()))
    return (y[:, :C] if pad else y), cnt


class _PoolFunction(torch.autograd.Function):
    """y[j] = sum_k x[fwd_tbl[k][j]] (/ count[j] if average); backward: the same sum over the transposed table."""

    @staticmethod
    def forward(ctx, x, plan, average):
        _lib.require_cuda(x)
        y, cnt = _gather_sum(x.float(), plan.fwd_tbl, plan.fwd_kmap, plan.K, plan.n_out, want_count=average)
        ctx.plan, ctx.cnt = plan, None
        if average:
            cnt = cnt.clamp_(min=1.0)[:, None]
            y = y / cnt
            ctx.cnt = cnt
        return y

    @staticmethod
    def backward(ctx, dy):
        plan = ctx.plan
        if ctx.cnt is not None:
            dy = dy / ctx.cnt
        dx, _ = _gather_sum(dy.contiguous(), plan.dg_tbl, plan.dg_kmap, plan.K, plan.n_in)
        return dx, None, None


class _PoolingBase(nn.Module):
    AVERAGE, TRANSPOSE = False, False

    def __init__(self, kernel_size=-1, stride=1, dilation=1, kernel_generator=None, dimension=-1):
        super().__init__()
        if dimension <= 0:
            raise ValueError("dimension must be positive")
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size, stride, dilation, dimension=dimension)
        self.kernel_generator = kernel_generator
        self.stride = _listify(stride, dimension)
        self.dimension = dimension

    def forward(self, input):
        cm = input.coords_man
        if not self.TRANSPOSE:
            out_key = cm.stride(input.coords_key, self.stride)
        else:
            ts = tuple(t // s for t, s in zip(input.coords_key.ts, self.stride))
            if ts not in cm.levels:
                raise _lib.PcbError(f"{type(self).__name__} needs the cached finer coordinate map")
            out_key = CoordsKey(cm.D, ts)
        plan = cm.conv_plan(input.coords_key, out_key, self.kernel_generator, self.TRANSPOSE)
        return SparseTensor(_PoolFunction.apply(input.F, plan, self.AVERAGE), coords_key=out_key, coords_manager=cm)


class MinkowskiSumPooling(_PoolingBase):
    pass


class MinkowskiAvgPooling(_PoolingBase):
    AVERAGE = True


class MinkowskiPoolingTranspose(_PoolingBase):
    TRANSPOSE = True


class MinkowskiAvgUnpooling(_PoolingBase):
    AVERAGE, TRANSPOSE = True, True


def _instances(input):
    """(batch index per row as int64 [N], number of instances) of a SparseTensor."""
    b = input.C[:, 0].long()
    return b, int(b.max().item()) + 1 if b.numel() else 0


class MinkowskiGlobalPooling(nn.Module):
    """Per-instance mean (or sum) of the features: one row per batch index, on the origin coordinate map (tensor stride 0)."""

    def __init__(self, average=True, dimension=-1):
        super().__init__()
        self.average = average

    def forward(self, input):
        _lib.require_cuda(input.F)
        b, nb = _instances(input)
        out = torch.zeros(nb, input.F.shape[1], dtype=input.F.dtype, device=input.F.device).index_add_(0, b, input.F)
        if self.average:
            out = out / torch.bincount(b, minlength=nb).clamp(min=1)[:, None].to(out.dtype)
        return _GlobalTensor(out, input)


class _GlobalTensor:
    """Result of a global pooling: one feature row per instance (`.F`), remembering the tensor it was pooled from."""

    def __init__(self, feats, source):
        self.F, self.coords_key, self.coords_man = feats, source.coords_key, source.coords_man

    feats = property(lambda self: self.F)


class _BroadcastBase(nn.Module):
    def __init__(self, dimension=-1):
        super().__init__()

    def forward(self, input, input_glob):
        b, _ = _instances(input)
        return SparseTensor(self._op(input.F, input_glob.F[b]), coords_key=input.coords_key, coords_manager=input.coords_man)


class MinkowskiBroadcastAddition(_BroadcastBase):
    _op = staticmethod(torch.add)


class MinkowskiBroadcastMultiplication(_BroadcastBase):
    _op = staticmethod(torch.mul)


class MinkowskiInstanceNorm(nn.Module):
    """Per-instance, per-channel normalisation over the instance's rows, affine (`model/modules/common.py:22-23`)."""

    def __init__(self, num_features, D=-1, dimension=-1, eps=1e-6):
        super().__init__()
        self.num_features, self.eps = num_features, eps
        self.weight = nn.Parameter(torch.ones(1, num_features))
        self.bias = nn.Parameter(torch.zeros(1, num_features))

    def forward(self, input):
        _lib.require_cuda(input.F)
        x = input.F
        b, nb = _instances(input)
        cnt = torch.bincount(b, minlength=nb).clamp(min=1)[:, None].to(x.dtype)
        mean = torch.zeros(nb, x.shape[1], dtype=x.dtype, device=x.device).index_add_(0, b, x) / cnt
        xc = x - mean[b]
        var = torch.zeros(nb, x.shape[1], dtype=x.dtype, device=x.device).index_add_(0, b, xc * xc) / cnt
        y = xc * torch.rsqrt(var + self.eps)[b] * self.weight + self.bias
        return SparseTensor(y, coords_key=input.coords_key, coords_manager=input.coords_man)


def cat(*tensors):
    key = tensors[0].coords_key
    for t in tensors:
        if t.coords_key != key:
            raise ValueError("cat: all tensors must share one coords_key")
    return SparseTensor(torch.cat([t.F for t in tensors], dim=1), coords_key=key, coords_manager=tensors[0].coords_man)


def convert_to_int_tensor(arg, expand_dimension):
    """ME 0.4.3 `MinkowskiCommon.convert_to_int_tensor`: an IntTensor of `expand_dimension` entries from a scalar or a sequence."""
    if isinstance(arg, torch.IntTensor):
        assert arg.numel() == expand_dimension
        return arg
    if isinstance(arg, (list, tuple, np.ndarray)):
        tmp = torch.IntTensor([i for i in arg])
        assert tmp.numel() == expand_dimension
    elif np.isscalar(arg):
        tmp = torch.IntTensor([int(arg) for _ in range(expand_dimension)])
    else:
        raise ValueError("Input must be a scalar or a sequence")
    return tmp


_CRF_ONLY = ("{} is used only by the CRF wrappers of the sparse-conv model package (`models/conditional_random_fields.py`: "
             "BilateralCRF / TrilateralCRF), which this library does not provide; it exists so that the package imports")


def convert_region_type(*args, **kwargs):
    raise NotImplementedError(_CRF_ONLY.format("convert_region_type"))


class MinkowskiConvolutionFunction:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError(_CRF_ONLY.format("MinkowskiConvolutionFunction"))

    @staticmethod
    def apply(*args, **kwargs):
        raise NotImplementedError(_CRF_ONLY.format("MinkowskiConvolutionFunction"))


def install(name="MinkowskiEngine"):
    """Register this module as `MinkowskiEngine` (and `MinkowskiEngine.MinkowskiOps`)."""
    me = sys.modules[__name__]
    ops = types.ModuleType(name + ".MinkowskiOps")
    ops.cat = cat
    me.MinkowskiOps = ops
    sys.modules[name] = me
    sys.modules[name + ".MinkowskiOps"] = ops
    import collections
    import collections.abc
    if not hasattr(collections, "Sequence"):     # py>=3.10 removed the alias `model/modules/common.py:78,93` uses
        collections.Sequence = collections.abc.Sequence
    return me
