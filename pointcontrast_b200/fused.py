"""Fused training executor for Res16UNet on libpcb200.

The modular surface in `me.py` (one autograd node per MinkowskiConvolution / BatchNorm / ReLU, as in MinkowskiEngine)
is what makes the reference's model file run unchanged; it costs ~1.5k Python-dispatched autograd nodes per step.
This module runs the SAME graph (`pretrain/pointcontrast/model/res16unet.py:206-268`) as one autograd node per forward:

  * unit = conv -> BatchNorm statistics -> one elementwise pass doing normalise + residual add + ReLU
    (`model/modules/resnet_block.py:44-60` collapses to two units per BasicBlock), issued by ONE C call
    (`pcb_unit_forward`, include/pcb200.h); on the offset-split levels the convolution's reduction pass also produces the BatchNorm column sums;
  * `me.cat` is free: the two producers write straight into the column halves of one wider buffer (row strides);
  * backward is a hand-written reverse sweep, one C call per unit (`pcb_unit_backward`): ReLU mask + BatchNorm backward +
    residual-gradient fan-out in one pass, the weight gradient accumulated straight into the (flat) parameter gradient
    buffer, the data gradient written / accumulated into its consumer's gradient buffer;
  * activations live in two bump-allocated arenas per pass (a handful of allocator calls per step instead of ~400);
  * the coordinate manager of a batch (hash tables, strided levels, kernel maps: the only part of a step that needs
    device->host reads) is built on a SIDE stream (`prepare_pair`), so those reads never wait for the previous step's
    backward pass and the integer kernels overlap it.

The executor reads the graph once per model from the attribute names into its unit schedule (`schedule`), so it serves this
package's model class and the reference's own, unmodified `model/res16unet.py` alike; everything else -- issue order,
buffers, gradient modes, workspace size, neighbour tables -- reads the schedule.
"""
import collections
import ctypes

import torch

from . import _lib, me
from ._lib import PcbUnit, check, lib, ptr, stream

ENABLED = True
# Both views of a pair batch in ONE pass (see `stack_views`): half the launches, twice the rows per launch on the deep,
# latency-bound levels.  BatchNorm keeps the reference's per-view statistics through the row-segmented kernels.  Test hook:
# False runs the two forward calls of the reference (tests/test_gpu_model.py compares the two).
PAIR = True
VIEW1_BATCH_OFFSET = 1 << 14      # batch indices of view 1 in a stacked tensor (packed keys hold batch < 65535)
# Test hook: True takes the BatchNorm statistics by a separate pass over z instead of the convolution's reduction pass (the
# cross-check of the fused reduce + statistics pass).
SEPARATE_STATS = False
# Test hook: a list to which every ReLU unit of a training forward pass appends (rows of view 0, bool [n, C] = the ReLU decision
# its backward pass will use), in the order the model file calls its ReLUs.  tests/test_gpu_model.py replays these decisions in
# the fp64 oracle: a pre-activation within rounding distance of zero is a coin flip in ANY finite precision, and one flipped
# entry on a deep level moves every upstream gradient by ~1/sqrt(rows x channels) of its norm.
CAPTURE_RELU = None


# ------------------------------------------------------------------------------------------------ the unit schedule
INPUT = "input"


class Unit:
    """One entry of a model's unit schedule: out = [relu]( BN(conv(x)) [+ res] ), one pcb_unit_forward and one pcb_unit_backward
    call.  (The schedule's `final` entry is the 1x1 output layer: no BatchNorm, issued as plain convolutions.)

    Buffers are named: INPUT (the network's input), "cat5".."cat8" (the decoder's concatenations, read whole) or the index of the
    unit that wrote it.  `out` is None for a fresh buffer, with an fp32 plane if `need_f32`, or (concatenation, first column) for a
    column slice.  `plan` indexes the neighbour-table plans of a `Geometry` (one per distinct `plan_key`).  `gin_mode` / `gres_mode`
    are the backward call's data- and residual-gradient modes (0: none, 1: write, 2: accumulate)."""
    __slots__ = ("conv", "bn", "level_in", "level_out", "transpose", "relu", "x", "res", "out", "need_f32", "K", "Cin", "Cout", "tc",
                 "plan_key", "plan", "gin_mode", "gres_mode")

    def __init__(self, conv, bn, x, level_in, level_out, relu=True, res=None, out=None, need_f32=False):
        self.conv, self.bn, self.x, self.res, self.out, self.relu = conv, bn, x, res, out, relu
        self.level_in, self.level_out, self.transpose = level_in, level_out, conv.is_transpose
        self.need_f32 = need_f32 and out is None
        self.K, self.Cin, self.Cout = (int(v) for v in conv.kernel.shape)
        self.tc = me.tensor_core_shape(self.Cin, self.Cout)
        self.plan_key = (level_in, level_out, conv.kernel_generator.cache_key, self.transpose)
        self.gin_mode = self.gres_mode = 0


# a model's units in issue order, its concatenation buffers as (name, level, width) in allocation order, its final layer, and one
# entry per neighbour-table plan in build order
Schedule = collections.namedtuple("Schedule", "units cats final plans")


class _NotWired(Exception):
    pass


def schedule(model):
    """`model`'s unit schedule -- the one description of the graph the executor runs -- or None if it is not wired like
    `pretrain/pointcontrast/model/res16unet.py:36-268` (Res16UNet with BasicBlock stages) with the widths the tensor-core tiling
    needs (every hidden width % 32).  Read from the attribute names, so ANY class with this wiring -- this package's model file
    or the reference's own, unmodified -- runs fused.  Built once per model (cached on it) from module attributes and kernel
    shapes only: a model on the meta device has one too."""
    d = model.__dict__
    if "_fused_schedule" not in d:
        try:
            d["_fused_schedule"] = _build_schedule(model)
        except (AttributeError, TypeError, IndexError, _NotWired):
            d["_fused_schedule"] = None
    return d["_fused_schedule"]


def matches(model):
    return schedule(model) is not None


def _build_schedule(m):
    P, I = m.PLANES, m.INIT_DIM
    final = m.final
    if not isinstance(final, me.MinkowskiConvolution) or final.kernel_volume != 1:
        raise _NotWired
    units = []

    def unit(conv, bn, x, level_in, level_out, **kw):
        if not isinstance(conv, me._ConvolutionBase) or not isinstance(bn, me.MinkowskiBatchNorm) \
                or conv.is_transpose != (level_out < level_in):
            raise _NotWired
        units.append(Unit(conv, bn, x, level_in, level_out, **kw))
        return len(units) - 1

    def stage(blocks, x, level, out=None, need_f32=False):
        """A stage of BasicBlocks.  A block's output needs its fp32 plane only if the NEXT block adds it back as the identity
        residual (`resnet_block.py:51-57`: no downsample branch); `need_f32` says so for the stage's own output."""
        for i, blk in enumerate(blocks):
            if not isinstance(blk.conv1, me.MinkowskiConvolution) or not isinstance(blk.conv2, me.MinkowskiConvolution) \
                    or hasattr(blk, "conv3") or (blk.downsample is not None and len(blk.downsample) != 2):
                raise _NotWired
            last = i == len(blocks) - 1
            h = unit(blk.conv1, blk.norm1, x, level, level)
            res = x if blk.downsample is None else unit(blk.downsample[0], blk.downsample[1], x, level, level, relu=False, need_f32=True)
            x = unit(blk.conv2, blk.norm2, h, level, level, res=res, out=out if last else None,
                     need_f32=need_f32 if last else blocks[i + 1].downsample is None)
        return x

    # the concatenations: decoder branch in the left columns, encoder skip in the right ones
    cats = (("cat8", 0, P[7] + I), ("cat7", 1, P[6] + P[0]), ("cat6", 2, P[5] + P[1]), ("cat5", 3, P[4] + P[2]))
    x = unit(m.conv0p1s1, m.bn0, INPUT, 0, 0, out=("cat8", P[7]))
    for i, (c, b) in enumerate((("conv1p1s2", "bn1"), ("conv2p2s2", "bn2"), ("conv3p4s2", "bn3"), ("conv4p8s2", "bn4"))):
        blocks = list(getattr(m, f"block{i + 1}"))
        x = unit(getattr(m, c), getattr(m, b), x, i, i + 1, need_f32=blocks[0].downsample is None)
        x = stage(blocks, x, i + 1, out=(f"cat{7 - i}", P[6 - i]) if i < 3 else None)
    fin_tc = me.tensor_core_shape(final.in_channels, final.out_channels)
    for i, (c, b) in enumerate((("convtr4p16s2", "bntr4"), ("convtr5p8s2", "bntr5"), ("convtr6p4s2", "bntr6"), ("convtr7p2s2", "bntr7"))):
        unit(getattr(m, c), getattr(m, b), x, 4 - i, 3 - i, out=(f"cat{5 + i}", 0))
        x = stage(list(getattr(m, f"block{5 + i}")), f"cat{5 + i}", 3 - i, need_f32=i == 3 and not fin_tc)
    fin = Unit(final, None, x, 0, 0, relu=False)
    # the exact fp32 stem (3 input channels), tensor-core widths everywhere else
    if units[0].Cout != I or fin.Cin != P[7] or units[0].tc or not all(u.tc for u in units[1:]) or any(w % 32 for w in (I, *P)):
        raise _NotWired

    # gradient modes: the reverse sweep writes a buffer's gradient first, then accumulates into it (a column slice shares its
    # concatenation's gradient buffer); the final layer's data gradient is the first write
    root = lambda b: units[b].out[0] if isinstance(b, int) and units[b].out is not None else b
    has_grad = {root(fin.x)}
    for i in reversed(range(len(units))):
        u = units[i]
        assert root(i) in has_grad, f"unit {i}: its output gets no gradient before its own backward call"
        for b, mode in ((u.res, "gres_mode"), (u.x, "gin_mode")):
            if b is not None and b != INPUT:
                setattr(u, mode, 2 if root(b) in has_grad else 1)
                has_grad.add(root(b))

    # plans in a fixed build order: tensor-core layers before the exact fp32 stem, stride-1 before strided, larger kernels first,
    # level by level.  The caching allocator splits its blocks by allocation order; schedule order cost a C1 step on an H100
    # 250 KB more peak memory.
    index, plans = {}, []
    for u in sorted(units + [fin], key=lambda u: (not u.tc, u.level_in != u.level_out, -u.K, u.level_in)):
        if u.plan_key not in index:
            index[u.plan_key] = len(plans)
            plans.append(u)
        u.plan = index[u.plan_key]
    return Schedule(tuple(units), cats, fin, tuple(plans))


# ------------------------------------------------------------------------------------------------ side-stream preparation
_SIDE = {}
_READY = {}       # (data_ptr, version, numel) of a device-resident input -> event recorded on the compute stream when first seen


def _side_stream(device):
    s = _SIDE.get(device.index)
    if s is None:
        s = _SIDE[device.index] = torch.cuda.Stream(device=device)
    return s


def _await_input(t, side):
    """Device-resident input about to be read on the side stream.  Its producer ran on some stream before this call; the
    first time a tensor (same storage, same version) is seen, the side stream waits for everything queued on the current
    stream so far.  A tensor seen before -- a dataset resident in HBM, `bench.py`'s batches -- needs no wait once the
    event recorded back then has completed."""
    if not t.is_cuda:
        return
    key = (t.data_ptr(), t._version, t.numel())
    ev = _READY.get(key)
    if ev is None:
        if len(_READY) > 4096:
            _READY.clear()
        ev = _READY[key] = torch.cuda.Event()
        ev.record()
    if not ev.query():
        side.wait_event(ev)


class Prepared:
    """A stacked pair batch with its coordinate geometry built: what `run` needs to start issuing convolutions."""
    __slots__ = ("sinput", "n0", "geom")


def stack_views(feats0, coords0, feats1, coords1, device):
    """One SparseTensor holding view 0's rows followed by view 1's, view 1's batch indices shifted by VIEW1_BATCH_OFFSET.
    Scenes never interact in the network (the batch index is part of the coordinate key), so every convolution of the
    stacked tensor equals the two separate forwards row for row; on every strided level (rows in packed-key order,
    batch most significant) view 0's rows still come first.  Returns (SparseTensor on `device`, rows of view 0)."""
    if not coords0.is_cuda and coords0.shape[0] and int(coords0[:, 0].max()) >= VIEW1_BATCH_OFFSET:
        raise _lib.PcbError(f"batch index >= {VIEW1_BATCH_OFFSET} cannot be stacked")
    n0 = coords0.shape[0]
    C = torch.cat([coords0.to(device, non_blocking=True).to(torch.int32), coords1.to(device, non_blocking=True).to(torch.int32)])
    C[n0:, 0] += VIEW1_BATCH_OFFSET
    F = torch.cat([feats0.to(device, non_blocking=True), feats1.to(device, non_blocking=True)])
    return me.SparseTensor(F, coords=C), n0


def prepare_pair(model, feats0, coords0, feats1, coords1, device):
    """Host->device copies, view stacking, coordinate-manager build and every kernel map the network will ask for -- on the
    side stream.  The current stream is made to wait for the result (a device-side wait: the host does not block on it),
    so the returned object can be consumed by `run` right away; call this for batch i+1 before reading back the loss of
    batch i and none of it is on the critical path."""
    device = torch.device(device)
    p = Prepared()
    with torch.cuda.device(device):
        main = torch.cuda.current_stream()
        side = _side_stream(device)
        for t in (feats0, coords0, feats1, coords1):
            _await_input(t, side)
        with torch.cuda.stream(side):
            p.sinput, p.n0 = stack_views(feats0, coords0, feats1, coords1, device)
            p.geom = Geometry(model, p.sinput, p.n0, tile_orders=True)
            done = torch.cuda.Event()
            done.record(side)
        main.wait_event(done)
        for t in p.geom.tensors():          # allocated on the side stream's pool, consumed by kernels of the compute stream
            t.record_stream(main)
    return p


class Geometry:
    """Levels, row counts, per-view row splits and kernel maps of one input: everything the executor needs from the
    coordinate manager (`SparseTensor` -> 4 strided levels -> one plan per distinct `Unit.plan_key` of the model's schedule,
    each on the tables of its own units' kernel generator: 19 plans on 19 neighbour tables for Res16UNet), built in one go
    with a single device->host read at the end for the per-level view split."""

    def __init__(self, model, sinput, view0_rows=None, tile_orders=False):
        sched = schedule(model)
        cm = sinput.coords_man
        self.sinput = sinput
        with torch.cuda.device(sinput.F.device):
            keys = [sinput.coords_key]
            for _ in range(4):
                keys.append(cm.stride(keys[-1], [2, 2, 2]))
            n = [cm.num_rows(k) for k in keys]
            # With `tile_orders` (prepare_pair, whose side stream keeps the sorts off the critical path), tile orders for the forward
            # launches of the transposed convolutions only.  Their tables give each fine row exactly one coarse neighbour, so a
            # window-sorted tile stages about 1 of the 8 offsets instead of 5-8, and those launches ran 1.7-2.9x faster on an H100.
            # Ordering every other table too (3x3x3: 20-22 of 27 offsets per tile instead of 27) sped some launches up by up to 15 %
            # and slowed others by up to 26 %, 0.35 ms more per C1 step than this choice: DESIGN.md section 7.
            self.plans = [cm.conv_plan(keys[u.level_in], keys[u.level_out], u.conv.kernel_generator, u.transpose,
                                       tile_order=tile_orders and u.tc and u.transpose) for u in sched.plans]
            if view0_rows is None or view0_rows >= n[0]:
                seg = list(n)
            else:                                # rows of view 0 per level: strided levels are sorted by key, batch most significant
                if view0_rows < 1:
                    raise _lib.PcbError("view 0 of a stacked pair is empty")
                thr = VIEW1_BATCH_OFFSET << 48
                cnt = torch.stack([(cm.levels[k.ts].keys < thr).sum() for k in keys[1:]]).tolist()
                seg = [int(view0_rows)] + [int(c) for c in cnt]
        self.keys, self.n, self.seg = keys, n, seg
        self.calls = 2 if seg[0] < n[0] else 1
        self.cm = cm

    def tensors(self):
        out = [self.sinput.F]
        for lvl in self.cm.levels.values():
            out += [t for t in (lvl.keys, lvl.tkeys, lvl.tvals, lvl._coords) if t is not None]
        for ent in self.cm.plans.values():
            out += [t for t in ent.values() if isinstance(t, torch.Tensor)]
        return out


# ------------------------------------------------------------------------------------------------ buffers
class Arena:
    """Bump allocator over a few large torch allocations (stream-ordered, freed together when the pass is done)."""

    def __init__(self, device, hint):
        self.device = device
        self.blocks = []
        self.cur = None
        self.off = 0
        self.cap = 0
        self.total = 0
        self.block_bytes = max(int(hint), 32 << 20)

    def alloc(self, nbytes):
        nbytes = (int(nbytes) + 255) & ~255
        if self.off + nbytes > self.cap:
            size = max(nbytes, self.block_bytes)
            self.cur = torch.empty(size, dtype=torch.uint8, device=self.device)
            self.blocks.append(self.cur)
            self.off, self.cap = 0, size
        p = self.cur.data_ptr() + self.off
        self.off += nbytes
        self.total += nbytes
        return p


def _grow_hint(old, used):
    """Arena size for the next pass: never shrinks and moves in 64 MiB steps, so that after a few steps every pass asks the
    caching allocator for the SAME block size (alternating batch sizes would otherwise leave it a zoo of multi-GB blocks)."""
    step = 64 << 20
    need = (int(used * 1.03) + step - 1) // step * step
    return max(old, need)


class Buf:
    """Matrix [n, C] with row stride ld.  `p`: fp32 storage (or 0), `hi`/`lo`: the same values as bf16 split planes (or 0)
    -- the operand format of the tensor-core kernels.  Storage belongs to an Arena (or `owner` keeps a tensor alive)."""
    __slots__ = ("owner", "p", "hi", "lo", "bh", "bl", "n", "C", "ld", "_grad", "parent", "col", "device")

    def __init__(self, owner, p, n, C, ld, device, hi=0, lo=0, parent=None, col=0, bh=0, bl=0):
        self.owner, self.p, self.hi, self.lo, self.n, self.C, self.ld, self.device = owner, p, hi, lo, n, C, ld, device
        self.bh, self.bl = bh, bl             # me.FWD_FP16: hi/lo are fp16 planes (forward gathers), bh/bl the bf16 planes (weight gradient)
        self.parent, self.col = parent, col
        self._grad = None

    @staticmethod
    def new(arena, n, C, fp32=True, split=False, dual=False):
        """split: 16-bit hi/lo planes; dual: the activation format of me.FWD_FP16 (fp16 hi/lo + bf16 hi/lo)."""
        p = arena.alloc(4 * n * C) if fp32 else 0
        hi = lo = bh = bl = 0
        if split:
            hi = arena.alloc((8 if dual else 4) * n * C)
            lo = hi + 2 * n * C
            if dual:
                bh = lo + 2 * n * C
                bl = bh + 2 * n * C
        return Buf(None, p, n, C, C, arena.device, hi, lo, bh=bh, bl=bl)

    def cols(self, c0, C):
        return Buf(self.owner, self.p + 4 * c0 if self.p else 0, self.n, C, self.ld, self.device, self.hi + 2 * c0 if self.hi else 0,
                   self.lo + 2 * c0 if self.lo else 0, parent=self, col=c0, bh=self.bh + 2 * c0 if self.bh else 0,
                   bl=self.bl + 2 * c0 if self.bl else 0)

    def grad(self, arena):
        """fp32 gradient buffer with the same geometry (column slices share their parent's buffer)."""
        if self._grad is None:
            if self.parent is not None:
                g = self.parent.grad(arena)
                self._grad = Buf(None, g.p + 4 * self.col, self.n, self.C, g.ld, self.device)
            else:
                self._grad = Buf(None, arena.alloc(4 * self.n * self.ld), self.n, self.C, self.ld, self.device)
        return self._grad


class _Plane:
    def __init__(self, p, n, C, ld):
        self.__cuda_array_interface__ = {"shape": (n, C), "strides": (2 * ld, 2), "typestr": "<i2", "data": (p, False), "version": 2}


def _plane_i16(p, n, C, ld, device):
    """A 16-bit plane of a Buf as an int16 tensor view (positive fp16 / bf16 values are positive int16 bit patterns)."""
    with torch.cuda.device(device):
        return torch.as_tensor(_Plane(p, n, C, ld), device=device)


_Tape = collections.namedtuple("_Tape", "structs bufs arena stats geom ws")


class Runner:
    def __init__(self, model):
        self.model = model
        self.schedule = schedule(model)
        self.anchor = torch.zeros(1, requires_grad=True)
        self._fwd_hint = 0
        self._bwd_hint = 0
        self._ws_cache = {}
        self._tile_batch = None

    # ------------------------------------------------------------------------------------------ single launches (final layer)
    def _conv(self, kind, plan, fin, x, out, bias=None):
        """The final layer's forward ("fwd") or data gradient ("dgrad") into `out`."""
        kern, Cin, Cout = fin.conv.kernel, fin.Cin, fin.Cout
        if fin.tc:
            assert x.hi, "tensor-core conv needs the split planes of its input"
            tiles = fin.conv._prepared.tiles(kern, me.FWD_FP16)[0 if kind == "fwd" else 1]
            fp16 = me.FWD_FP16 and kind == "fwd"          # forward roles: fp16 activation planes x fp16 weight tiles
            me.conv(kind, plan, Cin, Cout, (x.hi, x.lo), x.ld, out.p, out.ld, tiles=ptr(tiles), bias=ptr(bias), fp16=fp16)
        else:
            # exact fp32 kernel: output widths the tensor-core tiling does not cover (13 / 20 semantic classes); as a data gradient it
            # runs on the per-offset transposed weights
            assert x.p, "the exact fp32 conv reads the fp32 plane"
            w = kern.detach() if kind == "fwd" else kern.detach().transpose(1, 2).contiguous()
            me.conv(kind, plan, Cin, Cout, x.p, x.ld, out.p, out.ld, w=ptr(w), bias=ptr(bias))

    def _wgrad(self, fin, plan, a_in, dz):
        kern = fin.conv.kernel
        if kern.grad is None:
            kern.grad = torch.zeros_like(kern)
        if fin.tc:
            pl = lambda b: (b.bh, b.bl) if b.bh else (b.hi, b.lo)          # activations: their bf16 planes (gradients only have those)
            me.wgrad(plan, fin.Cin, fin.Cout, pl(a_in), a_in.ld, pl(dz), dz.ld, kern.grad.data_ptr(), True, accumulate=True)
        else:
            me.wgrad(plan, fin.Cin, fin.Cout, a_in.p, a_in.ld, dz.p, dz.ld, kern.grad.data_ptr(), False, accumulate=True)

    def _refresh_tiles(self):
        """Re-tile the weights of every tensor-core convolution in ONE launch when the parameters changed (after each optimiser
        step) and hand the results to the per-layer caches (`me._PreparedWeights`), instead of one small launch per layer."""
        m = self.model
        convs = [c for c in m.modules() if isinstance(c, me._ConvolutionBase) and me.tensor_core_shape(c.in_channels, c.out_channels)]
        tags = [me._PreparedWeights.tag(c.kernel, me.FWD_FP16) for c in convs]
        if all(c._prepared.tile_tag == t for c, t in zip(convs, tags)):
            return
        cache = self._tile_batch
        key = tuple((c.kernel.data_ptr(), tuple(c.kernel.shape)) for c in convs) + (me.FWD_FP16,)
        if cache is None or cache[0] != key:
            dev = convs[0].kernel.device
            sizes_f = [lib.pcb_weight_tile_bytes(*c.kernel.shape, 0) for c in convs]
            sizes_d = [lib.pcb_weight_tile_bytes(*c.kernel.shape, 1) for c in convs]
            al = lambda v: (v + 255) & ~255
            buf = torch.zeros(sum(al(v) for v in sizes_f + sizes_d), dtype=torch.uint8, device=dev)
            descs = (_lib.PcbTileDesc * len(convs))()
            views, off, start = [], 0, 0
            for i, c in enumerate(convs):
                f = buf[off:off + sizes_f[i]]; off += al(sizes_f[i])
                d = buf[off:off + sizes_d[i]]; off += al(sizes_d[i])
                K, Cin, Cout = c.kernel.shape
                check(lib.pcb_tile_desc_fill(ctypes.byref(descs[i]), c.kernel.data_ptr(), K, Cin, Cout, f.data_ptr(), d.data_ptr(),
                                             _lib.PLANES_B_FP16 if me.FWD_FP16 else 0, start))
                start += K * Cin * Cout
                views.append((f, d))
            host = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8)
            cache = self._tile_batch = (key, host.to(dev), views, start, buf)
        _, ddev, views, total, _ = cache
        check(lib.pcb_weight_tile_batch(ddev.data_ptr(), len(convs), total, stream()))
        for c, t, v in zip(convs, tags, views):
            c._prepared._tiles, c._prepared.tile_tag = v, t

    def _ws_bytes(self, n):
        """Scratch for the largest unit at `n` rows per level (the units run back to back on one stream and share it)."""
        n = tuple(n)
        best = self._ws_cache.get(n)
        if best is None:
            if len(self._ws_cache) > 64:
                self._ws_cache.clear()
            best = self._ws_cache[n] = max(lib.pcb_unit_ws_bytes(u.K, n[u.level_in], n[u.level_out], u.Cin, u.Cout)
                                           for u in self.schedule.units)
        return best

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, sinput, view0_rows=None, geom=None, eval_mode=False):
        """`view0_rows`: the input is a `stack_views` tensor whose first `view0_rows` rows are view 0.
        `eval_mode`: forward only with eval-mode BatchNorm (running statistics); nothing is kept for a backward pass.
        Each unit: out = [relu]( BN(conv(x)) [+ residual] ), one pcb_unit_forward call."""
        m, sched = self.model, self.schedule
        dual = me.FWD_FP16 and not eval_mode          # bf16 copies of the activations are only needed by the weight gradient
        feats = sinput.F
        _lib.require_cuda(feats)
        dev = feats.device
        g = geom if geom is not None else Geometry(m, sinput, view0_rows)
        n = g.n
        flags = ((_lib.UNIT_SEPARATE_STATS if SEPARATE_STATS else 0) | (_lib.UNIT_FP16_FORWARD if me.FWD_FP16 else 0)
                 | (_lib.UNIT_EVAL if eval_mode else 0))
        with torch.cuda.device(dev):
            st = stream()
            stats = torch.empty(4 * sum(mod.bn.num_features for mod in m.modules() if isinstance(mod, me.MinkowskiBatchNorm)),
                                dtype=torch.float32, device=dev)
            stat_p = stats.data_ptr()
            ws = _lib.workspace(self._ws_bytes(n), dev)
            self._refresh_tiles()
            arena = Arena(dev, self._fwd_hint)
            x_in = feats.detach().contiguous().float()
            bufs = {INPUT: Buf(x_in, x_in.data_ptr(), n[0], x_in.shape[1], x_in.shape[1], dev)}
            for name, level, C in sched.cats:             # consumed by convolutions only: split planes
                bufs[name] = Buf.new(arena, n[level], C, fp32=False, split=True, dual=dual)
            structs = []
            for i, s in enumerate(sched.units):
                bn, kern, plan, a_in = s.bn.bn, s.conv.kernel, g.plans[s.plan], bufs[s.x]
                n_out, n0 = plan.n_out, g.seg[s.level_out]      # n0: rows of view 0 at the output level (== n_out: a single view)
                nseg = 2 if n0 < n_out else 1
                z = Buf.new(arena, n_out, s.Cout)
                if s.out is None:
                    out = Buf.new(arena, n_out, s.Cout, fp32=s.need_f32, split=True, dual=dual)
                else:
                    out = bufs[s.out[0]].cols(s.out[1], s.Cout)
                u = PcbUnit()
                u.n_in, u.n_out, u.n0 = plan.n_in, n_out, n0
                u.K, u.Cin, u.Cout, u.relu = s.K, s.Cin, s.Cout, 1 if s.relu else 0
                u.fwd_tbl, u.fwd_stride = plan.fwd_tbl.data_ptr(), plan.fwd_tbl.shape[1]
                km = plan.c_kmap("fwd_kmap")
                u.fwd_kmap = ctypes.cast(km, ctypes.c_void_p) if km is not None else None
                u.fwd_perm = ptr(plan.fwd_perm)
                u.W = kern.data_ptr()
                if s.tc:
                    tiles = s.conv._prepared.tiles(kern, me.FWD_FP16)
                    u.wt_fwd, u.wt_dg = tiles[0].data_ptr(), tiles[1].data_ptr()
                    u.x_hi, u.x_lo, u.x_lds = a_in.hi, a_in.lo, a_in.ld
                    if a_in.bh:
                        u.x_bhi, u.x_blo = a_in.bh, a_in.bl
                if a_in.p:
                    u.x_p, u.x_ld = a_in.p, a_in.ld
                u.gamma, u.beta = bn.weight.data_ptr(), bn.bias.data_ptr()
                u.running_mean, u.running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                if bn.momentum is None:
                    raise NotImplementedError("BatchNorm with momentum=None (cumulative average) is not on the hot path")
                u.eps, u.momentum = bn.eps, bn.momentum
                u.mean, u.invstd = stat_p, stat_p + 4 * nseg * s.Cout
                stat_p += 8 * nseg * s.Cout
                u.z_p, u.z_ld = z.p, z.ld
                if out.p:
                    u.out_p, u.out_ld = out.p, out.ld
                u.out_hi, u.out_lo, u.out_lds = out.hi, out.lo, out.ld
                if out.bh:
                    u.out_bhi, u.out_blo = out.bh, out.bl
                if s.res is not None:
                    res = bufs[s.res]
                    assert res.p, "a residual input needs its fp32 plane"
                    u.res_p, u.res_ld = res.p, res.ld
                u.ws, u.ws_bytes = ws.data_ptr(), ws.numel()
                u.flags = flags
                me.record_profile("fwd", plan, s.K, s.Cin, s.Cout, s.tc)
                check(lib.pcb_unit_forward(ctypes.byref(u), st))
                if CAPTURE_RELU is not None and s.relu:
                    CAPTURE_RELU.append((n0, _plane_i16(out.hi, n_out, s.Cout, out.ld, dev) > 0))
                bufs[i] = out
                structs.append(u)
            fin = sched.final
            out_t = torch.empty(n[0], fin.Cout, dtype=torch.float32, device=dev)
            out = Buf(out_t, out_t.data_ptr(), n[0], fin.Cout, fin.Cout, dev)
            bias = fin.conv.bias
            self._conv("fwd", g.plans[fin.plan], fin, bufs[fin.x], out, bias=bias.detach().reshape(-1) if bias is not None else None)
            if not eval_mode:
                torch._foreach_add_([s.bn.bn.num_batches_tracked for s in sched.units], g.calls)       # one multi-tensor launch, not 62
        self._fwd_hint = _grow_hint(self._fwd_hint, arena.total)
        if eval_mode:
            return out_t, None
        # the units' u.ws is used again by the backward sweep, and a later, larger request replaces the cached buffer: the tape holds it
        return out_t, _Tape(structs, bufs, arena, stats, g, ws)

    # ------------------------------------------------------------------------------------------ backward
    def backward(self, tape, d_out):
        sched, g, bufs = self.schedule, tape.geom, tape.bufs
        fin = sched.final
        d_out = d_out.contiguous()
        dev = d_out.device
        with torch.cuda.device(dev):
            st = stream()
            arena = Arena(dev, self._bwd_hint)
            if fin.tc:
                dfin = Buf.new(arena, d_out.shape[0], d_out.shape[1], fp32=False, split=True)
                check(lib.pcb_split_rows(d_out.data_ptr(), d_out.shape[1], d_out.shape[0], d_out.shape[1], dfin.hi, dfin.lo, dfin.ld, 0, st))
            else:                                # e.g. 13 / 20 classes: the final layer's backward runs on the exact fp32 kernels
                dfin = Buf(d_out, d_out.data_ptr(), d_out.shape[0], d_out.shape[1], d_out.shape[1], dev)
            bias = fin.conv.bias
            if bias is not None:
                if bias.grad is None:
                    bias.grad = torch.zeros_like(bias)
                bias.grad += d_out.sum(0, keepdim=True)
            p_final, x_last = g.plans[fin.plan], bufs[fin.x]
            self._wgrad(fin, p_final, x_last, dfin)
            self._conv("dgrad", p_final, fin, dfin, x_last.grad(arena))
            after_unit = self.model.__dict__.get("_fused_after_unit")       # trainer hook: gradient all-reduce of the chunk this unit completes
            for i in reversed(range(len(sched.units))):
                s, u = sched.units[i], tape.structs[i]
                bn, kern, plan = s.bn.bn, s.conv.kernel, g.plans[s.plan]
                gb = bufs[i].grad(arena)
                u.g_p, u.g_ld = gb.p, gb.ld
                dz = Buf.new(arena, u.n_out, s.Cout, fp32=not s.tc, split=s.tc)       # consumed only by the conv kernels: split planes suffice
                u.dz_p, u.dz_hi, u.dz_lo, u.dz_ld = dz.p or None, dz.hi or None, dz.lo or None, dz.ld
                u.gres_p, u.gres_ld, u.gres_mode = None, 0, s.gres_mode
                if s.gres_mode:
                    rg = bufs[s.res].grad(arena)
                    u.gres_p, u.gres_ld = rg.p, rg.ld
                for prm in (bn.weight, bn.bias, kern):
                    if prm.grad is None:
                        prm.grad = torch.zeros_like(prm)
                u.dgamma, u.dbeta, u.dW = bn.weight.grad.data_ptr(), bn.bias.grad.data_ptr(), kern.grad.data_ptr()
                u.wg_tbl, u.wg_stride, u.wg_gather_x = plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], 1 if plan.wg_gather_x else 0
                u.gin_p, u.gin_ld, u.gin_mode = None, 0, s.gin_mode
                if s.gin_mode:
                    ga = bufs[s.x].grad(arena)
                    u.gin_p, u.gin_ld = ga.p, ga.ld
                    u.dg_tbl, u.dg_stride = plan.dg_tbl.data_ptr(), plan.dg_tbl.shape[1]
                    km = plan.c_kmap("dg_kmap")
                    u.dg_kmap = ctypes.cast(km, ctypes.c_void_p) if km is not None else None
                me.record_profile("wgrad", plan, s.K, s.Cin, s.Cout, s.tc)
                if s.gin_mode:
                    me.record_profile("dgrad", plan, s.K, s.Cin, s.Cout, s.tc)
                check(lib.pcb_unit_backward(ctypes.byref(u), st))
                if after_unit is not None:
                    after_unit(s.conv)
            self._bwd_hint = _grow_hint(self._bwd_hint, arena.total)
            # the arenas (and the geometry's tables) are released here, in stream order after the last kernel that reads them


class _FusedFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, runner, sinput, view0_rows, geom):
        out, tape = runner.forward(sinput, view0_rows, geom)
        ctx.runner, ctx.tape = runner, tape
        return out

    @staticmethod
    def backward(ctx, d_out):
        ctx.runner.backward(ctx.tape, d_out)
        ctx.tape = None
        return None, None, None, None, None


def applicable_on(model, device):
    return (ENABLED and model.training and torch.is_grad_enabled() and torch.device(device).type == "cuda"
            and not me.FORCE_SIMT and matches(model))


def applicable(model, sinput):
    return applicable_on(model, sinput.F.device)


def applicable_eval(model, sinput):
    """Inference (`model.eval()` under `torch.no_grad()`, `downstream/semseg/lib/test.py:95-117`): the same units, forward only."""
    return (ENABLED and not model.training and not torch.is_grad_enabled() and sinput.F.is_cuda and not me.FORCE_SIMT and matches(model))


def run_eval(model, sinput):
    runner = model.__dict__.get("_fused_runner")
    if runner is None:
        runner = Runner(model)
        model.__dict__["_fused_runner"] = runner
    return runner.forward(sinput, None, None, eval_mode=True)[0]


def _normalised(model, F):
    if getattr(model, "normalize_feature", False):       # `model/res16unet.py:262-266` (no epsilon)
        from .losses import l2_normalize
        return l2_normalize(F)
    return F


def run_prepared(model, prep):
    """(F0, F1) of a `prepare_pair` batch."""
    F = _normalised(model, run(model, prep.sinput, prep.n0, prep.geom))
    return F[:prep.n0], F[prep.n0:]


def can_stack(model, device):
    return PAIR and isinstance(model, me.MinkowskiNetwork) and applicable_on(model, device)


def forward_pair(model, feats0, coords0, feats1, coords1, device):
    """Features (F0, F1) of the two views of a pair batch -- what `lib/ddp_trainer.py:290-297,392-398` gets from two
    calls of the model.  With the fused executor both views go through ONE stacked pass (`stack_views`), each BatchNorm
    still normalising every view with its own statistics; otherwise this is the two calls.  Works for any model class
    that `matches` (this package's or the reference's own `model/res16unet.py`)."""
    if can_stack(model, device) and len(coords0) and len(coords1):
        return run_prepared(model, prepare_pair(model, feats0, coords0, feats1, coords1, device))
    F0 = model(me.SparseTensor(feats0, coords=coords0).to(device)).F
    F1 = model(me.SparseTensor(feats1, coords=coords1).to(device)).F
    return F0, F1


def run(model, sinput, view0_rows=None, geom=None):
    """Final-layer features [N, out_channels] (before the optional L2 normalisation) as ONE autograd node."""
    runner = model.__dict__.get("_fused_runner")
    if runner is None:
        runner = Runner(model)
        model.__dict__["_fused_runner"] = runner
    return _FusedFunction.apply(runner.anchor, runner, sinput, view0_rows, geom)
