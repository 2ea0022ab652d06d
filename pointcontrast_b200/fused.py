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

The executor reads the graph from the attribute names (`matches`), so it serves this package's model class and the
reference's own, unmodified `model/res16unet.py` alike.
"""
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
            p.geom = Geometry(model, p.sinput, p.n0)
            done = torch.cuda.Event()
            done.record(side)
        main.wait_event(done)
        for t in p.geom.tensors():          # allocated on the side stream's pool, consumed by kernels of the compute stream
            t.record_stream(main)
    return p


class Geometry:
    """Levels, row counts, per-view row splits and kernel maps of one input: everything the executor needs from the
    coordinate manager (`SparseTensor` -> 4 strided levels -> 5 + 5 + 4 + 4 + 1 neighbour tables), built in one go with a
    single device->host read at the end for the per-level view split."""

    def __init__(self, model, sinput, view0_rows=None):
        m = model
        cm = sinput.coords_man
        self.sinput = sinput
        with torch.cuda.device(sinput.F.device):
            keys = [sinput.coords_key]
            for _ in range(4):
                keys.append(cm.stride(keys[-1], [2, 2, 2]))
            n = [cm.num_rows(k) for k in keys]
            kg3 = m.block1[0].conv1.kernel_generator
            kg1 = m.final.kernel_generator
            kg2 = m.conv1p1s2.kernel_generator
            self.p3 = [cm.conv_plan(k, k, kg3, False) for k in keys]
            self.p1 = [cm.conv_plan(k, k, kg1, False) for k in keys]
            self.down = [cm.conv_plan(keys[i], keys[i + 1], kg2, False) for i in range(4)]
            self.up = [cm.conv_plan(keys[i + 1], keys[i], kg2, True) for i in range(4)]
            self.p0 = cm.conv_plan(keys[0], keys[0], m.conv0p1s1.kernel_generator, False)
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
    __slots__ = ("owner", "p", "hi", "lo", "bh", "bl", "n", "C", "ld", "slot", "_grad", "parent", "col", "device")

    def __init__(self, owner, p, n, C, ld, device, hi=0, lo=0, parent=None, col=0, bh=0, bl=0):
        self.owner, self.p, self.hi, self.lo, self.n, self.C, self.ld, self.device = owner, p, hi, lo, n, C, ld, device
        self.bh, self.bl = bh, bl             # me.FWD_FP16: hi/lo are fp16 planes (forward gathers), bh/bl the bf16 planes (weight gradient)
        self.parent, self.col = parent, col
        self._grad = None
        self.slot = parent.slot if parent is not None else [False]     # [gradient buffer initialised?]

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


class _Tape:
    __slots__ = ("units", "arena", "x_last", "p_final", "stats", "geom", "ws")


class Runner:
    def __init__(self, model):
        self.model = model
        self.anchor = torch.zeros(1, requires_grad=True)
        self._fwd_hint = 0
        self._bwd_hint = 0

    # ------------------------------------------------------------------------------------------ single launches (final layer)
    def _conv(self, kind, plan, conv, x, out, bias=None):
        """The final layer's forward ("fwd") or data gradient ("dgrad") into `out`."""
        kern = conv.kernel
        Cin, Cout = kern.shape[1:]
        if Cin % 32 == 0 and Cout % 32 == 0:
            assert x.hi, "tensor-core conv needs the split planes of its input"
            tiles = conv._prepared.tiles(kern, me.FWD_FP16)[0 if kind == "fwd" else 1]
            fp16 = me.FWD_FP16 and kind == "fwd"          # forward roles: fp16 activation planes x fp16 weight tiles
            me.conv(kind, plan, Cin, Cout, (x.hi, x.lo), x.ld, out.p, out.ld, tiles=ptr(tiles), bias=ptr(bias), fp16=fp16)
        else:
            # exact fp32 kernel: output widths the tensor-core tiling does not cover (13 / 20 semantic classes); as a data gradient it
            # runs on the per-offset transposed weights
            assert x.p, "the exact fp32 conv reads the fp32 plane"
            w = kern.detach() if kind == "fwd" else kern.detach().transpose(1, 2).contiguous()
            me.conv(kind, plan, Cin, Cout, x.p, x.ld, out.p, out.ld, w=ptr(w), bias=ptr(bias))

    def _wgrad(self, conv, plan, a_in, dz):
        kern = conv.kernel
        Cin, Cout = kern.shape[1:]
        if kern.grad is None:
            kern.grad = torch.zeros_like(kern)
        if Cin % 32 == 0 and Cout % 32 == 0:
            pl = lambda b: (b.bh, b.bl) if b.bh else (b.hi, b.lo)          # activations: their bf16 planes (gradients only have those)
            me.wgrad(plan, Cin, Cout, pl(a_in), a_in.ld, pl(dz), dz.ld, kern.grad.data_ptr(), True, accumulate=True)
        else:
            me.wgrad(plan, Cin, Cout, a_in.p, a_in.ld, dz.p, dz.ld, kern.grad.data_ptr(), False, accumulate=True)

    # ------------------------------------------------------------------------------------------ forward
    def _unit(self, conv, bnm, a_in, plan, relu, residual=None, out=None, need_f32=False):
        """out = [relu]( BN(conv(a_in)) [+ residual] )   -- one pcb_unit_forward call"""
        bn = bnm.bn
        kern = conv.kernel
        K, Cin, Cout = kern.shape
        n = plan.n_out
        n0 = self.seg_of[id(plan)]                       # rows of view 0 at the output level (== n: a single view)
        nseg = 2 if n0 < n else 1
        arena = self.arena
        tc = Cin % 32 == 0 and Cout % 32 == 0
        z = Buf.new(arena, n, Cout)
        if out is None:
            out = Buf.new(arena, n, Cout, fp32=need_f32, split=True, dual=self.dual)
        u = PcbUnit()
        u.n_in, u.n_out, u.n0 = plan.n_in, n, n0
        u.K, u.Cin, u.Cout, u.relu = K, Cin, Cout, 1 if relu else 0
        u.fwd_tbl, u.fwd_stride = plan.fwd_tbl.data_ptr(), plan.fwd_tbl.shape[1]
        km = plan.c_kmap("fwd_kmap")
        u.fwd_kmap = ctypes.cast(km, ctypes.c_void_p) if km is not None else None
        u.W = kern.data_ptr()
        if tc:
            tiles = conv._prepared.tiles(kern, me.FWD_FP16)
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
        u.mean = self._stat(nseg * Cout)
        u.invstd = self._stat(nseg * Cout)
        u.z_p, u.z_ld = z.p, z.ld
        if out.p:
            u.out_p, u.out_ld = out.p, out.ld
        u.out_hi, u.out_lo, u.out_lds = out.hi, out.lo, out.ld
        if out.bh:
            u.out_bhi, u.out_blo = out.bh, out.bl
        if residual is not None:
            assert residual.p, "a residual input needs its fp32 plane"
            u.res_p, u.res_ld = residual.p, residual.ld
        u.ws, u.ws_bytes = self.ws.data_ptr(), self.ws.numel()
        u.flags = ((_lib.UNIT_SEPARATE_STATS if SEPARATE_STATS else 0) | (_lib.UNIT_FP16_FORWARD if me.FWD_FP16 else 0)
                   | (_lib.UNIT_EVAL if self.eval_mode else 0))
        me.record_profile("fwd", plan, K, Cin, Cout, tc)
        check(lib.pcb_unit_forward(ctypes.byref(u), self.st))
        if CAPTURE_RELU is not None and relu:
            CAPTURE_RELU.append((n0, _plane_i16(out.hi, n, Cout, out.ld, self.device) > 0))
        if not self.eval_mode:
            self.bns.append(bn)
            self.units.append((u, conv, bn, a_in, out, plan, residual))
        return out

    def _refresh_tiles(self):
        """Re-tile the weights of every tensor-core convolution in ONE launch when the parameters changed (after each optimiser
        step) and hand the results to the per-layer caches (`me._PreparedWeights`), instead of one small launch per layer."""
        m = self.model
        convs = [c for c in m.modules() if isinstance(c, me._ConvolutionBase) and c.in_channels % 32 == 0 and c.out_channels % 32 == 0]
        tags = [me._PreparedWeights.tag(c.kernel, me.FWD_FP16) for c in convs]
        if all(c._prepared.tile_tag == t for c, t in zip(convs, tags)):
            return
        cache = self.__dict__.get("_tile_batch")
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

    def _stat(self, C):
        p = self.stats.data_ptr() + 4 * self.stat_off
        self.stat_off += C
        return p

    def _block(self, blk, x, plan3, plan1, out=None, need_f32=False):
        h = self._unit(blk.conv1, blk.norm1, x, plan3, True)
        res = x if blk.downsample is None else self._unit(blk.downsample[0], blk.downsample[1], x, plan1, False, need_f32=True)
        return self._unit(blk.conv2, blk.norm2, h, plan3, True, residual=res, out=out, need_f32=need_f32)

    def _stage(self, seq, x, plan3, plan1, out=None, need_f32=False):
        """A stage of BasicBlocks.  A block's output needs its fp32 plane only if the NEXT block adds it back as the identity
        residual (`resnet_block.py:51-57`: no downsample branch); `need_f32` says so for the stage's own output."""
        blocks = list(seq)
        for i, blk in enumerate(blocks):
            last = i == len(blocks) - 1
            x = self._block(blk, x, plan3, plan1, out if last else None, need_f32 if last else blocks[i + 1].downsample is None)
        return x

    def _ws_bytes(self, g):
        """Scratch for the largest unit of this geometry (the units run back to back on one stream and share it)."""
        m = self.model
        n, best = g.n, 0
        cached = self.__dict__.setdefault("_ws_cache", {})
        if tuple(n) in cached:
            return cached[tuple(n)]
        shapes = {(27, n[0], n[0], m.conv0p1s1.in_channels, m.INIT_DIM)}
        for name, lvl in (("block1", 1), ("block2", 2), ("block3", 3), ("block4", 4), ("block5", 3), ("block6", 2), ("block7", 1), ("block8", 0)):
            for blk in getattr(m, name):
                shapes.add((27, n[lvl], n[lvl], blk.conv1.in_channels, blk.conv1.out_channels))
                shapes.add((27, n[lvl], n[lvl], blk.conv2.in_channels, blk.conv2.out_channels))
                if blk.downsample is not None:
                    shapes.add((1, n[lvl], n[lvl], blk.downsample[0].in_channels, blk.downsample[0].out_channels))
        for i, (dn, upn) in enumerate((("conv1p1s2", "convtr7p2s2"), ("conv2p2s2", "convtr6p4s2"), ("conv3p4s2", "convtr5p8s2"),
                                       ("conv4p8s2", "convtr4p16s2"))):
            d, u = getattr(m, dn), getattr(m, upn)
            shapes.add((8, n[i], n[i + 1], d.in_channels, d.out_channels))
            shapes.add((8, n[i + 1], n[i], u.in_channels, u.out_channels))
        for (K, n_in, n_out, ci, co) in shapes:
            best = max(best, lib.pcb_unit_ws_bytes(K, n_in, n_out, ci, co))
        if len(cached) > 64:
            cached.clear()
        cached[tuple(n)] = best
        return best

    def forward(self, sinput, view0_rows=None, geom=None, eval_mode=False):
        """`view0_rows`: the input is a `stack_views` tensor whose first `view0_rows` rows are view 0.
        `eval_mode`: forward only with eval-mode BatchNorm (running statistics); nothing is kept for a backward pass."""
        m = self.model
        self.eval_mode = eval_mode
        self.dual = me.FWD_FP16 and not eval_mode          # bf16 copies of the activations are only needed by the weight gradient
        feats = sinput.F
        _lib.require_cuda(feats)
        self.device = dev = feats.device
        g = geom if geom is not None else Geometry(m, sinput, view0_rows)
        self.units, self.bns = [], []
        with torch.cuda.device(dev):
            self.st = stream()
            n, seg = g.n, g.seg
            p3, p1, down, up, p0 = g.p3, g.p1, g.down, g.up, g.p0
            self.seg_of = {id(p0): seg[0]}
            for l in range(5):
                self.seg_of[id(p3[l])] = seg[l]
                self.seg_of[id(p1[l])] = seg[l]
            for i in range(4):
                self.seg_of[id(down[i])] = seg[i + 1]
                self.seg_of[id(up[i])] = seg[i]
            self.stats = torch.empty(4 * sum(mod.bn.num_features for mod in m.modules() if isinstance(mod, me.MinkowskiBatchNorm)),
                                     dtype=torch.float32, device=dev)
            self.stat_off = 0
            self.ws = _lib.workspace(self._ws_bytes(g), dev)
            self._refresh_tiles()
            self.arena = arena = Arena(dev, self._fwd_hint)
            P = m.PLANES
            x_in = feats.detach().contiguous().float()
            a0 = Buf(x_in, x_in.data_ptr(), n[0], x_in.shape[1], x_in.shape[1], dev)
            a0.slot[0] = None                    # network input: no gradient wanted
            fin = m.final
            fin_tc = fin.in_channels % 32 == 0 and fin.out_channels % 32 == 0
            # concatenation buffers (left = decoder branch, right = encoder skip); consumed by convolutions only: split planes
            cat8 = Buf.new(arena, n[0], P[7] + m.INIT_DIM, fp32=False, split=True, dual=self.dual)
            cat7 = Buf.new(arena, n[1], P[6] + P[0], fp32=False, split=True, dual=self.dual)
            cat6 = Buf.new(arena, n[2], P[5] + P[1], fp32=False, split=True, dual=self.dual)
            cat5 = Buf.new(arena, n[3], P[4] + P[2], fp32=False, split=True, dual=self.dual)
            out_p1 = self._unit(m.conv0p1s1, m.bn0, a0, p0, True, out=cat8.cols(P[7], m.INIT_DIM))
            x = self._unit(m.conv1p1s2, m.bn1, out_p1, down[0], True, need_f32=m.block1[0].downsample is None)
            b1 = self._stage(m.block1, x, p3[1], p1[1], out=cat7.cols(P[6], P[0]))
            x = self._unit(m.conv2p2s2, m.bn2, b1, down[1], True, need_f32=m.block2[0].downsample is None)
            b2 = self._stage(m.block2, x, p3[2], p1[2], out=cat6.cols(P[5], P[1]))
            x = self._unit(m.conv3p4s2, m.bn3, b2, down[2], True, need_f32=m.block3[0].downsample is None)
            b3 = self._stage(m.block3, x, p3[3], p1[3], out=cat5.cols(P[4], P[2]))
            x = self._unit(m.conv4p8s2, m.bn4, b3, down[3], True, need_f32=m.block4[0].downsample is None)
            x = self._stage(m.block4, x, p3[4], p1[4])
            self._unit(m.convtr4p16s2, m.bntr4, x, up[3], True, out=cat5.cols(0, P[4]))
            x = self._stage(m.block5, cat5, p3[3], p1[3])
            self._unit(m.convtr5p8s2, m.bntr5, x, up[2], True, out=cat6.cols(0, P[5]))
            x = self._stage(m.block6, cat6, p3[2], p1[2])
            self._unit(m.convtr6p4s2, m.bntr6, x, up[1], True, out=cat7.cols(0, P[6]))
            x = self._stage(m.block7, cat7, p3[1], p1[1])
            self._unit(m.convtr7p2s2, m.bntr7, x, up[0], True, out=cat8.cols(0, P[7]))
            x = self._stage(m.block8, cat8, p3[0], p1[0], need_f32=not fin_tc)
            out_t = torch.empty(n[0], fin.out_channels, dtype=torch.float32, device=dev)
            out = Buf(out_t, out_t.data_ptr(), n[0], fin.out_channels, fin.out_channels, dev)
            self._conv("fwd", p1[0], fin, x, out, bias=fin.bias.detach().reshape(-1) if fin.bias is not None else None)
            if self.bns:
                torch._foreach_add_([bn.num_batches_tracked for bn in self.bns], g.calls)       # one multi-tensor launch, not 62
        self._fwd_hint = _grow_hint(self._fwd_hint, arena.total)
        if eval_mode:
            self.units = self.arena = self.stats = None
            return out_t, None
        tape = _Tape()
        # the units' u.ws is used again by the backward sweep, and a later, larger request replaces the cached buffer: the tape holds it
        tape.units, tape.arena, tape.x_last, tape.p_final, tape.stats, tape.geom, tape.ws = self.units, arena, x, p1[0], self.stats, g, self.ws
        self.units = self.arena = self.stats = None
        return out_t, tape

    # ------------------------------------------------------------------------------------------ backward
    def backward(self, tape, d_out):
        m = self.model
        d_out = d_out.contiguous()
        dev = d_out.device
        self.device = dev
        x_last, p_final = tape.x_last, tape.p_final
        with torch.cuda.device(dev):
            st = stream()
            arena = Arena(dev, self._bwd_hint)
            fin = m.final
            if fin.out_channels % 32 == 0:
                dfin = Buf.new(arena, d_out.shape[0], d_out.shape[1], fp32=False, split=True)
                check(lib.pcb_split_rows(d_out.data_ptr(), d_out.shape[1], d_out.shape[0], d_out.shape[1], dfin.hi, dfin.lo, dfin.ld, 0, st))
            else:                                # e.g. 13 / 20 classes: the final layer's backward runs on the exact fp32 kernels
                dfin = Buf(d_out, d_out.data_ptr(), d_out.shape[0], d_out.shape[1], d_out.shape[1], dev)
            if fin.bias is not None:
                if fin.bias.grad is None:
                    fin.bias.grad = torch.zeros_like(fin.bias)
                fin.bias.grad += d_out.sum(0, keepdim=True)
            self._wgrad(fin, p_final, x_last, dfin)
            gx = x_last.grad(arena)
            self._conv("dgrad", p_final, fin, dfin, gx)
            x_last.slot[0] = True
            after_unit = m.__dict__.get("_fused_after_unit")       # trainer hook: gradient all-reduce of the chunk this unit completes
            for (u, conv, bn, a_in, out, plan, residual) in reversed(tape.units):
                kern = conv.kernel
                g = out.grad(arena)
                assert out.slot[0], "gradient of a unit output was never produced"
                tc = u.Cin % 32 == 0 and u.Cout % 32 == 0
                n, Cout = u.n_out, u.Cout
                u.g_p, u.g_ld = g.p, g.ld
                dz = Buf.new(arena, n, Cout, fp32=not tc, split=tc)       # consumed only by the conv kernels: split planes suffice
                u.dz_p, u.dz_hi, u.dz_lo, u.dz_ld = dz.p or None, dz.hi or None, dz.lo or None, dz.ld
                u.gres_p, u.gres_ld, u.gres_mode = None, 0, 0
                if residual is not None and residual.slot[0] is not None:
                    rg = residual.grad(arena)
                    u.gres_p, u.gres_ld = rg.p, rg.ld
                    u.gres_mode = 2 if residual.slot[0] else 1
                    residual.slot[0] = True
                for prm in (bn.weight, bn.bias, kern):
                    if prm.grad is None:
                        prm.grad = torch.zeros_like(prm)
                u.dgamma, u.dbeta, u.dW = bn.weight.grad.data_ptr(), bn.bias.grad.data_ptr(), kern.grad.data_ptr()
                u.wg_tbl, u.wg_stride, u.wg_gather_x = plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], 1 if plan.wg_gather_x else 0
                u.gin_p, u.gin_ld, u.gin_mode = None, 0, 0
                if a_in.slot[0] is not None:
                    ga = a_in.grad(arena)
                    u.gin_p, u.gin_ld, u.gin_mode = ga.p, ga.ld, 2 if a_in.slot[0] else 1
                    a_in.slot[0] = True
                    u.dg_tbl, u.dg_stride = plan.dg_tbl.data_ptr(), plan.dg_tbl.shape[1]
                    km = plan.c_kmap("dg_kmap")
                    u.dg_kmap = ctypes.cast(km, ctypes.c_void_p) if km is not None else None
                me.record_profile("wgrad", plan, u.K, u.Cin, u.Cout, tc)
                if u.gin_mode:
                    me.record_profile("dgrad", plan, u.K, u.Cin, u.Cout, tc)
                check(lib.pcb_unit_backward(ctypes.byref(u), st))
                if after_unit is not None:
                    after_unit(conv)
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


_STAGES = ("block1", "block2", "block3", "block4", "block5", "block6", "block7", "block8")
_UNITS = (("conv0p1s1", "bn0"), ("conv1p1s2", "bn1"), ("conv2p2s2", "bn2"), ("conv3p4s2", "bn3"), ("conv4p8s2", "bn4"),
          ("convtr4p16s2", "bntr4"), ("convtr5p8s2", "bntr5"), ("convtr6p4s2", "bntr6"), ("convtr7p2s2", "bntr7"))


def matches(model):
    """Is `model` wired like `pretrain/pointcontrast/model/res16unet.py:36-268` (Res16UNet with BasicBlock stages)?  The
    executor reads the graph from the attribute names, so ANY class with this wiring -- this package's model file or the
    reference's own, unmodified -- runs fused.  Also checks what the tensor-core tiling needs (all hidden widths % 32)."""
    ok = model.__dict__.get("_fused_ok")
    if ok is None:
        ok = _matches(model)
        model.__dict__["_fused_ok"] = ok
    return ok


def _matches(m):
    try:
        for c, b in _UNITS:
            if not isinstance(getattr(m, c), me._ConvolutionBase) or not isinstance(getattr(m, b), me.MinkowskiBatchNorm):
                return False
        if not isinstance(m.final, me.MinkowskiConvolution) or m.final.kernel_volume != 1:
            return False
        widths = [m.INIT_DIM] + list(m.PLANES)
        for name in _STAGES:
            for blk in getattr(m, name):
                if not all(isinstance(getattr(blk, a), t) for a, t in (("conv1", me.MinkowskiConvolution), ("conv2", me.MinkowskiConvolution),
                                                                       ("norm1", me.MinkowskiBatchNorm), ("norm2", me.MinkowskiBatchNorm))):
                    return False
                if hasattr(blk, "conv3") or (blk.downsample is not None and len(blk.downsample) != 2):
                    return False
                widths += [blk.conv1.in_channels, blk.conv1.out_channels, blk.conv2.out_channels]
        if m.conv0p1s1.out_channels != m.INIT_DIM or m.final.in_channels != m.PLANES[7]:
            return False
        return all(w % 32 == 0 for w in widths) and m.conv0p1s1.in_channels % 32 != 0      # exact fp32 stem (3 input channels)
    except (AttributeError, TypeError):
        return False


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
