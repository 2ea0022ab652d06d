"""VoteNet's PointNet++ set-abstraction and feature-propagation modules on libpcb200 (DESIGN.md 8f-16): the shared MLPs
(`pytorch_utils.SharedMLP`: 1x1 Conv2d -> BatchNorm2d -> ReLU per layer) and the max pool of `pointnet2_modules.py` as one autograd node
per module forward, in place of the original's torch layers.

    from pointcontrast_b200 import pointnet2_modules
    pointnet2_modules.install()     # `import pointnet2_modules` (backbone_module.py, proposal_module.py) now resolves here

`PointnetSAModuleVotes` and `PointnetFPModule` take the original's keyword arguments and return what it returns; their parameters and
buffers have the original's names, order, shapes, dtypes and seeded initial values, held by real nn.Conv2d / nn.BatchNorm2d modules, so
original checkpoints load, optimiser state lines up and BNMomentumScheduler reaches them.  Each forward reads `bn.momentum`, honours
train() / eval() and counts `num_batches_tracked` as nn.BatchNorm2d does.  Eval mode is forward only (run it under torch.no_grad(), as
VoteNet's evaluation does).

Set abstraction, rows r = (centre, sample) of the ball-query neighbourhoods:
  * layer 0 applies its feature columns to every POINT once (exact fp32 K = 1 convolution), then `pcb_sa_layer0` adds the relative-xyz
    columns per row: the grouped [R, 3 + C] input is never built;
  * the middle layers are fused units (`pcb_unit_forward`, K = 1 identity table, fp16 hi/lo forward operands);
  * the last layer's convolution writes z, and `pcb_sa_pool` picks per (centre, channel) the sample on gamma's side of z and normalises
    only that one: the normalised [R, C] tensor is never written.
The backward sweep is hand-written and deterministic; it reaches the features, every parameter and xyz (through the relative
coordinates and through new_xyz).  Outputs are channel-major views of point-major storage, so the set-abstraction modules pass features
to each other without a transpose copy; the feature-propagation module still copies its inputs into one point-major buffer.

Supported: what VoteNet builds -- pooling='max', bn=True, use_xyz=True, npoint set, normalize_xyz either way, features None or given,
hidden and output widths multiples of 32 (the tensor-core tiling); PointnetFPModule with `known` given and a first-layer width that is a
multiple of 32.  Any other option raises at construction (or, for `known=None`, at the call).
"""
import ctypes
import sys

import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib, me, pointnet2
from ._lib import PcbError, PcbUnit, check, lib, ptr, stream, workspace
from .det_eval import register

ext = pointnet2.ext
_F16 = _lib.PLANES_A_FP16 | _lib.PLANES_B_FP16


# ------------------------------------------------------------------------------------------------ parameters (the original's tree)
def _layer(cin, cout):
    """`pytorch_utils.Conv2d(cin, cout, bn=True)`: conv (bias-free, kaiming-normal), bn.bn (weight 1, bias 0), activation -- built in the
    original's order, so a seeded construction draws the same numbers."""
    layer = nn.Sequential()
    conv = nn.Conv2d(cin, cout, kernel_size=(1, 1), stride=(1, 1), padding=(0, 0), bias=False)
    nn.init.kaiming_normal_(conv.weight)
    bn = nn.Sequential()
    bn.add_module("bn", nn.BatchNorm2d(cout))
    nn.init.constant_(bn[0].weight, 1.0)
    nn.init.constant_(bn[0].bias, 0)
    layer.add_module("conv", conv)
    layer.add_module("bn", bn)
    layer.add_module("activation", nn.ReLU(inplace=True))
    return layer


def _shared_mlp(spec):
    """The parameter tree of `pytorch_utils.SharedMLP(spec, bn=True)`.  It holds the parameters; the forward pass is this module's."""
    mlp = nn.Sequential()
    for i in range(len(spec) - 1):
        mlp.add_module(f"layer{i}", _layer(spec[i], spec[i + 1]))
    return mlp


def _check_widths(spec, first):
    bad = [w for w in spec[first:] if w % 32]
    if bad:
        raise NotImplementedError(f"mlp={spec}: widths {bad} are not multiples of 32 (the tensor-core tiling of the shared MLP)")


def _layers(mlp):
    """[(conv, bn)] of a shared-MLP tree, in order."""
    return [(layer.conv, layer.bn.bn) for layer in mlp]


def _params(mlp):
    return [t for conv, bn in _layers(mlp) for t in (conv.weight, bn.weight, bn.bias)]


def _momentum(bn):
    if bn.momentum is None:
        raise NotImplementedError("BatchNorm2d with momentum=None (cumulative average) is not supported")
    return float(bn.momentum)


# ------------------------------------------------------------------------------------------------ native building blocks
_IDENT = {}


def _identity(n, device):
    """int32 [1, >= n] identity table: a K = 1 convolution over it is a per-row matrix product (tbl_stride = its length)."""
    t = _IDENT.get(device.index)
    if t is None or t.shape[1] < n:
        t = _IDENT[device.index] = torch.arange(max(int(n), 1 << 16), dtype=torch.int32, device=device).view(1, -1)
    return t


def _pad32(n):
    return (n + 31) // 32 * 32


def _tiles(conv):
    """(weights [Cin][Cout], forward tiles (fp16 x 2^10), data-gradient tiles) of a 1x1 conv, rebuilt whenever the weight or bias
    changes: its version counter moves on every in-place update (an optimiser step), a raw-pointer rewrite bumps me's weights epoch.
    A conv with a bias gets 32 more input rows: row Cin holds the bias (its input column is constant 1), the rest are zero; output
    columns are padded with zeros to a multiple of 32."""
    w, bias = conv.weight, conv.bias
    tag = (w.data_ptr(), w._version, me._WEIGHTS_EPOCH[0]) + (() if bias is None else (bias.data_ptr(), bias._version))
    cache = conv.__dict__.get("_pcb_tiles")
    if cache is None or cache[0] != tag:
        cout, cin = w.shape[:2]
        wl = w.detach().reshape(cout, cin).t().contiguous()
        if bias is not None or cout % 32:
            full = torch.zeros(cin + (0 if bias is None else 32), _pad32(cout), dtype=torch.float32, device=w.device)
            full[:cin, :cout] = wl
            if bias is not None:
                full[cin, :cout] = bias.detach()
            wl = full
        cin, cout = wl.shape
        f = torch.empty(lib.pcb_weight_tile_bytes(1, cin, cout, 0), dtype=torch.uint8, device=w.device)
        d = torch.empty(lib.pcb_weight_tile_bytes(1, cin, cout, 1), dtype=torch.uint8, device=w.device)
        check(lib.pcb_weight_tile(ptr(wl), 1, cin, cout, ptr(f), ptr(d), _lib.PLANES_B_FP16, stream()))
        cache = conv.__dict__["_pcb_tiles"] = (tag, wl, f, d)
    return cache[1:]


class _Planes:
    """An activation [n, C] as fp16 hi/lo planes (forward gathers) and, when a backward pass follows, bf16 hi/lo planes (weight gradient)."""

    def __init__(self, n, C, device, dual):
        self.t = torch.empty(4 if dual else 2, n, C, dtype=torch.int16, device=device)
        self.n, self.C, self.dual = n, C, dual

    def ptrs(self):
        p = [self.t[k].data_ptr() for k in range(self.t.shape[0])]
        return p + [None, None] if not self.dual else p


def _stats(bn, z, n, C, train, ws_dev):
    """mean / invstd [C] of z [n, C] (training: batch statistics, running statistics updated with bn.momentum) or the running ones."""
    mean = torch.empty(C, dtype=torch.float32, device=z.device)
    invstd = torch.empty_like(mean)
    if train:
        wsb = lib.pcb_bn_ws_bytes(n, C)
        ws = workspace(wsb, ws_dev)
        check(lib.pcb_bn_stats_seg(ptr(z), C, n, n, C, bn.eps, _momentum(bn), ptr(mean), ptr(invstd), ptr(bn.running_mean),
                                   ptr(bn.running_var), ptr(ws), wsb, stream()))
    else:
        mean.copy_(bn.running_mean)
        torch.reciprocal(torch.sqrt(bn.running_var + bn.eps), out=invstd)
    return mean, invstd


def _unit(n, tbl, conv, bn, x, out, z, mean, invstd, train, out_p=None):
    """pcb_unit of one K = 1 layer over n rows: x / out are _Planes, z fp32 [n, Cout].  With a conv bias, x carries the constant
    columns _tiles' bias row reads (x.C = Cin + 32)."""
    wl, tf, td = _tiles(conv)
    cin, cout = wl.shape
    u = PcbUnit()
    u.keep = (tbl, wl, tf, td)                # the backward call reads the table and the tiles of the forward's weights
    u.n_in = u.n_out = u.n0 = n
    u.K, u.Cin, u.Cout, u.relu = 1, cin, cout, 1
    u.fwd_tbl = u.dg_tbl = u.wg_tbl = tbl.data_ptr()
    u.fwd_stride = u.dg_stride = u.wg_stride = tbl.shape[1]
    u.wg_gather_x = 1
    u.W, u.wt_fwd, u.wt_dg = wl.data_ptr(), tf.data_ptr(), td.data_ptr()
    u.gamma, u.beta = bn.weight.data_ptr(), bn.bias.data_ptr()
    u.running_mean, u.running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
    u.eps, u.momentum = bn.eps, _momentum(bn)
    u.mean, u.invstd = mean.data_ptr(), invstd.data_ptr()
    u.x_hi, u.x_lo, u.x_bhi, u.x_blo = x.ptrs()
    u.x_lds = x.C
    u.z_p, u.z_ld = z.data_ptr(), cout
    u.out_hi, u.out_lo, u.out_bhi, u.out_blo = out.ptrs()
    u.out_lds = out.C
    if out_p is not None:
        u.out_p, u.out_ld = out_p.data_ptr(), cout
    u.flags = _lib.UNIT_FP16_FORWARD | (0 if train else _lib.UNIT_EVAL)
    return u


def _run_unit(u, dev, backward=False):
    wsb = lib.pcb_unit_ws_bytes(1, u.n_in, u.n_out, u.Cin, u.Cout)
    ws = workspace(wsb, dev)
    u.ws, u.ws_bytes = ws.data_ptr(), ws.numel()
    check((lib.pcb_unit_backward if backward else lib.pcb_unit_forward)(ctypes.byref(u), stream()))


def _conv_grads(conv, dW):
    """The parameter gradients of a 1x1 conv from dW [Cin(+32)][Cout(pad)] in _tiles' layout: (weight,) or (weight, bias)."""
    cout, cin = conv.weight.shape[:2]
    dw = dW[:cin, :cout].t().reshape(conv.weight.shape)
    return (dw,) if conv.bias is None else (dw, dW[cin, :cout])


def _unit_backward(u, conv, bn, g, gin, dev, gin_mode=1):
    """Backward of a forward unit `u`: g = gradient of its output (fp32 [n, Cout], row stride g.stride(0)) -> gin (fp32 [n, Cin],
    written (gin_mode 1) or accumulated (2)) and the parameter gradients (returned: _conv_grads, then dgamma, dbeta)."""
    n, cin, cout = u.n_out, u.Cin, u.Cout
    dzt = torch.empty(2, n, cout, dtype=torch.int16, device=dev)
    dW = torch.zeros(cin, cout, dtype=torch.float32, device=dev)
    dgamma = torch.zeros(cout, dtype=torch.float32, device=dev)
    dbeta = torch.zeros_like(dgamma)
    u.g_p, u.g_ld = g.data_ptr(), g.stride(0)
    u.dz_hi, u.dz_lo, u.dz_ld = dzt[0].data_ptr(), dzt[1].data_ptr(), cout
    u.dW, u.dgamma, u.dbeta = dW.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr()
    u.gin_p, u.gin_ld, u.gin_mode = gin.data_ptr(), cin, gin_mode
    u.gres_mode = 0
    _run_unit(u, dev, backward=True)
    return _conv_grads(conv, dW) + (dgamma, dbeta)


def _eval_forward_only(params):
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        raise NotImplementedError("eval-mode PointNet++ modules run forward only: call them under torch.no_grad()")


# ------------------------------------------------------------------------------------------------ set abstraction
class _SAFunction(Function):
    @staticmethod
    def forward(ctx, mod, xyz, features, inds, *params):
        dev = xyz.device
        st = stream()
        train = mod.training
        layers = _layers(mod.mlp_module)
        B, N, _ = xyz.shape
        npoint, S = mod.npoint, mod.nsample
        M, R = B * npoint, B * npoint * mod.nsample
        radius = float(mod.radius) if mod.normalize_xyz else 0.0
        x = xyz.detach().contiguous()
        new_xyz = ext.gather_points(x.transpose(1, 2).contiguous(), inds).transpose(1, 2).contiguous()
        idx = ext.ball_query(new_xyz, x, mod.radius, S)
        tbl = _identity(max(R, B * N), dev)
        C = 0 if features is None else features.shape[1]
        F = None if features is None else features.detach().transpose(1, 2).reshape(B * N, C).contiguous()

        # layer 0: feature columns per point, xyz columns per row
        conv0, bn0 = layers[0]
        C0 = conv0.weight.shape[0]
        W0 = conv0.weight.detach().reshape(C0, 3 + C)
        P = None
        if C:
            P = torch.empty(B * N, C0, dtype=torch.float32, device=dev)
            wf = W0[:, 3:].t().contiguous()
            check(lib.pcb_conv_forward(ptr(F), C, ptr(tbl), tbl.shape[1], None, 1, B * N, C, C0, ptr(wf), None, ptr(P), C0, st))
        wx = W0[:, :3].t().contiguous()
        rel = torch.empty(R, 3, dtype=torch.float32, device=dev)
        rows_idx = torch.empty(R + M, dtype=torch.int32, device=dev)
        z0 = torch.empty(R, C0, dtype=torch.float32, device=dev)
        check(lib.pcb_sa_layer0(ptr(x), ptr(new_xyz), ptr(idx), B, N, npoint, S, radius, ptr(P), C0, ptr(wx), C0, ptr(rel), ptr(rows_idx),
                                ptr(z0), C0, st))
        rows_idx[R:] = (inds + torch.arange(B, dtype=torch.int32, device=dev).view(B, 1) * N).view(-1)
        mean0, invstd0 = _stats(bn0, z0, R, C0, train, dev)
        a0 = _Planes(R, C0, dev, train)
        h, l, bh, bl = a0.ptrs()
        check(lib.pcb_bn_apply_seg(ptr(z0), C0, R, R, C0, ptr(mean0), ptr(invstd0), ptr(bn0.weight), ptr(bn0.bias), None, 0,
                                   _lib.BN_RELU | _lib.PLANES_A_FP16, None, 0, h, l, C0, bh, bl, st))

        # middle layers: fused units
        acts, units, zs = [a0], [], []
        for conv, bn in layers[1:-1]:
            cout = conv.weight.shape[0]
            z = torch.empty(R, cout, dtype=torch.float32, device=dev)
            mean = torch.empty(cout, dtype=torch.float32, device=dev)
            invstd = torch.empty_like(mean)
            out = _Planes(R, cout, dev, train)
            u = _unit(R, tbl, conv, bn, acts[-1], out, z, mean, invstd, train)
            _run_unit(u, dev)
            acts.append(out)
            units.append(u)
            zs.append((z, mean, invstd))

        # last layer: convolution, statistics, pooled by selection
        convL, bnL = layers[-1]
        CL, cin = convL.weight.shape[:2]
        tilesL = _tiles(convL)
        tf = tilesL[1]
        zL = torch.empty(R, CL, dtype=torch.float32, device=dev)
        h, l = acts[-1].ptrs()[:2]
        wsb = lib.pcb_conv_forward_split_ws_bytes(1, R, cin, CL)
        ws = workspace(wsb, dev)
        check(lib.pcb_conv_forward_split(h, l, cin, ptr(tbl), tbl.shape[1], None, 1, R, cin, CL, ptr(tf), None, ptr(zL), CL, ptr(ws), wsb,
                                         _F16, st))
        meanL, invstdL = _stats(bnL, zL, R, CL, train, dev)
        sel = torch.empty(M, CL, dtype=torch.int32, device=dev)
        pooled = torch.empty(M, CL, dtype=torch.float32, device=dev)
        check(lib.pcb_sa_pool(ptr(zL), CL, M, S, CL, ptr(meanL), ptr(invstdL), ptr(bnL.weight), ptr(bnL.bias), ptr(sel), ptr(pooled), CL, st))
        if train:
            torch._foreach_add_([bn.num_batches_tracked for _, bn in layers], 1)
            ctx.state = (mod, B, N, C, npoint, S, radius, tbl, F, W0, rel, rows_idx, z0, mean0, invstd0, acts, units, zs, zL, meanL,
                         invstdL, sel, pooled, tilesL)
        return new_xyz, pooled.view(B, npoint, CL)

    @staticmethod
    def backward(ctx, d_new_xyz, d_pooled):
        (mod, B, N, C, npoint, S, radius, tbl, F, W0, rel, rows_idx, z0, mean0, invstd0, acts, units, zs, zL, meanL, invstdL, sel,
         pooled, tilesL) = ctx.state
        ctx.state = None
        dev = zL.device
        st = stream()
        layers = _layers(mod.mlp_module)
        M, R = B * npoint, B * npoint * S
        grads = []

        # last layer: pool -> BatchNorm backward -> weight and data gradients
        convL, bnL = layers[-1]
        CL, cin = convL.weight.shape[:2]
        g = d_pooled.reshape(M, CL).contiguous()
        dY = torch.empty(R, CL, dtype=torch.float32, device=dev)
        check(lib.pcb_sa_pool_grad(ptr(g), CL, ptr(sel), ptr(pooled), CL, M, S, CL, ptr(dY), st))
        dz = torch.empty(2, R, CL, dtype=torch.int16, device=dev)
        dgL, dbL = torch.zeros(CL, dtype=torch.float32, device=dev), torch.zeros(CL, dtype=torch.float32, device=dev)
        wsb = lib.pcb_bn_ws_bytes(R, CL)
        ws = workspace(wsb, dev)
        check(lib.pcb_bn_backward_seg(ptr(dY), CL, ptr(zL), CL, None, 0, R, R, CL, ptr(meanL), ptr(invstdL), ptr(bnL.weight), None, 0,
                                      ptr(dgL), ptr(dbL), 1, None, 0, 0, dz[0].data_ptr(), dz[1].data_ptr(), CL, ptr(ws), wsb, st))
        del dY
        dWL = torch.zeros(cin, CL, dtype=torch.float32, device=dev)
        _, _, bh, bl = acts[-1].ptrs()
        wsb = lib.pcb_conv_wgrad_split_ws_bytes(1, R, cin, CL)
        ws = workspace(wsb, dev)
        check(lib.pcb_conv_wgrad_split(bh, bl, cin, dz[0].data_ptr(), dz[1].data_ptr(), CL, ptr(tbl), tbl.shape[1], 1, R, cin, CL, ptr(dWL),
                                       0, ptr(ws), wsb, _lib.CONV_ACCUMULATE, st))
        td = tilesL[2]
        g = torch.empty(R, cin, dtype=torch.float32, device=dev)
        wsb = lib.pcb_conv_forward_split_ws_bytes(1, R, CL, cin)
        ws = workspace(wsb, dev)
        check(lib.pcb_conv_forward_split(dz[0].data_ptr(), dz[1].data_ptr(), CL, ptr(tbl), tbl.shape[1], None, 1, R, CL, cin, ptr(td), None,
                                         ptr(g), cin, ptr(ws), wsb, 0, st))
        del dz
        grads.append((dWL.t().reshape(CL, cin, 1, 1), dgL, dbL))

        # middle units, last to first
        for (conv, bn), u in zip(reversed(layers[1:-1]), reversed(units)):
            gin = torch.empty(R, u.Cin, dtype=torch.float32, device=dev)
            grads.append(_unit_backward(u, conv, bn, g, gin, dev))
            g = gin

        # layer 0: BatchNorm (ReLU mask from the fp16 hi plane) -> dz0
        conv0, bn0 = layers[0]
        C0 = conv0.weight.shape[0]
        dz0 = torch.empty(R, C0, dtype=torch.float32, device=dev)
        dg0, db0 = torch.zeros(C0, dtype=torch.float32, device=dev), torch.zeros(C0, dtype=torch.float32, device=dev)
        wsb = lib.pcb_bn_ws_bytes(R, C0)
        ws = workspace(wsb, dev)
        check(lib.pcb_bn_backward_seg(ptr(g), C0, ptr(z0), C0, acts[0].ptrs()[0], C0, R, R, C0, ptr(mean0), ptr(invstd0), ptr(bn0.weight),
                                      ptr(dz0), C0, ptr(dg0), ptr(db0), 1, None, 0, 0, None, None, 0, ptr(ws), wsb, st))
        del g
        # xyz columns: dWx = rel^T dz0; the gradient of rel = dz0 Wx
        dWx = torch.empty(C0, 3, dtype=torch.float32, device=dev)
        wsb = lib.pcb_conv_wgrad_ws_bytes(1, R, 3, C0)
        ws = workspace(wsb, dev)
        check(lib.pcb_conv_wgrad(ptr(rel), 3, ptr(dz0), C0, ptr(tbl), tbl.shape[1], 1, R, 3, C0, ptr(dWx), 1, ptr(ws), wsb, 0, st))
        d_xyz = None
        if ctx.needs_input_grad[1]:
            grel = torch.empty(R, 3, dtype=torch.float32, device=dev)
            wx = W0[:, :3].contiguous()
            check(lib.pcb_conv_forward(ptr(dz0), C0, ptr(tbl), tbl.shape[1], None, 1, R, C0, 3, ptr(wx), None, ptr(grel), 3, st))
            rows = torch.empty(R + M, 3, dtype=torch.float32, device=dev)
            dn = d_new_xyz.reshape(M, 3).contiguous() if d_new_xyz is not None else None
            check(lib.pcb_sa_xyz_rows(ptr(grel), ptr(dn), M, S, radius, ptr(rows), st))
            d_xyz = pointnet2.gather_rows_grad(rows, rows_idx, B * N).view(B, N, 3)
        # feature columns: dP = the gather's adjoint, dWf = F^T dP, dF = dP Wf
        dW0, d_feat = dWx, None
        if C:
            dP = pointnet2.gather_rows_grad(dz0, rows_idx[:R], B * N)
            dWf = torch.empty(C0, C, dtype=torch.float32, device=dev)
            wsb = lib.pcb_conv_wgrad_ws_bytes(1, B * N, C, C0)
            ws = workspace(wsb, dev)
            check(lib.pcb_conv_wgrad(ptr(F), C, ptr(dP), C0, ptr(tbl), tbl.shape[1], 1, B * N, C, C0, ptr(dWf), 1, ptr(ws), wsb, 0, st))
            dW0 = torch.cat([dWx, dWf], 1)
            if ctx.needs_input_grad[2]:
                dF = torch.empty(B * N, C, dtype=torch.float32, device=dev)
                wf = W0[:, 3:].contiguous()
                check(lib.pcb_conv_forward(ptr(dP), C0, ptr(tbl), tbl.shape[1], None, 1, B * N, C0, C, ptr(wf), None, ptr(dF), C, st))
                d_feat = dF.view(B, N, C).transpose(1, 2)
        grads.append((dW0.reshape(C0, 3 + C, 1, 1), dg0, db0))
        return (None, d_xyz, d_feat, None) + tuple(t for layer in reversed(grads) for t in layer)


class PointnetSAModuleVotes(nn.Module):
    """`pointnet2_modules.PointnetSAModuleVotes` on this library (see the module docstring for what is supported)."""

    def __init__(self, *, mlp, npoint=None, radius=None, nsample=None, bn=True, use_xyz=True, pooling="max", sigma=None, normalize_xyz=False,
                 sample_uniformly=False, ret_unique_cnt=False):
        super().__init__()
        for name, bad in (("pooling", pooling != "max"), ("bn", not bn), ("use_xyz", not use_xyz), ("npoint", npoint is None),
                          ("sample_uniformly", sample_uniformly), ("ret_unique_cnt", ret_unique_cnt), ("mlp", len(mlp) < 3)):
            if bad:
                raise NotImplementedError(f"PointnetSAModuleVotes({name}={locals()[name]!r}) is not supported on this library "
                                          "(max pooling, bn=True, use_xyz=True, npoint set, no uniform sampling, at least two layers)")
        self.npoint, self.radius, self.nsample, self.pooling = npoint, radius, nsample, pooling
        self.use_xyz, self.sigma, self.normalize_xyz, self.ret_unique_cnt = use_xyz, radius / 2 if sigma is None else sigma, normalize_xyz, False
        mlp[0] += 3                                   # on the caller's list, as the original does
        _check_widths(mlp, 1)
        self.mlp_module = _shared_mlp(mlp)

    def forward(self, xyz, features=None, inds=None):
        """xyz fp32 [B, N, 3], features [B, C, N] or None, inds int32 [B, npoint] or None (furthest-point sampling) ->
        (new_xyz [B, npoint, 3], new_features [B, mlp[-1], npoint] (a view of point-major storage), inds int32 [B, npoint])."""
        _lib.require_cuda(xyz)
        if xyz.dtype != torch.float32 or (features is not None and features.dtype != torch.float32):
            raise PcbError("PointnetSAModuleVotes takes fp32 xyz and features")
        c_in = self.mlp_module.layer0.conv.in_channels - 3
        if (0 if features is None else features.shape[1]) != c_in:
            raise PcbError(f"features have {0 if features is None else features.shape[1]} channels, the first layer expects {c_in}")
        params = _params(self.mlp_module)
        if not self.training:
            _eval_forward_only(params + [xyz] + ([features] if features is not None else []))
        if inds is None:
            inds = pointnet2.furthest_point_sample(xyz.detach().contiguous(), self.npoint)
        else:
            assert inds.shape[1] == self.npoint
        new_xyz, pooled = _SAFunction.apply(self, xyz, features, inds.to(torch.int32).contiguous(), *params)
        return new_xyz, pooled.transpose(1, 2), inds


# ------------------------------------------------------------------------------------------------ feature propagation
class _FPFunction(Function):
    @staticmethod
    def forward(ctx, mod, known_feats, unknow_feats, idx, weight, *params):
        dev = known_feats.device
        st = stream()
        train = mod.training
        layers = _layers(mod.mlp)
        B, C2, m = known_feats.shape
        n = idx.shape[1]
        C1 = 0 if unknow_feats is None else unknow_feats.shape[1]
        rows, ctot = B * n, C2 + C1
        tbl = _identity(rows, dev)
        x = torch.empty(B, n, ctot, dtype=torch.float32, device=dev)
        x[:, :, :C2] = ext.three_interpolate(known_feats.detach().contiguous(), idx, weight).transpose(1, 2)
        if C1:
            x[:, :, C2:] = unknow_feats.detach().transpose(1, 2)
        a = _Planes(rows, ctot, dev, train)
        h, l, bh, bl = a.ptrs()
        check(lib.pcb_split_rows(ptr(x), ctot, rows, ctot, h, l, ctot, _lib.PLANES_A_FP16, st))
        if train:
            check(lib.pcb_split_rows(ptr(x), ctot, rows, ctot, bh, bl, ctot, 0, st))
        del x
        acts, units = [a], []
        out_p = None
        for k, (conv, bn) in enumerate(layers):
            cout = conv.weight.shape[0]
            last = k == len(layers) - 1
            z = torch.empty(rows, cout, dtype=torch.float32, device=dev)
            mean = torch.empty(cout, dtype=torch.float32, device=dev)
            invstd = torch.empty_like(mean)
            out = _Planes(rows, cout, dev, train)
            out_p = torch.empty(rows, cout, dtype=torch.float32, device=dev) if last else None
            u = _unit(rows, tbl, conv, bn, acts[-1], out, z, mean, invstd, train, out_p=out_p)
            _run_unit(u, dev)
            acts.append(out)
            units.append((u, z, mean, invstd))
        if train:
            torch._foreach_add_([bn.num_batches_tracked for _, bn in layers], 1)
            ctx.state = (mod, B, n, m, C1, C2, idx, weight, acts, units)
        return out_p.view(B, n, -1)

    @staticmethod
    def backward(ctx, d_out):
        mod, B, n, m, C1, C2, idx, weight, acts, units = ctx.state
        ctx.state = None
        dev = d_out.device
        layers = _layers(mod.mlp)
        g = d_out.reshape(B * n, -1).contiguous()
        grads = []
        for (conv, bn), (u, *_) in zip(reversed(layers), reversed(units)):
            gin = torch.empty(B * n, u.Cin, dtype=torch.float32, device=dev)
            grads.append(_unit_backward(u, conv, bn, g, gin, dev))
            g = gin
        g = g.view(B, n, C1 + C2)
        d_known = ext.three_interpolate_grad(g[:, :, :C2].transpose(1, 2).contiguous(), idx, weight, m) if ctx.needs_input_grad[1] else None
        d_unknow = g[:, :, C2:].transpose(1, 2) if C1 and ctx.needs_input_grad[2] else None
        return (None, d_known, d_unknow, None, None) + tuple(t for layer in reversed(grads) for t in layer)


class PointnetFPModule(nn.Module):
    """`pointnet2_modules.PointnetFPModule` on this library: three-NN inverse-distance interpolation of known_feats onto the unknown
    points, concatenated with unknow_feats, through the shared MLP."""

    def __init__(self, *, mlp, bn=True):
        super().__init__()
        if not bn:
            raise NotImplementedError("PointnetFPModule(bn=False) is not supported on this library")
        _check_widths(mlp, 0)
        self.mlp = _shared_mlp(mlp)

    def forward(self, unknown, known, unknow_feats, known_feats):
        """unknown [B, n, 3], known [B, m, 3], unknow_feats [B, C1, n] or None, known_feats [B, C2, m] -> [B, mlp[-1], n] (a view of
        point-major storage)."""
        if known is None:
            raise NotImplementedError("PointnetFPModule with known=None is not supported on this library")
        _lib.require_cuda(known_feats)
        params = _params(self.mlp)
        if not self.training:
            _eval_forward_only(params + [t for t in (known_feats, unknow_feats) if t is not None])
        dist2, idx = ext.three_nn(unknown.detach().contiguous(), known.detach().contiguous())
        dist_recip = 1.0 / (torch.sqrt(dist2) + 1e-8)                 # the original's weights
        weight = (dist_recip / torch.sum(dist_recip, dim=2, keepdim=True)).contiguous()
        out = _FPFunction.apply(self, known_feats, unknow_feats, idx, weight, *params)
        return out.transpose(1, 2)


def install():
    """pointnet2.install() (the `_ext` operators and pointnet2_utils' native import), then register this module as `pointnet2_modules`
    and `models.backbone.pointnet2.pointnet2_modules`, the names VoteNet's backbone_module.py and proposal_module.py import.  Returns it."""
    pointnet2.install()
    mod = sys.modules[__name__]
    register(mod, "pointnet2_modules")
    return register(mod, "models.backbone.pointnet2.pointnet2_modules")
