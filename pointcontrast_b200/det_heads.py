"""VoteNet's voting module and proposal head on libpcb200 (DESIGN.md 8f-18): `models/voting_module.py` (`VotingModule`) and
`models/proposal_module.py` (`ProposalModule`, `decode_scores`), each head one autograd node per forward in place of the original's
Conv1d / BatchNorm1d / ReLU layers and its slice-and-add tail.

    from pointcontrast_b200 import det_heads
    det_heads.install()     # `from voting_module import ...` / `from proposal_module import ...` (votenet.py) now resolve here

The modules take the original's constructor and call arguments and return what it returns.  Their parameters and buffers have the
original's names, order, shapes and seeded initial values, held by real nn.Conv1d / nn.BatchNorm1d modules, so original checkpoints load,
optimiser state lines up and BNMomentumScheduler reaches them.  Each forward reads `bn.momentum`, honours train() / eval() and counts
`num_batches_tracked`.  Eval mode is forward only (run it under torch.no_grad(), as VoteNet's evaluation does).

Each head is two fused units (`pcb_unit_forward`, K = 1 identity table: conv1 -> bn1 -> relu, conv2 -> bn2 -> relu), the last 1x1
convolution (`pcb_conv_forward_split`) into z [rows, Cpad], and one epilogue kernel (csrc/det_head.cu).  Conv biases ride as one more
input channel of constant 1: every layer's input planes carry 32 extra columns (1, 0, ..., 0), and the weight tiles a bias row, so z
includes the bias and the bias gradient is row Cin of the weight gradient.  Rows are point-major throughout:
  * VotingModule reads the seed features as [B S, C] rows (a view when they are point-major storage, as both backbones return them),
    writes vote_xyz [B, S V, 3] contiguous and vote_features as the channel-major view [B, C, S V] of point-major [B S V, C] storage;
  * ProposalModule reads the vote aggregation's output rows the same way; six of decode_scores' nine end_points are strided views of z
    [B, K, Xpad], as in the original they are views of `net`; center, heading_residuals and size_residuals are the epilogue's, bit for
    bit the original's torch expressions on the same z.
The backward sweeps are hand-written and deterministic: the epilogue adjoint assembles the gradient of z as bf16 hi/lo planes (and the
residual gradients of the seed features and xyz, or of aggregated_vote_xyz), then the conv weight and data gradients and the units'
backward passes.

Supported: feature widths that are multiples of 32 (the tensor-core tiling), BatchNorm momentum set, the three sampling modes.  Anything
else raises.
"""
import ctypes
import sys

import numpy as np
import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib, pointnet2, pointnet2_modules
from ._lib import PcbError, PcbStrided, check, lib, ptr, stream, workspace
from .det_eval import register
from .pointnet2_modules import _F16, _Planes, _conv_grads, _eval_forward_only, _identity, _momentum, _run_unit, _tiles, _unit, \
    _unit_backward

_ONE_F16, _ONE_BF16 = 0x3C00, 0x3F80          # 1.0 as an fp16 and a bf16 bit pattern: hi = 1, lo = 0 in either split format
DECODE = ("objectness_scores", "center", "heading_scores", "heading_residuals_normalized", "heading_residuals", "size_scores",
          "size_residuals_normalized", "size_residuals", "sem_cls_scores")


def _check_width(name, c):
    if c % 32:
        raise NotImplementedError(f"{name}={c} is not a multiple of 32 (the tensor-core tiling of the head's layers)")


def _planes(n, C, dev, dual):
    """_Planes [n, C + 32] whose last 32 columns are the bias input (1, 0, ..., 0) of the next layer."""
    p = _Planes(n, C + 32, dev, dual)
    p.t[:, :, C:] = 0
    p.t[0, :, C] = _ONE_F16
    if dual:
        p.t[2, :, C] = _ONE_BF16
    return p


def _rows(features, n, C):
    """Channel-major features [B, C, P] as point-major rows [n = B P, C]: a view when they are point-major storage."""
    X = features.detach().transpose(1, 2).reshape(n, C)
    if X.stride(1) != 1 or X.stride(0) % 4:
        X = X.contiguous()
    return X


def _strided(t):
    if t is None:
        return None
    return ctypes.byref(PcbStrided(t.data_ptr(), *(list(t.stride()) + [0] * (4 - t.dim()))))


def _head_forward(ctx, convs, bns, X, n, train, dev):
    """conv1/bn1/relu, conv2/bn2/relu as fused units over the rows X [n, C], then conv3 into z [n, Cpad].  Returns z; keeps what the
    backward pass reads on ctx."""
    st = stream()
    C = X.shape[1]
    tbl = _identity(n, dev)
    a0 = _planes(n, C, dev, train)
    h, l, bh, bl = a0.ptrs()
    check(lib.pcb_split_rows(X.data_ptr(), X.stride(0), n, C, h, l, C + 32, _lib.PLANES_A_FP16, st))
    if train:
        check(lib.pcb_split_rows(X.data_ptr(), X.stride(0), n, C, bh, bl, C + 32, 0, st))
    acts, units = [a0], []
    for conv, bn in zip(convs[:2], bns):
        cout = conv.weight.shape[0]
        z = torch.empty(n, cout, dtype=torch.float32, device=dev)
        mean = torch.empty(cout, dtype=torch.float32, device=dev)
        invstd = torch.empty_like(mean)
        out = _planes(n, cout, dev, train)
        u = _unit(n, tbl, conv, bn, acts[-1], out, z, mean, invstd, train)
        _run_unit(u, dev)
        acts.append(out)
        units.append((u, z, mean, invstd))
    tiles3 = _tiles(convs[2])
    cin, cpad = tiles3[0].shape
    z = torch.empty(n, cpad, dtype=torch.float32, device=dev)
    h, l = acts[-1].ptrs()[:2]
    wsb = lib.pcb_conv_forward_split_ws_bytes(1, n, cin, cpad)
    ws = workspace(wsb, dev)
    check(lib.pcb_conv_forward_split(h, l, cin, ptr(tbl), tbl.shape[1], None, 1, n, cin, cpad, ptr(tiles3[1]), None, ptr(z), cpad,
                                     ptr(ws), wsb, _F16, st))
    if train:
        torch._foreach_add_([bn.num_batches_tracked for bn in bns], 1)
        ctx.head = (convs, bns, n, tbl, acts, units, tiles3)
    return z


def _head_backward(ctx, dz, dev, gin, gin_mode):
    """From the gradient of z (bf16 hi/lo planes [2, n, Cpad]): conv3's weight and data gradients, then the two units' backward
    passes; conv1's data gradient goes to gin ([n, C + 32], written (gin_mode 1) or accumulated (2)).  Returns the parameter
    gradients in registration order: conv1 (weight, bias), conv2, conv3, bn1 (weight, bias), bn2."""
    convs, bns, n, tbl, acts, units, tiles3 = ctx.head
    ctx.head = None
    st = stream()
    cin, cpad = tiles3[0].shape
    C = cin - 32
    dW = torch.zeros(cin, cpad, dtype=torch.float32, device=dev)
    _, _, bh, bl = acts[-1].ptrs()
    wsb = lib.pcb_conv_wgrad_split_ws_bytes(1, n, cin, cpad)
    ws = workspace(wsb, dev)
    check(lib.pcb_conv_wgrad_split(bh, bl, cin, dz[0].data_ptr(), dz[1].data_ptr(), cpad, ptr(tbl), tbl.shape[1], 1, n, cin, cpad, ptr(dW),
                                   0, ptr(ws), wsb, _lib.CONV_ACCUMULATE, st))
    g = torch.empty(n, cin, dtype=torch.float32, device=dev)
    wsb = lib.pcb_conv_forward_split_ws_bytes(1, n, cpad, cin)
    ws = workspace(wsb, dev)
    check(lib.pcb_conv_forward_split(dz[0].data_ptr(), dz[1].data_ptr(), cpad, ptr(tbl), tbl.shape[1], None, 1, n, cpad, cin,
                                     ptr(tiles3[2]), None, ptr(g), cin, ptr(ws), wsb, 0, st))
    del dz
    grads3 = _conv_grads(convs[2], dW)
    (u1, *_), (u2, *_) = units
    g1 = torch.empty(n, u2.Cin, dtype=torch.float32, device=dev)
    w2, b2, gm2, bt2 = _unit_backward(u2, convs[1], bns[1], g[:, :C], g1, dev)
    w1, b1, gm1, bt1 = _unit_backward(u1, convs[0], bns[0], g1[:, :u1.Cout], gin, dev, gin_mode=gin_mode)
    return (w1, b1, w2, b2) + grads3 + (gm1, bt1, gm2, bt2)


def _head_params(mod):
    return [mod.conv1.weight, mod.conv1.bias, mod.conv2.weight, mod.conv2.bias, mod.conv3.weight, mod.conv3.bias, mod.bn1.weight,
            mod.bn1.bias, mod.bn2.weight, mod.bn2.bias]


def _check_momentum(mod):
    if mod.training:
        for bn in (mod.bn1, mod.bn2):
            _momentum(bn)


def _prepare(mod, inputs):
    """Checks shared by both heads' forwards, before anything touches a device; returns the head's parameters."""
    _check_momentum(mod)
    _lib.require_cuda(inputs[0])
    if any(t.dtype != torch.float32 for t in inputs):
        raise PcbError(f"{type(mod).__name__} takes fp32 inputs")
    params = _head_params(mod)
    if not mod.training:
        _eval_forward_only(params + list(inputs))
    return params


# ------------------------------------------------------------------------------------------------ voting
class _VoteFunction(Function):
    @staticmethod
    def forward(ctx, mod, seed_xyz, seed_features, *params):
        ctx.set_materialize_grads(False)
        dev = seed_xyz.device
        B, S, _ = seed_xyz.shape
        C, V = mod.in_dim, mod.vote_factor
        n = B * S
        xs = seed_xyz.detach().contiguous()
        X = _rows(seed_features, n, C)
        z = _head_forward(ctx, (mod.conv1, mod.conv2, mod.conv3), (mod.bn1, mod.bn2), X, n, mod.training, dev)
        vote_xyz = torch.empty(B, S * V, 3, dtype=torch.float32, device=dev)
        vote_features = torch.empty(n * V, C, dtype=torch.float32, device=dev)
        check(lib.pcb_vote_epilogue(ptr(xs), X.data_ptr(), X.stride(0), ptr(z), z.shape[1], B, S, V, C, ptr(vote_xyz), ptr(vote_features),
                                    stream()))
        ctx.dims = (B, S, V, C, z.shape[1])
        return vote_xyz, vote_features.view(B, S * V, C)

    @staticmethod
    def backward(ctx, d_vote_xyz, d_vote_features):
        B, S, V, C, cpad = ctx.dims
        dev = ctx.head[3].device
        n = B * S
        dz = torch.empty(2, n, cpad, dtype=torch.int16, device=dev)
        gin = torch.empty(n, C + 32, dtype=torch.float32, device=dev)    # the residual gradient, then conv1's data gradient added
        gin[:, C:] = 0
        d_xyz = torch.empty(B, S, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        check(lib.pcb_vote_epilogue_grad(_strided(d_vote_xyz), _strided(d_vote_features), B, S, V, C, dz[0].data_ptr(), dz[1].data_ptr(),
                                         cpad, cpad, gin.data_ptr(), C + 32, ptr(d_xyz), stream()))
        grads = _head_backward(ctx, dz, dev, gin, 2)
        d_feat = gin[:, :C].view(B, S, C).transpose(1, 2) if ctx.needs_input_grad[2] else None
        return (None, d_xyz, d_feat) + grads


class VotingModule(nn.Module):
    """`voting_module.VotingModule` on this library: votes from seed xyz and features (see the module docstring)."""

    def __init__(self, vote_factor, seed_feature_dim):
        super().__init__()
        _check_width("seed_feature_dim", seed_feature_dim)
        self.vote_factor = vote_factor
        self.in_dim = seed_feature_dim
        self.out_dim = self.in_dim
        self.conv1 = torch.nn.Conv1d(self.in_dim, self.in_dim, 1)
        self.conv2 = torch.nn.Conv1d(self.in_dim, self.in_dim, 1)
        self.conv3 = torch.nn.Conv1d(self.in_dim, (3 + self.out_dim) * self.vote_factor, 1)
        self.bn1 = torch.nn.BatchNorm1d(self.in_dim)
        self.bn2 = torch.nn.BatchNorm1d(self.in_dim)

    def forward(self, seed_xyz, seed_features):
        """seed_xyz fp32 [B, S, 3], seed_features fp32 [B, C, S] -> (vote_xyz [B, S V, 3] contiguous, vote_features [B, C, S V], a
        channel-major view of point-major storage)."""
        params = _prepare(self, (seed_xyz, seed_features))
        if seed_features.shape[1] != self.in_dim or seed_features.shape[2] != seed_xyz.shape[1]:
            raise PcbError(f"seed_features {tuple(seed_features.shape)} do not match seed_xyz {tuple(seed_xyz.shape)} and "
                           f"seed_feature_dim {self.in_dim}")
        vote_xyz, vote_features = _VoteFunction.apply(self, seed_xyz, seed_features, *params)
        return vote_xyz, vote_features.transpose(1, 2)


# ------------------------------------------------------------------------------------------------ decode_scores
class _Decode:
    """The column layout of decode_scores for (NH, NS, C) and mean_size, and the epilogue calls on z [B, K, >= X]."""

    def __init__(self, num_class, num_heading_bin, num_size_cluster, mean_size_arr):
        self.NH, self.NS, self.C = int(num_heading_bin), int(num_size_cluster), int(num_class)
        self.X = 5 + 2 * self.NH + 4 * self.NS + self.C
        self.ms = np.ascontiguousarray(np.asarray(mean_size_arr).astype(np.float32))
        if self.ms.shape != (self.NS, 3):
            raise PcbError(f"mean_size_arr has shape {self.ms.shape}, expected ({self.NS}, 3)")
        self.unit = float(np.float32(np.pi / self.NH))          # torch's fp32 tensor times the Python float pi / NH

    def outputs(self, z, agg):
        """The nine end_points in DECODE order: six strided views of z, center / heading_residuals / size_residuals computed."""
        B, K, ldz = z.shape
        NH, NS = self.NH, self.NS
        dev = z.device
        center = torch.empty(B, K, 3, dtype=torch.float32, device=dev)
        hr = torch.empty(B, K, NH, dtype=torch.float32, device=dev)
        sr = torch.empty(B, K, NS, 3, dtype=torch.float32, device=dev)
        check(lib.pcb_proposal_epilogue(ptr(z), ldz, ptr(agg), B, K, NH, NS, self.unit, self.ms.ctypes.data, ptr(center), ptr(hr), ptr(sr),
                                        stream()))
        s0 = 5 + 2 * NH
        c0 = s0 + 4 * NS
        return (z[:, :, 0:2], center, z[:, :, 5:5 + NH], z[:, :, 5 + NH:s0], hr, z[:, :, s0:s0 + NS],
                z[:, :, s0 + NS:c0].view(B, K, NS, 3), sr, z[:, :, c0:self.X])

    def grad(self, grads, B, K, ldz, dev, planes, d_agg):
        """The gradient of z [B K, ldz] from the nine end_points' gradients: bf16 hi/lo planes [2, B K, ldz] (planes) or fp32."""
        arr = (PcbStrided * len(DECODE))()
        for i, g in enumerate(grads):
            if g is not None:
                arr[i] = PcbStrided(g.data_ptr(), *(list(g.stride()) + [0] * (4 - g.dim())))
        if planes:
            dz = torch.empty(2, B * K, ldz, dtype=torch.int16, device=dev)
            hi, lo, f = dz[0].data_ptr(), dz[1].data_ptr(), None
        else:
            dz = torch.empty(B * K, ldz, dtype=torch.float32, device=dev)
            hi, lo, f = None, None, dz.data_ptr()
        check(lib.pcb_proposal_epilogue_grad(arr, B, K, self.NH, self.NS, self.C, self.unit, self.ms.ctypes.data, hi, lo, f, ldz, ldz,
                                             ptr(d_agg), stream()))
        return dz


class _DecodeFunction(Function):
    @staticmethod
    def forward(ctx, dec, net, agg):
        ctx.set_materialize_grads(False)
        B, X, K = net.shape
        z = torch.empty(B, K, X, dtype=torch.float32, device=net.device)
        z.copy_(net.detach().transpose(1, 2))
        ctx.dec, ctx.dims = dec, (B, K, X)
        return dec.outputs(z, agg.detach().contiguous())

    @staticmethod
    def backward(ctx, *grads):
        B, K, X = ctx.dims
        dev = next(g for g in grads if g is not None).device
        d_agg = torch.empty(B, K, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
        dz = ctx.dec.grad(grads, B, K, X, dev, False, d_agg)
        return None, dz.view(B, K, X).transpose(1, 2), d_agg


def decode_scores(net, end_points, num_class, num_heading_bin, num_size_cluster, mean_size_arr):
    """`proposal_module.decode_scores`: net [B, 2+3+NH*2+NS*4+C, K] -> the nine score and residual end_points, with
    end_points['aggregated_vote_xyz'] as the base of `center`.  Returns end_points."""
    _lib.require_cuda(net)
    dec = _Decode(num_class, num_heading_bin, num_size_cluster, mean_size_arr)
    if net.dtype != torch.float32 or net.dim() != 3 or net.shape[1] != dec.X:
        raise PcbError(f"decode_scores: net must be fp32 [B, {dec.X}, K], got {net.dtype} {tuple(net.shape)}")
    end_points.update(zip(DECODE, _DecodeFunction.apply(dec, net, end_points["aggregated_vote_xyz"])))
    return end_points


# ------------------------------------------------------------------------------------------------ proposal head
class _ProposalFunction(Function):
    @staticmethod
    def forward(ctx, mod, agg, features, *params):
        ctx.set_materialize_grads(False)
        dev = features.device
        B, C, K = features.shape
        n = B * K
        X = _rows(features, n, C)
        z = _head_forward(ctx, (mod.conv1, mod.conv2, mod.conv3), (mod.bn1, mod.bn2), X, n, mod.training, dev)
        ctx.dims = (mod.decode, B, K, z.shape[1])
        return mod.decode.outputs(z.view(B, K, -1), agg.detach().contiguous())

    @staticmethod
    def backward(ctx, *grads):
        dec, B, K, xpad = ctx.dims
        dev = ctx.head[3].device
        d_agg = torch.empty(B, K, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
        dz = dec.grad(grads, B, K, xpad, dev, True, d_agg)
        cin = ctx.head[0][0].weight.shape[1] + 32
        gin = torch.empty(B * K, cin, dtype=torch.float32, device=dev)
        pgrads = _head_backward(ctx, dz, dev, gin, 1)
        d_feat = gin[:, :cin - 32].view(B, K, cin - 32).transpose(1, 2) if ctx.needs_input_grad[2] else None
        return (None, d_agg, d_feat) + pgrads


class ProposalModule(nn.Module):
    """`proposal_module.ProposalModule` on this library: vote aggregation (this library's PointnetSAModuleVotes), then the proposal
    layers and decode_scores (see the module docstring)."""

    def __init__(self, num_class, num_heading_bin, num_size_cluster, mean_size_arr, num_proposal, sampling, seed_feat_dim=256):
        super().__init__()
        if sampling not in ("vote_fps", "seed_fps", "random"):
            raise NotImplementedError(f"sampling={sampling!r}: the original knows 'vote_fps', 'seed_fps' and 'random'")
        _check_width("seed_feat_dim", seed_feat_dim)
        self.num_class = num_class
        self.num_heading_bin = num_heading_bin
        self.num_size_cluster = num_size_cluster
        self.mean_size_arr = mean_size_arr
        self.num_proposal = num_proposal
        self.sampling = sampling
        self.seed_feat_dim = seed_feat_dim
        self.vote_aggregation = pointnet2_modules.PointnetSAModuleVotes(npoint=self.num_proposal, radius=0.3, nsample=16,
                                                                        mlp=[self.seed_feat_dim, 128, 128, 128], use_xyz=True,
                                                                        normalize_xyz=True)
        self.conv1 = torch.nn.Conv1d(128, 128, 1)
        self.conv2 = torch.nn.Conv1d(128, 128, 1)
        self.conv3 = torch.nn.Conv1d(128, 2 + 3 + num_heading_bin * 2 + num_size_cluster * 4 + self.num_class, 1)
        self.bn1 = torch.nn.BatchNorm1d(128)
        self.bn2 = torch.nn.BatchNorm1d(128)
        self.decode = _Decode(num_class, num_heading_bin, num_size_cluster, mean_size_arr)

    def forward(self, xyz, features, end_points):
        """xyz [B, N, 3] (votes), features [B, C, N] -> end_points with aggregated_vote_xyz, aggregated_vote_inds and decode_scores'
        nine entries."""
        _check_momentum(self)
        if self.sampling == "vote_fps":
            xyz, features, fps_inds = self.vote_aggregation(xyz, features)
            sample_inds = fps_inds
        elif self.sampling == "seed_fps":
            sample_inds = pointnet2.furthest_point_sample(end_points["seed_xyz"].contiguous(), self.num_proposal)
            xyz, features, _ = self.vote_aggregation(xyz, features, sample_inds)
        else:
            num_seed = end_points["seed_xyz"].shape[1]
            batch_size = end_points["seed_xyz"].shape[0]
            sample_inds = torch.randint(0, num_seed, (batch_size, self.num_proposal), dtype=torch.int).to(xyz.device)
            xyz, features, _ = self.vote_aggregation(xyz, features, sample_inds)
        end_points["aggregated_vote_xyz"] = xyz
        end_points["aggregated_vote_inds"] = sample_inds
        params = _prepare(self, (xyz, features))
        end_points.update(zip(DECODE, _ProposalFunction.apply(self, xyz, features, *params)))
        return end_points


def install():
    """pointnet2_modules.install() (the library's PointNet++ operators and modules), then register this module as `voting_module`,
    `models.voting_module`, `proposal_module` and `models.proposal_module`, the names VoteNet's votenet.py imports.  Returns it."""
    pointnet2_modules.install()
    mod = sys.modules[__name__]
    for name in ("voting_module", "models.voting_module", "proposal_module"):
        register(mod, name)
    return register(mod, "models.proposal_module")
