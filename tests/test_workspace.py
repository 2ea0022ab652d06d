"""Workspace contract of libpcb200 (include/pcb200.h, "Conventions"): every entry point that takes `ws` accepts any ws_bytes >= its
*_ws_bytes query, rejects a shorter one with PCB_ERR_ARG before it touches the device, never touches a byte at or beyond the query,
and computes the same bits whatever the size of ws.

Each case below builds one call's inputs from a seed and returns (query, call(ws_ptr, ws_bytes) -> status, outputs() -> arrays), and
names the entry points its call invokes; every entry point that takes a workspace has a case (test_every_workspace_entry_point_has_a_case).
Without a GPU the tensors live in host memory: only the argument checks run, and they return before any pointer is used."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle.det_eval_cpu import get_3d_box
from pointcontrast_b200 import _lib, det_loss, synth

L = _lib.lib
GPU = torch.cuda.is_available()
DEV = torch.device("cuda:0" if GPU else "cpu")
TAIL = 64 << 10
HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "pcb200.h")


def _st():
    return _lib.stream() if GPU else None


class _In:
    """Seeded inputs on DEV; every output starts zeroed, so whole buffers compare bit for bit."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def rand(self, *shape, scale=1.0, dtype=torch.float32):
        return (torch.rand(*shape, generator=self.g, dtype=torch.float64) * scale).to(dtype).to(DEV)

    def randint(self, lo, hi, *shape, dtype=torch.int32):
        return torch.randint(lo, hi, shape, generator=self.g).to(dtype).to(DEV)

    @staticmethod
    def zeros(*shape, dtype=torch.float32):
        return torch.zeros(*shape, dtype=dtype, device=DEV)


def _host(x):
    return np.ctypeslib.as_array(x).copy() if isinstance(x, ctypes.Array) else np.array(x.value if hasattr(x, "value") else x)


def _outputs(*xs):
    return lambda: [x.cpu().numpy() if isinstance(x, torch.Tensor) else _host(x) for x in xs]


def _split(x):
    """fp32 [n, C] -> bf16 hi / lo planes (uint16 [n, C])"""
    n, C = x.shape
    hi, lo = _In.zeros(n, C, dtype=torch.int16), _In.zeros(n, C, dtype=torch.int16)
    if GPU:
        _lib.check(L.pcb_split_rows(x.data_ptr(), C, n, C, hi.data_ptr(), lo.data_ptr(), C, 0, _st()))
    return hi, lo


def _tiles(W, K, Cin, Cout):
    fwd = _In.zeros(L.pcb_weight_tile_bytes(K, Cin, Cout, 0), dtype=torch.uint8)
    dg = _In.zeros(L.pcb_weight_tile_bytes(K, Cin, Cout, 1), dtype=torch.uint8)
    if GPU:
        _lib.check(L.pcb_weight_tile(W.data_ptr(), K, Cin, Cout, fwd.data_ptr(), dg.data_ptr(), 0, _st()))
    return fwd, dg


def _device_bytes(p, n):
    """The n device bytes at address p as a uint8 tensor (a view, not a copy)."""
    view = type("View", (), {"__cuda_array_interface__": dict(shape=(n,), typestr="|u1", data=(p, False), version=2)})
    return torch.as_tensor(view(), device=DEV)


def _calls(*names):
    """Declares the library functions a case's call invokes."""
    def mark(case):
        case.calls = names
        return case
    return mark


# ------------------------------------------------------------------------------------------------ cases (seeded, one call each)

@_calls("pcb_voxelize")
def voxelize(n):
    i = _In(1)
    xyz, oc, sel, m = i.rand(n, 3, scale=10.0), i.zeros(n, 3, dtype=torch.int32), i.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_voxelize_ws_bytes(n),
            lambda ws, b: L.pcb_voxelize(xyz.data_ptr(), n, 0.25, oc.data_ptr(), sel.data_ptr(), ctypes.byref(m), ws, b, _st()),
            _outputs(oc, sel, m))


@_calls("pcb_voxelize_labels")
def voxelize_labels(n):
    i = _In(2)
    c, lab = i.randint(-60, 60, n, 3), i.randint(0, 4, n)
    oc, sel, ol, m = i.zeros(n, 3, dtype=torch.int32), i.zeros(n, dtype=torch.int32), i.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_voxelize_labels_ws_bytes(n),
            lambda ws, b: L.pcb_voxelize_labels(c.data_ptr(), lab.data_ptr(), n, 255, oc.data_ptr(), sel.data_ptr(), ol.data_ptr(),
                                                ctypes.byref(m), ws, b, _st()),
            _outputs(oc, sel, ol, m))


@_calls("pcb_voxelize_scenes")
def voxelize_scenes(B, N):
    i = _In(3)
    xyz, oc, inds, off = i.rand(B, N, 3, scale=5.0), i.zeros(B * N, 4, dtype=torch.int32), i.zeros(B * N, dtype=torch.int32), i.zeros(B + 1, dtype=torch.int64)
    oh = (ctypes.c_int64 * (B + 1))()
    return (L.pcb_voxelize_scenes_ws_bytes(B, N),
            lambda ws, b: L.pcb_voxelize_scenes(xyz.data_ptr(), B, N, 0.1, oc.data_ptr(), inds.data_ptr(), off.data_ptr(), oh, ws, b, _st()),
            _outputs(oc, inds, off, oh))


@_calls("pcb_radius_pairs")
def radius_pairs(ns, nd):
    i = _In(4)
    src, dst = i.rand(ns, 3, scale=4.0), i.rand(nd, 3, scale=4.0)
    cap = 64 * ns
    pairs, npairs = i.zeros(cap, 2, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_radius_pairs_ws_bytes(ns, nd),
            lambda ws, b: L.pcb_radius_pairs(src.data_ptr(), ns, dst.data_ptr(), nd, 0.1, pairs.data_ptr(), cap, ctypes.byref(npairs), ws, b,
                                             _st()),
            _outputs(pairs, npairs))


@_calls("pcb_coords_stride")
def coords_stride(n):
    g = np.random.default_rng(5)
    b, xyz = g.integers(0, 2, n).astype(np.uint64), (g.integers(-300, 300, (n, 3)) + 32768).astype(np.uint64)
    keys = torch.from_numpy(((b << 48) | (xyz[:, 0] << 32) | (xyz[:, 1] << 16) | xyz[:, 2]).view(np.int64)).to(DEV)
    ok, parent, nout = _In.zeros(n, dtype=torch.int64), _In.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_coords_stride_ws_bytes(n),
            lambda ws, bb: L.pcb_coords_stride(keys.data_ptr(), n, 4, ok.data_ptr(), parent.data_ptr(), ctypes.byref(nout), ws, bb, _st()),
            _outputs(ok, parent, nout))


@_calls("pcb_gather_points_grad")
def gather_points_grad(B, C, N, Lr):
    i = _In(6)
    g, idx, out = i.rand(B, C, Lr), i.randint(0, N, B, Lr), i.zeros(B, C, N)
    return (L.pcb_points_grad_ws_bytes(B, N, Lr),
            lambda ws, b: L.pcb_gather_points_grad(g.data_ptr(), idx.data_ptr(), B, C, N, Lr, out.data_ptr(), ws, b, _st()),
            _outputs(out))


@_calls("pcb_three_interpolate_grad")
def three_interpolate_grad(B, C, n, m):
    i = _In(7)
    g, idx, w, out = i.rand(B, C, n), i.randint(0, m, B, n, 3), i.rand(B, n, 3), i.zeros(B, C, m)
    return (L.pcb_points_grad_ws_bytes(B, m, 3 * n),
            lambda ws, b: L.pcb_three_interpolate_grad(g.data_ptr(), idx.data_ptr(), w.data_ptr(), B, C, n, m, out.data_ptr(), ws, b, _st()),
            _outputs(out))


@_calls("pcb_gather_rows_grad")
def gather_rows_grad(Lr, C, M):
    i = _In(8)
    g, idx, out = i.rand(Lr, C), i.randint(0, M, Lr), i.zeros(M, C)
    return (L.pcb_points_grad_ws_bytes(1, M, Lr),
            lambda ws, b: L.pcb_gather_rows_grad(g.data_ptr(), idx.data_ptr(), Lr, C, M, out.data_ptr(), ws, b, _st()),
            _outputs(out))


@_calls("pcb_point_bounds")
def point_bounds(n):
    xyz = _In(9).rand(n, 3, scale=7.0)
    lo, hi = (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    return (L.pcb_point_bounds_ws_bytes(), lambda ws, b: L.pcb_point_bounds(xyz.data_ptr(), n, lo, hi, ws, b, _st()), _outputs(lo, hi))


@_calls("pcb_elastic_distort")
def elastic_distort(n, gx, gy, gz):
    i = _In(10)
    xyz, noise = i.rand(n, 3, scale=10.0), i.rand(gx, gy, gz, 3)
    axes = torch.from_numpy(np.concatenate([np.linspace(-1.0, 11.0, k) for k in (gx, gy, gz)])).to(DEV)
    return (L.pcb_elastic_distort_ws_bytes(gx, gy, gz),
            lambda ws, b: L.pcb_elastic_distort(xyz.data_ptr(), n, noise.data_ptr(), gx, gy, gz, axes.data_ptr(), 0.5, ws, b, _st()),
            _outputs(xyz, noise))


@_calls("pcb_affine_floor")
def affine_floor(n):
    xyz, out = _In(11).rand(n, 3, scale=4.0), _In.zeros(n, 3, dtype=torch.int32)
    T = np.ascontiguousarray([[50.0, 1.0, 0, 3], [0, 45.0, 2.0, -1], [1.0, 0, 55.0, 0.5], [0, 0, 0, 1]], np.float64).reshape(16)
    mn = (ctypes.c_int32 * 3)()
    return (L.pcb_affine_floor_ws_bytes(),
            lambda ws, b: L.pcb_affine_floor(xyz.data_ptr(), n, T.ctypes.data, out.data_ptr(), mn, ws, b, _st()),
            _outputs(out, mn))


@_calls("pcb_semseg_input_transform")
def input_transform(n):
    i = _In(12)
    coords, feats, noise = i.randint(0, 100, n, 3), i.rand(n, 3, scale=255.0), i.rand(n, 3, dtype=torch.float64)
    tr = (ctypes.c_double * 3)(1.0, -2.0, 3.0)
    return (L.pcb_semseg_input_transform_ws_bytes(),
            lambda ws, b: L.pcb_semseg_input_transform(coords.data_ptr(), feats.data_ptr(), n, 5, 1, 0.3, tr, noise.data_ptr(), 12.75, 1, ws, b,
                                                       _st()),
            _outputs(coords, feats))


@_calls("pcb_bn_stats_seg")
def bn_stats(n, n0, C):
    i = _In(13)
    X, mean, invstd, rm, rv = i.rand(n, C, scale=3.0), i.zeros(2 * C), i.zeros(2 * C), i.zeros(C), i.rand(C)
    return (L.pcb_bn_ws_bytes(n, C),
            lambda ws, b: L.pcb_bn_stats_seg(X.data_ptr(), C, n, n0, C, 1e-5, 0.1, mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(),
                                             rv.data_ptr(), ws, b, _st()),
            _outputs(mean, invstd, rm, rv))


@_calls("pcb_bn_backward_seg")
def bn_backward(n, n0, C):
    i = _In(14)
    dY, X, relu = i.rand(n, C), i.rand(n, C), (i.rand(n, C, scale=2.0) - 0.5).to(torch.bfloat16)      # relu: a bf16 hi plane
    mean, invstd, gamma = i.rand(2 * C), i.rand(2 * C) + 0.5, i.rand(C)
    dX, dgamma, dbeta = i.zeros(n, C), i.zeros(C), i.zeros(C)
    return (L.pcb_bn_ws_bytes(n, C),
            lambda ws, b: L.pcb_bn_backward_seg(dY.data_ptr(), C, X.data_ptr(), C, relu.data_ptr(), C, n, n0, C, mean.data_ptr(), invstd.data_ptr(),
                                                gamma.data_ptr(), dX.data_ptr(), C, dgamma.data_ptr(), dbeta.data_ptr(), 0, None, 0, 0, None, None,
                                                0, ws, b, _st()),
            _outputs(dX, dgamma, dbeta))


@_calls("pcb_nce_forward_backward")
def nce(n, D):
    i = _In(15)
    q, k = torch.nn.functional.normalize(i.rand(n, D) - 0.5, dim=1), torch.nn.functional.normalize(i.rand(n, D) - 0.5, dim=1)
    loss, dq, dk = i.zeros(1), i.zeros(n, D), i.zeros(n, D)
    return (L.pcb_nce_ws_bytes(n),
            lambda ws, b: L.pcb_nce_forward_backward(q.data_ptr(), k.data_ptr(), n, D, 1 / 0.07, loss.data_ptr(), dq.data_ptr(), dk.data_ptr(), ws,
                                                     b, _st()),
            _outputs(loss, dq, dk))


@_calls("pcb_ce_forward_backward")
def ce(n, C):
    i = _In(16)
    x, t = i.rand(n, C, scale=4.0), i.randint(0, C + 3, n, dtype=torch.int64)      # targets >= C: ignored
    loss, dx = i.zeros(1), i.zeros(n, C)
    return (L.pcb_ce_ws_bytes(n),
            lambda ws, b: L.pcb_ce_forward_backward(x.data_ptr(), t.data_ptr(), n, C, C, 1.0, loss.data_ptr(), dx.data_ptr(), ws, b, _st()),
            _outputs(loss, dx))


@_calls("pcb_conv_wgrad")
def conv_wgrad(K, n_out, Ca, Cb):
    i = _In(17)
    n_in = n_out + 17
    A, Bm, tbl, dW = i.rand(n_in, Ca), i.rand(n_out, Cb), i.randint(-1, n_in, K, n_out), i.zeros(K, Ca, Cb)
    return (L.pcb_conv_wgrad_ws_bytes(K, n_out, Ca, Cb),
            lambda ws, b: L.pcb_conv_wgrad(A.data_ptr(), Ca, Bm.data_ptr(), Cb, tbl.data_ptr(), n_out, K, n_out, Ca, Cb, dW.data_ptr(), 0, ws, b,
                                           0, _st()),
            _outputs(dW))


@_calls("pcb_conv_forward_split")
def conv_forward_split(K, n_out, Cin, Cout):
    i = _In(18)
    n_in = n_out + 29
    xh, xl = _split(i.rand(n_in, Cin, scale=2.0) - 1.0)
    fwd, _ = _tiles(i.rand(K, Cin, Cout) - 0.5, K, Cin, Cout)
    tbl, Y = i.randint(-1, n_in, K, n_out), i.zeros(n_out, Cout)
    return (L.pcb_conv_forward_split_ws_bytes(K, n_out, Cin, Cout),
            lambda ws, b: L.pcb_conv_forward_split(xh.data_ptr(), xl.data_ptr(), Cin, tbl.data_ptr(), n_out, None, K, n_out, Cin, Cout,
                                                   fwd.data_ptr(), None, Y.data_ptr(), Cout, ws, b, 0, _st()),
            _outputs(Y))


@_calls("pcb_conv_wgrad_split")
def conv_wgrad_split(K, n_out, Ca, Cb):
    i = _In(19)
    n_in = n_out + 13
    ah, al = _split(i.rand(n_in, Ca) - 0.5)
    bh, bl = _split(i.rand(n_out, Cb) - 0.5)
    tbl, dW = i.randint(-1, n_in, K, n_out), i.zeros(K, Ca, Cb)
    return (L.pcb_conv_wgrad_split_ws_bytes(K, n_out, Ca, Cb),
            lambda ws, b: L.pcb_conv_wgrad_split(ah.data_ptr(), al.data_ptr(), Ca, bh.data_ptr(), bl.data_ptr(), Cb, tbl.data_ptr(), n_out, K,
                                                 n_out, Ca, Cb, dW.data_ptr(), 0, ws, b, 0, _st()),
            _outputs(dW))


@_calls("pcb_unit_forward", "pcb_unit_backward")
def unit(n, n0, Cin, Cout, backward):
    """pcb_unit_forward (on a small level its split convolution also produces the BatchNorm statistics) and pcb_unit_backward"""
    i, K = _In(20), 27
    x = i.rand(n, Cin, scale=2.0) - 1.0
    xh, xl = _split(x)
    W = i.rand(K, Cin, Cout) - 0.5
    fwd, dg = _tiles(W, K, Cin, Cout)
    tbl = i.randint(-1, n, K, n)
    keep = [x, xh, xl, W, fwd, dg, tbl]
    u = _lib.PcbUnit()
    u.n_in = u.n_out = n
    u.n0, u.K, u.Cin, u.Cout, u.relu = n0, K, Cin, Cout, 1
    u.fwd_tbl = u.dg_tbl = u.wg_tbl = tbl.data_ptr()
    u.fwd_stride = u.dg_stride = u.wg_stride = n
    u.wg_gather_x = 1
    u.W, u.wt_fwd, u.wt_dg = W.data_ptr(), fwd.data_ptr(), dg.data_ptr()
    u.x_hi, u.x_lo, u.x_lds = xh.data_ptr(), xl.data_ptr(), Cin
    outs = dict(gamma=i.rand(Cout) + 0.5, beta=i.rand(Cout), running_mean=i.zeros(Cout), running_var=i.rand(Cout), mean=i.zeros(2 * Cout),
                invstd=i.zeros(2 * Cout), z_p=i.zeros(n, Cout), out_hi=i.zeros(n, Cout, dtype=torch.int16),
                out_lo=i.zeros(n, Cout, dtype=torch.int16), dW=i.zeros(K, Cin, Cout), dgamma=i.zeros(Cout), dbeta=i.zeros(Cout),
                dz_hi=i.zeros(n, Cout, dtype=torch.int16), dz_lo=i.zeros(n, Cout, dtype=torch.int16), gin_p=i.zeros(n, Cin))
    for k, t in outs.items():
        setattr(u, k, t.data_ptr())
    g = i.rand(n, Cout) - 0.5
    keep.append(g)
    u.eps, u.momentum = 1e-5, 0.1
    u.z_ld = u.out_lds = u.dz_ld = u.g_ld = Cout
    u.gin_ld, u.gin_mode = Cin, 1
    u.g_p = g.data_ptr()

    def call(ws, b, keep=keep):                          # keep: the inputs the struct points to stay alive with the call
        u.ws, u.ws_bytes = ws, b
        rc = L.pcb_unit_forward(ctypes.byref(u), _st())
        if rc == 0 and backward:
            rc = L.pcb_unit_backward(ctypes.byref(u), _st())
        return rc
    return L.pcb_unit_ws_bytes(K, n, n, Cin, Cout), call, _outputs(*outs.values())


def _sparse_table(i, K, n_out, n_in):
    """a neighbour table with about half of its entries -1, so that rows differ in their neighbour masks"""
    return torch.where(i.rand(K, n_out) < 0.5, -1, i.randint(0, n_in, K, n_out))


@_calls("pcb_conv_tile_order")
def conv_tile_order(K, n, window, stride):
    """the order of the first n rows of a table `stride` rows wide"""
    i = _In(23)
    tbl, perm = _sparse_table(i, K, stride, stride), i.zeros(n, dtype=torch.int32)
    return (L.pcb_conv_tile_order_ws_bytes(n),
            lambda ws, b: L.pcb_conv_tile_order(tbl.data_ptr(), stride, K, n, window, perm.data_ptr(), ws, b, _st()),
            _outputs(perm))


@_calls("pcb_conv_forward_split_ordered")
def conv_forward_split_ordered(K, n_out, Cin, Cout):
    """in the tile order the executor uses; a level small enough to split over offsets runs in the identity order"""
    i = _In(24)
    n_in = n_out + 29
    xh, xl = _split(i.rand(n_in, Cin, scale=2.0) - 1.0)
    fwd, _ = _tiles(i.rand(K, Cin, Cout) - 0.5, K, Cin, Cout)
    tbl, perm, Y = _sparse_table(i, K, n_out, n_in), i.zeros(n_out, dtype=torch.int32), i.zeros(n_out, Cout)
    if GPU:
        tws = i.zeros(L.pcb_conv_tile_order_ws_bytes(n_out), dtype=torch.uint8)
        _lib.check(L.pcb_conv_tile_order(tbl.data_ptr(), n_out, K, n_out, 16384, perm.data_ptr(), tws.data_ptr(), tws.numel(), _st()))
    return (L.pcb_conv_forward_split_ws_bytes(K, n_out, Cin, Cout),
            lambda ws, b: L.pcb_conv_forward_split_ordered(xh.data_ptr(), xl.data_ptr(), Cin, tbl.data_ptr(), n_out, None, K, perm.data_ptr(),
                                                           n_out, Cin, Cout, fwd.data_ptr(), None, Y.data_ptr(), Cout, ws, b, 0, _st()),
            _outputs(Y))


@_calls("pcb_seg_metrics")
def seg_metrics(n, C):
    i = _In(21)
    x, t = i.rand(n, C, scale=4.0), i.randint(0, C + 3, n, dtype=torch.int64)
    pred, prob = _In.zeros(n, dtype=torch.int32), _In.zeros(n, C)
    hist, stats = _In.zeros(C * C, dtype=torch.int64), _In.zeros(3, dtype=torch.float64)
    return (L.pcb_seg_metrics_ws_bytes(n),
            lambda ws, b: L.pcb_seg_metrics(x.data_ptr(), t.data_ptr(), n, C, C, pred.data_ptr(), prob.data_ptr(), hist.data_ptr(),
                                            stats.data_ptr(), ws, b, _st()),
            _outputs(pred, prob, hist, stats))


@_calls("pcb_average_precision")
def average_precision(n, C):
    i = _In(22)
    s, t = i.rand(n, C), i.randint(0, C, n, dtype=torch.int64)
    ap_sum, ap_cnt = _In.zeros(C, dtype=torch.float64), _In.zeros(C, dtype=torch.int64)
    return (L.pcb_average_precision_ws_bytes(n, C),
            lambda ws, b: L.pcb_average_precision(s.data_ptr(), t.data_ptr(), n, C, ap_sum.data_ptr(), ap_cnt.data_ptr(), ws, b, _st()),
            _outputs(ap_sum, ap_cnt))


@_calls("pcb_det_ap")
def det_ap(P, D, G, C):
    """D detections of P proposals against G boxes over 4 scans, with tied scores, at three IoU thresholds"""
    g = np.random.default_rng(3)
    boxes = lambda n: torch.from_numpy(np.array([get_3d_box(g.uniform(0.3, 1.5, 3), g.uniform(-3, 3), g.uniform(-2, 2, 3))
                                                 for _ in range(n)])).to(DEV)
    prop, gtc = boxes(P), boxes(G)
    t = lambda a, dt: torch.from_numpy(np.asarray(a, dt)).to(DEV)
    row, cls = t(g.integers(0, P, D), np.int32), t(g.integers(-1, C, D), np.int32)
    score, scan = t(np.round(g.random(D) * 16) / 16, np.float32), t(np.sort(g.integers(0, 4, D)), np.int32)
    gscan, gcls = t(g.integers(0, 4, G), np.int32), t(g.integers(-1, C, G), np.int32)
    thr, out = (ctypes.c_double * 3)(0.1, 0.25, 0.5), _In.zeros(3, C, 4, dtype=torch.float64)
    return (L.pcb_det_ap_ws_bytes(D, G, C, 3),
            lambda ws, b: L.pcb_det_ap(prop.data_ptr(), P, row.data_ptr(), cls.data_ptr(), score.data_ptr(), scan.data_ptr(), D,
                                       gtc.data_ptr(), gscan.data_ptr(), gcls.data_ptr(), G, C, thr, 3, out.data_ptr(), ws, b, _st()),
            _outputs(out))


def _det_loss_args(B, N, S, K, K2):
    """pcb_det_loss_args over a synthetic ScanNet-shaped VoteNet batch, filled as det_loss.py fills it; (args, what it points to)"""
    NH, NS, C = 1, 18, 18
    ms = np.random.default_rng(B).uniform(0.3, 2.0, (NS, 3))
    ep = synth.synth_votenet_loss_batch(25, B, N, S, K, 1, NH, ms, C, max_obj=K2)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in ep.items()}
    mean = np.ascontiguousarray(ms, np.float32)
    a = _lib.PcbDetLossArgs(B, S, 1, N, K, K2, NH, NS, C, 0, float(np.float32(1.0) / np.float32(np.pi / NH)), mean.ctypes.data)
    for f, typ in _lib.PcbDetLossArgs._fields_:
        if f in t:
            setattr(a, f, t[f].data_ptr() if typ is ctypes.c_void_p else det_loss._strided(t[f]))
    a.center_label_ld = 3
    return a, (t, mean)


@_calls("pcb_det_loss_forward")
def det_loss_forward(B, N, S, K, K2):
    a, keep = _det_loss_args(B, N, S, K, K2)
    out, label, mask, assign = _In.zeros(13), _In.zeros(B, K, dtype=torch.int64), _In.zeros(B, K), _In.zeros(B, K, dtype=torch.int64)
    state = _In.zeros(L.pcb_det_loss_state_bytes(B, S, K, K2), dtype=torch.uint8)

    def call(ws, b, keep=keep):
        return L.pcb_det_loss_forward(ctypes.byref(a), out.data_ptr(), label.data_ptr(), mask.data_ptr(), assign.data_ptr(), state.data_ptr(),
                                      state.numel(), ws, b, _st())
    return L.pcb_det_loss_ws_bytes(B, S, K, K2), call, _outputs(out, label, mask, assign, state)


@_calls("pcb_det_loss_backward")
def det_loss_backward(B, N, S, K, K2):
    """The backward's buffer is the forward's state (pcb_det_loss_state_bytes): the forward runs here, and each call copies its state
    into the bytes under test, up to their size, before the backward reads it from there."""
    a, keep = _det_loss_args(B, N, S, K, K2)
    label, mask, assign = _In.zeros(B, K, dtype=torch.int64), _In.zeros(B, K), _In.zeros(B, K, dtype=torch.int64)
    q = L.pcb_det_loss_state_bytes(B, S, K, K2)
    state, grad = _In.zeros(q, dtype=torch.uint8), _In(26).rand(13) - 0.5
    if GPU:
        ws = _In.zeros(L.pcb_det_loss_ws_bytes(B, S, K, K2), dtype=torch.uint8)
        _lib.check(L.pcb_det_loss_forward(ctypes.byref(a), _In.zeros(13).data_ptr(), label.data_ptr(), mask.data_ptr(), assign.data_ptr(),
                                          state.data_ptr(), q, ws.data_ptr(), ws.numel(), _st()))
    grads = [_In.zeros(*keep[0][k].shape) for k in det_loss.GRAD_INPUTS]

    def call(ws, b, keep=keep):
        if GPU:
            _device_bytes(ws, min(b, q)).copy_(state[:min(b, q)])
        return L.pcb_det_loss_backward(ctypes.byref(a), grad.data_ptr(), label.data_ptr(), mask.data_ptr(), assign.data_ptr(), ws, b,
                                       *[g.data_ptr() for g in grads], _st())
    return q, call, _outputs(*grads)


def _offsets(ns):
    """offsets of scenes of sizes ns: (host int64 [B + 1], the same on DEV)"""
    off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)
    return off, torch.from_numpy(off).to(DEV)


@_calls("pcb_det_choices")
def det_choices(ns, k):
    off, d_off = _offsets(ns)
    out = _In.zeros(len(ns), k, dtype=torch.int64)
    return (L.pcb_det_choices_ws_bytes(int(off[-1])),
            lambda ws, b: L.pcb_det_choices(off.ctypes.data, d_off.data_ptr(), len(ns), k, 7, 4, out.data_ptr(), ws, b, _st()),
            _outputs(out))


@_calls("pcb_det_points")
def det_points(ns, k):
    """augmented ScanNet scenes with a floor-height column, as det_data.py assembles them (the box fields only pcb_det_boxes reads are
    left unset)"""
    i = _In(27)
    off, d_off = _offsets(ns)
    B, M = len(ns), int(off[-1])
    t = dict(params=i.rand(B, _lib.DET_NPARAM, dtype=torch.float64), floor=i.rand(B, dtype=torch.float64),
             choices=torch.cat([i.randint(0, n, 1, k, dtype=torch.int64) for n in ns]), vert=i.rand(M, 6, scale=4.0),
             sem=i.randint(0, 41, M), ins=i.randint(0, 30, M), nyu40ids=torch.arange(3, 21, dtype=torch.int64, device=DEV),
             point_clouds=i.zeros(B, k, 4), pcl_color=i.zeros(B, k, 3), vote_label=i.zeros(B, k, 9),
             vote_label_mask=i.zeros(B, k, dtype=torch.int64))
    a = _lib.PcbDetBatch()
    a.B, a.M, a.num_points, a.dataset, a.flags = B, M, k, _lib.DET_SCANNET, _lib.DET_HEIGHT | _lib.DET_AUGMENT
    a.offsets_host, a.offsets, a.n_ids, a.num_heading_bin = off.ctypes.data, d_off.data_ptr(), 18, 1
    for f, x in t.items():
        setattr(a, f, x.data_ptr())

    def call(ws, b, keep=(off, t)):
        return L.pcb_det_points(ctypes.byref(a), ws, b, _st())
    return L.pcb_det_points_ws_bytes(B, k), call, _outputs(*[t[f] for f in ("point_clouds", "pcl_color", "vote_label", "vote_label_mask")])


@_calls("pcb_furthest_point_sampling")
def furthest_point_sampling(B, N, npoint):
    i = _In(28)
    xyz, idx = i.rand(B, N, 3, scale=5.0), i.zeros(B, npoint, dtype=torch.int32)
    return (L.pcb_furthest_point_sampling_ws_bytes(B, N),
            lambda ws, b: L.pcb_furthest_point_sampling(xyz.data_ptr(), B, N, npoint, idx.data_ptr(), ws, b, _st()),
            _outputs(idx))


@_calls("pcb_furthest_point_sampling_ragged")
def furthest_point_sampling_ragged(ns, npoint):
    i = _In(29)
    off, d_off = _offsets(ns)
    B, M = len(ns), int(off[-1])
    xyz, idx = i.rand(M, 3, scale=5.0), i.zeros(B, npoint, dtype=torch.int32)
    return (L.pcb_furthest_point_sampling_ragged_ws_bytes(B, M, max(ns)),
            lambda ws, b: L.pcb_furthest_point_sampling_ragged(xyz.data_ptr(), d_off.data_ptr(), B, M, max(ns), npoint, idx.data_ptr(), ws, b,
                                                               _st()),
            _outputs(idx))


def _scan(frames, points_per_frame):
    """a synthetic scan's frames as one ragged batch: xyz fp64 [n, 3] and offsets int64 [F + 1] on DEV"""
    f = synth.synth_scan_frames(3, frames, points_per_frame=points_per_frame)
    return torch.from_numpy(np.concatenate(f)).to(DEV), _offsets([len(x) for x in f])[1]


@_calls("pcb_voxel_down_sample")
def voxel_down_sample(F, per_frame):
    xyz, off = _scan(F, per_frame)
    n = xyz.shape[0]
    out, doff, host = _In.zeros(n, 3, dtype=torch.float64), _In.zeros(F + 1, dtype=torch.int64), (ctypes.c_int64 * (F + 1))()
    return (L.pcb_voxel_down_sample_ws_bytes(n, F),
            lambda ws, b: L.pcb_voxel_down_sample(xyz.data_ptr(), n, off.data_ptr(), F, 0.05, out.data_ptr(), doff.data_ptr(), host, ws, b,
                                                  _st()),
            _outputs(out, doff, host))


@_calls("pcb_frame_overlap")
def frame_overlap(F, per_frame):
    xyz, off = _scan(F, per_frame)
    n = xyz.shape[0]
    counts, status = _In.zeros(F, F, dtype=torch.int64), _In.zeros(1, dtype=torch.int32)
    return (L.pcb_frame_overlap_ws_bytes(n, F),
            lambda ws, b: L.pcb_frame_overlap(xyz.data_ptr(), n, off.data_ptr(), F, 0.075, counts.data_ptr(), status.data_ptr(), ws, b, _st()),
            _outputs(counts, status))


@_calls("pcb_depth_to_points")
def depth_to_points(F, H, W):
    g = np.random.default_rng(30)
    depth = np.where(g.random((F, H, W)) < 0.3, 0, g.integers(1, 65536, (F, H, W))).astype(np.uint16)
    poses = np.tile(np.eye(4), (F, 1, 1))
    poses[:, :3] += g.normal(0, 1, (F, 3, 4))
    depth, poses = torch.from_numpy(depth.view(np.int16)).to(DEV), torch.from_numpy(poses).to(DEV)
    out, off = _In.zeros(F * H * W, 3, dtype=torch.float64), _In.zeros(F + 1, dtype=torch.int64)
    host, nan = (ctypes.c_int64 * (F + 1))(), (ctypes.c_int32 * F)()
    return (L.pcb_depth_to_points_ws_bytes(F, H, W),
            lambda ws, b: L.pcb_depth_to_points(depth.data_ptr(), F, H, W, 50.3, 51.7, W / 2 + 0.37, H / 2 - 0.21, 0.01, -0.02,
                                                poses.data_ptr(), out.data_ptr(), off.data_ptr(), host, nan, ws, b, _st()),
            _outputs(out, off, host, nan))


@_calls("pcb_nearest")
def nearest(m, n):
    i = _In(31)
    ref, query = i.rand(m, 3, dtype=torch.float64), i.rand(n, 3, scale=1.2, dtype=torch.float64) - 0.1
    idx, status = i.zeros(n, dtype=torch.int32), i.zeros(1, dtype=torch.int32)
    return (L.pcb_nearest_ws_bytes(m, n),
            lambda ws, b: L.pcb_nearest(ref.data_ptr(), m, query.data_ptr(), n, 0.03, idx.data_ptr(), status.data_ptr(), ws, b, _st()),
            _outputs(idx, status))


@_calls("pcb_text_lines")
def text_lines(nfiles, lines):
    """S3DIS annotation files: rows of six numbers ending in "\\n", "\\r\\n" or a lone "\\r", the last line of each file unterminated"""
    g = np.random.default_rng(32)
    files = []
    for _ in range(nfiles):
        rows = [" ".join(f"{v:.3f}" for v in r) for r in g.random((lines, 6)) * 100]
        ends = g.choice(["\n", "\r\n", "\r"], lines)
        files.append("".join(r + e for r, e in zip(rows, ends))[:-1].encode())
    off = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    n = int(off[-1])
    text = _In.zeros(-(-n // 16) * 16, dtype=torch.uint8)
    text[:n] = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy())
    d_off, chunk_off, flags = torch.from_numpy(off).to(DEV), _In.zeros(-(-n // 16) + 1, dtype=torch.int64), _In.zeros(nfiles, dtype=torch.int32)
    n_lines = ctypes.c_int64()
    return (L.pcb_text_lines_ws_bytes(n),
            lambda ws, b: L.pcb_text_lines(text.data_ptr(), n, d_off.data_ptr(), nfiles, chunk_off.data_ptr(), flags.data_ptr(),
                                           ctypes.byref(n_lines), ws, b, _st()),
            _outputs(chunk_off, flags, n_lines))


@_calls("pcb_scannet_annotate")
def scannet_annotate(V, n_seg, n_obj):
    """a mesh of V vertices in n_seg segments, a label write per segment, and n_obj objects that own the segments in turn"""
    i = _In(33)
    vin, seg = i.rand(V, 6, scale=3.0), i.randint(0, n_seg, V, dtype=torch.int64)
    align = (torch.eye(4, dtype=torch.float64) + 0.1 * i.rand(4, 4, dtype=torch.float64).cpu()).reshape(16).to(DEV)
    segs = torch.arange(n_seg, dtype=torch.int64, device=DEV)
    lab_val, ins_obj = i.randint(1, 41, n_seg), (segs % n_obj).to(torch.int32)
    obj_id = torch.arange(1, n_obj + 1, dtype=torch.int32, device=DEV)
    first_seg, obj_row = segs[:n_obj].clone(), obj_id - 1
    vout, sem, ins = i.zeros(V, 6), i.zeros(V, dtype=torch.int32), i.zeros(V, dtype=torch.int32)
    bbox, status = i.zeros(n_obj, 7, dtype=torch.float64), i.zeros(2, dtype=torch.int32)
    return (L.pcb_scannet_annotate_ws_bytes(V, n_obj, n_obj),
            lambda ws, b: L.pcb_scannet_annotate(vin.data_ptr(), align.data_ptr(), V, seg.data_ptr(), segs.data_ptr(), lab_val.data_ptr(),
                                                 n_seg, segs.data_ptr(), ins_obj.data_ptr(), n_seg, obj_id.data_ptr(), first_seg.data_ptr(),
                                                 obj_row.data_ptr(), n_obj, n_obj, vout.data_ptr(), sem.data_ptr(), ins.data_ptr(),
                                                 bbox.data_ptr(), status.data_ptr(), ws, b, _st()),
            _outputs(vout, sem, ins, bbox, status))


# Two shapes per entry point; for the sorting ones (CUB temporary storage) one below and one past the single-tile sort.
CASES = [
    (voxelize, (300,)), (voxelize, (150_000,)),
    (voxelize_labels, (300,)), (voxelize_labels, (150_000,)),
    (voxelize_scenes, (2, 150)), (voxelize_scenes, (3, 60_000)),
    (radius_pairs, (300, 280)), (radius_pairs, (100_000, 120_000)),
    (coords_stride, (300,)), (coords_stride, (150_000,)),
    (gather_points_grad, (2, 8, 100, 150)), (gather_points_grad, (2, 16, 4000, 100_000)),
    (three_interpolate_grad, (2, 8, 50, 40)), (three_interpolate_grad, (2, 8, 40_000, 5000)),
    (gather_rows_grad, (300, 8, 100)), (gather_rows_grad, (150_000, 8, 20_000)),
    (point_bounds, (1000,)), (point_bounds, (500_000,)),
    (elastic_distort, (1000, 4, 5, 6)), (elastic_distort, (100_000, 20, 22, 24)),
    (affine_floor, (1000,)), (affine_floor, (300_000,)),
    (input_transform, (1000,)), (input_transform, (300_000,)),
    (bn_stats, (200, 120, 32)), (bn_stats, (100_000, 40_000, 96)),
    (bn_backward, (200, 120, 32)), (bn_backward, (100_000, 40_000, 96)),
    (nce, (300, 64)), (nce, (4000, 64)), (nce, (300, 16)), (nce, (2000, 16)),
    (ce, (300, 20)), (ce, (100_000, 20)),
    (conv_wgrad, (27, 500, 3, 32)), (conv_wgrad, (27, 50_000, 3, 32)), (conv_wgrad, (27, 300, 5, 7)), (conv_wgrad, (27, 20_000, 5, 7)),
    (conv_forward_split, (27, 200, 32, 64)), (conv_forward_split, (27, 600, 64, 32)), (conv_forward_split, (27, 20_000, 64, 64)),
    (conv_wgrad_split, (27, 300, 32, 32)), (conv_wgrad_split, (27, 50_000, 64, 32)),
    (unit, (200, 120, 32, 32, False)), (unit, (200, 120, 32, 32, True)), (unit, (30_000, 12_000, 32, 64, True)),
    (conv_tile_order, (27, 300, 128, 300)), (conv_tile_order, (27, 200_000, 128, 200_077)), (conv_tile_order, (27, 200_000, 1024, 200_000)),
    (conv_tile_order, (8, 200_000, 16384, 200_000)), (conv_tile_order, (27, 200_000, 200_064, 200_000)),
    (conv_forward_split_ordered, (27, 200, 32, 64)), (conv_forward_split_ordered, (27, 20_000, 64, 64)),
    (seg_metrics, (300, 20)), (seg_metrics, (100_000, 20)),
    (average_precision, (300, 20)), (average_precision, (100_000, 20)),
    (det_ap, (300, 900, 120, 7)), (det_ap, (2000, 20_000, 1000, 18)),
    (det_loss_forward, (2, 3000, 256, 64, 64)), (det_loss_forward, (8, 20_000, 1024, 256, 64)),
    (det_loss_backward, (2, 3000, 256, 64, 64)), (det_loss_backward, (8, 20_000, 1024, 256, 64)),
    (det_choices, ((100, 200), 50)), (det_choices, ((60_000, 90_000, 30_000), 20_000)),
    (det_points, ((300, 500), 200)), (det_points, ((60_000,) * 4, 40_000)),
    (furthest_point_sampling, (2, 5000, 256)), (furthest_point_sampling, (2, 150_000, 128)),        # on chip; spilled to ws
    (furthest_point_sampling_ragged, ((3000, 5000, 2000), 256)), (furthest_point_sampling_ragged, ((120_000, 30_000), 128)),
    (voxel_down_sample, (2, 200)), (voxel_down_sample, (4, 30_000)),
    (frame_overlap, (2, 200)), (frame_overlap, (4, 30_000)),
    (depth_to_points, (3, 48, 64)), (depth_to_points, (4, 480, 640)),
    (nearest, (5000, 7000)), (nearest, (120_000, 150_000)),
    (text_lines, (2, 20)), (text_lines, (5, 20_000)),
    (scannet_annotate, (500, 40, 8)), (scannet_annotate, (200_000, 3000, 60)),
]
IDS = [f"{f.__name__}{args}".replace(" ", "") for f, args in CASES]


@pytest.mark.parametrize("case,args", CASES, ids=IDS)
def test_short_workspace_is_an_argument_error(case, args):
    q, call, _ = case(*args)
    if q == 0:
        pytest.skip("this shape needs no workspace")
    ws = torch.empty(q - 1, dtype=torch.uint8, device=DEV)
    assert call(ws.data_ptr(), q - 1) == 2
    assert b"bad argument" in L.pcb_last_error()


def test_every_workspace_entry_point_has_a_case():
    """The exports that take a workspace are the ones the cases call: those whose prototype has a size_t parameter (the header, since
    ctypes.c_size_t is ctypes.c_uint64 and would also count a uint64_t seed), and the fused unit's, whose ws sits in its struct."""
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    params = dict(re.findall(r"\b(pcb_\w+)\s*\(([^()]*)\)\s*;", hdr))
    takes_ws = {name for name in _lib._SIGS if re.search(r"\bsize_t\b", params[name])} | {"pcb_unit_forward", "pcb_unit_backward"}
    assert {name for case, _ in CASES for name in case.calls} == takes_ws


@pytest.mark.gpu
def test_python_workspace_is_one_growing_buffer_per_stream():
    """_lib.workspace: every caller on a stream shares one buffer, replaced by a larger one on demand; another stream (the side
    stream of fused.prepare_pair) gets its own."""
    a = _lib.workspace(1000, DEV)
    assert _lib.workspace(10, DEV).data_ptr() == a.data_ptr()
    big = _lib.workspace(a.numel() + 1, DEV)
    assert big.numel() > a.numel() and _lib.workspace(10, DEV).data_ptr() == big.data_ptr()
    with torch.cuda.stream(torch.cuda.Stream()):
        assert _lib.workspace(10, DEV).data_ptr() != big.data_ptr()


@pytest.mark.gpu
@pytest.mark.parametrize("case,args", CASES, ids=IDS)
def test_workspace_tail_untouched_and_size_independent(case, args):
    q, call, outputs = case(*args)
    ws = torch.full((q + TAIL,), 0xA5, dtype=torch.uint8, device=DEV)
    _lib.check(call(ws.data_ptr(), q))
    torch.cuda.synchronize()
    assert bool((ws[q:] == 0xA5).all()), "bytes at or beyond the query were written"
    exact = outputs()
    for size in (q, max(64 << 20, q + 1)):                  # fresh inputs, other workspace contents; the query and a larger size
        q2, call2, outputs2 = case(*args)
        big = torch.full((max(size, 1),), 0x5A, dtype=torch.uint8, device=DEV)
        _lib.check(call2(big.data_ptr(), size))
        torch.cuda.synchronize()
        assert bool((big[q:] == 0x5A).all()), f"bytes at or beyond the query were written with ws_bytes = {size}"
        for a, b in zip(exact, outputs2()):
            assert a.tobytes() == b.tobytes()
