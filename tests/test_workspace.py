"""Workspace contract of libpcb200 (include/pcb200.h, "Conventions"): every entry point that takes `ws` accepts any ws_bytes >= its
*_ws_bytes query, rejects a shorter one with PCB_ERR_ARG before it touches the device, never touches a byte at or beyond the query,
and computes the same bits whatever the size of ws.

Each case below builds one call's inputs from a seed and returns (query, call(ws_ptr, ws_bytes) -> status, outputs() -> arrays).
Without a GPU the tensors live in host memory: only the argument checks run, and they return before any pointer is used."""
import ctypes

import numpy as np
import pytest
import torch

from pointcontrast_b200 import _lib

L = _lib.lib
GPU = torch.cuda.is_available()
DEV = torch.device("cuda:0" if GPU else "cpu")
TAIL = 64 << 10


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


# ------------------------------------------------------------------------------------------------ cases (seeded, one call each)

def voxelize(n):
    i = _In(1)
    xyz, oc, sel, m = i.rand(n, 3, scale=10.0), i.zeros(n, 3, dtype=torch.int32), i.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_voxelize_ws_bytes(n),
            lambda ws, b: L.pcb_voxelize(xyz.data_ptr(), n, 0.25, oc.data_ptr(), sel.data_ptr(), ctypes.byref(m), ws, b, _st()),
            _outputs(oc, sel, m))


def voxelize_labels(n):
    i = _In(2)
    c, lab = i.randint(-60, 60, n, 3), i.randint(0, 4, n)
    oc, sel, ol, m = i.zeros(n, 3, dtype=torch.int32), i.zeros(n, dtype=torch.int32), i.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_voxelize_labels_ws_bytes(n),
            lambda ws, b: L.pcb_voxelize_labels(c.data_ptr(), lab.data_ptr(), n, 255, oc.data_ptr(), sel.data_ptr(), ol.data_ptr(),
                                                ctypes.byref(m), ws, b, _st()),
            _outputs(oc, sel, ol, m))


def voxelize_scenes(B, N):
    i = _In(3)
    xyz, oc, inds, off = i.rand(B, N, 3, scale=5.0), i.zeros(B * N, 4, dtype=torch.int32), i.zeros(B * N, dtype=torch.int32), i.zeros(B + 1, dtype=torch.int64)
    oh = (ctypes.c_int64 * (B + 1))()
    return (L.pcb_voxelize_scenes_ws_bytes(B, N),
            lambda ws, b: L.pcb_voxelize_scenes(xyz.data_ptr(), B, N, 0.1, oc.data_ptr(), inds.data_ptr(), off.data_ptr(), oh, ws, b, _st()),
            _outputs(oc, inds, off, oh))


def radius_pairs(ns, nd):
    i = _In(4)
    src, dst = i.rand(ns, 3, scale=4.0), i.rand(nd, 3, scale=4.0)
    cap = 64 * ns
    pairs, npairs = i.zeros(cap, 2, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_radius_pairs_ws_bytes(ns, nd),
            lambda ws, b: L.pcb_radius_pairs(src.data_ptr(), ns, dst.data_ptr(), nd, 0.1, pairs.data_ptr(), cap, ctypes.byref(npairs), ws, b,
                                             _st()),
            _outputs(pairs, npairs))


def coords_stride(n):
    g = np.random.default_rng(5)
    b, xyz = g.integers(0, 2, n).astype(np.uint64), (g.integers(-300, 300, (n, 3)) + 32768).astype(np.uint64)
    keys = torch.from_numpy(((b << 48) | (xyz[:, 0] << 32) | (xyz[:, 1] << 16) | xyz[:, 2]).view(np.int64)).to(DEV)
    ok, parent, nout = _In.zeros(n, dtype=torch.int64), _In.zeros(n, dtype=torch.int32), ctypes.c_int64()
    return (L.pcb_coords_stride_ws_bytes(n),
            lambda ws, bb: L.pcb_coords_stride(keys.data_ptr(), n, 4, ok.data_ptr(), parent.data_ptr(), ctypes.byref(nout), ws, bb, _st()),
            _outputs(ok, parent, nout))


def gather_points_grad(B, C, N, Lr):
    i = _In(6)
    g, idx, out = i.rand(B, C, Lr), i.randint(0, N, B, Lr), i.zeros(B, C, N)
    return (L.pcb_points_grad_ws_bytes(B, N, Lr),
            lambda ws, b: L.pcb_gather_points_grad(g.data_ptr(), idx.data_ptr(), B, C, N, Lr, out.data_ptr(), ws, b, _st()),
            _outputs(out))


def three_interpolate_grad(B, C, n, m):
    i = _In(7)
    g, idx, w, out = i.rand(B, C, n), i.randint(0, m, B, n, 3), i.rand(B, n, 3), i.zeros(B, C, m)
    return (L.pcb_points_grad_ws_bytes(B, m, 3 * n),
            lambda ws, b: L.pcb_three_interpolate_grad(g.data_ptr(), idx.data_ptr(), w.data_ptr(), B, C, n, m, out.data_ptr(), ws, b, _st()),
            _outputs(out))


def gather_rows_grad(Lr, C, M):
    i = _In(8)
    g, idx, out = i.rand(Lr, C), i.randint(0, M, Lr), i.zeros(M, C)
    return (L.pcb_points_grad_ws_bytes(1, M, Lr),
            lambda ws, b: L.pcb_gather_rows_grad(g.data_ptr(), idx.data_ptr(), Lr, C, M, out.data_ptr(), ws, b, _st()),
            _outputs(out))


def point_bounds(n):
    xyz = _In(9).rand(n, 3, scale=7.0)
    lo, hi = (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    return (L.pcb_point_bounds_ws_bytes(), lambda ws, b: L.pcb_point_bounds(xyz.data_ptr(), n, lo, hi, ws, b, _st()), _outputs(lo, hi))


def elastic_distort(n, gx, gy, gz):
    i = _In(10)
    xyz, noise = i.rand(n, 3, scale=10.0), i.rand(gx, gy, gz, 3)
    axes = torch.from_numpy(np.concatenate([np.linspace(-1.0, 11.0, k) for k in (gx, gy, gz)])).to(DEV)
    return (L.pcb_elastic_distort_ws_bytes(gx, gy, gz),
            lambda ws, b: L.pcb_elastic_distort(xyz.data_ptr(), n, noise.data_ptr(), gx, gy, gz, axes.data_ptr(), 0.5, ws, b, _st()),
            _outputs(xyz, noise))


def affine_floor(n):
    xyz, out = _In(11).rand(n, 3, scale=4.0), _In.zeros(n, 3, dtype=torch.int32)
    T = np.ascontiguousarray([[50.0, 1.0, 0, 3], [0, 45.0, 2.0, -1], [1.0, 0, 55.0, 0.5], [0, 0, 0, 1]], np.float64).reshape(16)
    mn = (ctypes.c_int32 * 3)()
    return (L.pcb_affine_floor_ws_bytes(),
            lambda ws, b: L.pcb_affine_floor(xyz.data_ptr(), n, T.ctypes.data, out.data_ptr(), mn, ws, b, _st()),
            _outputs(out, mn))


def input_transform(n):
    i = _In(12)
    coords, feats, noise = i.randint(0, 100, n, 3), i.rand(n, 3, scale=255.0), i.rand(n, 3, dtype=torch.float64)
    tr = (ctypes.c_double * 3)(1.0, -2.0, 3.0)
    return (L.pcb_semseg_input_transform_ws_bytes(),
            lambda ws, b: L.pcb_semseg_input_transform(coords.data_ptr(), feats.data_ptr(), n, 5, 1, 0.3, tr, noise.data_ptr(), 12.75, 1, ws, b,
                                                       _st()),
            _outputs(coords, feats))


def bn_stats(n, n0, C):
    i = _In(13)
    X, mean, invstd, rm, rv = i.rand(n, C, scale=3.0), i.zeros(2 * C), i.zeros(2 * C), i.zeros(C), i.rand(C)
    return (L.pcb_bn_ws_bytes(n, C),
            lambda ws, b: L.pcb_bn_stats_seg(X.data_ptr(), C, n, n0, C, 1e-5, 0.1, mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(),
                                             rv.data_ptr(), ws, b, _st()),
            _outputs(mean, invstd, rm, rv))


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


def nce(n, D):
    i = _In(15)
    q, k = torch.nn.functional.normalize(i.rand(n, D) - 0.5, dim=1), torch.nn.functional.normalize(i.rand(n, D) - 0.5, dim=1)
    loss, dq, dk = i.zeros(1), i.zeros(n, D), i.zeros(n, D)
    return (L.pcb_nce_ws_bytes(n),
            lambda ws, b: L.pcb_nce_forward_backward(q.data_ptr(), k.data_ptr(), n, D, 1 / 0.07, loss.data_ptr(), dq.data_ptr(), dk.data_ptr(), ws,
                                                     b, _st()),
            _outputs(loss, dq, dk))


def ce(n, C):
    i = _In(16)
    x, t = i.rand(n, C, scale=4.0), i.randint(0, C + 3, n, dtype=torch.int64)      # targets >= C: ignored
    loss, dx = i.zeros(1), i.zeros(n, C)
    return (L.pcb_ce_ws_bytes(n),
            lambda ws, b: L.pcb_ce_forward_backward(x.data_ptr(), t.data_ptr(), n, C, C, 1.0, loss.data_ptr(), dx.data_ptr(), ws, b, _st()),
            _outputs(loss, dx))


def conv_wgrad(K, n_out, Ca, Cb):
    i = _In(17)
    n_in = n_out + 17
    A, Bm, tbl, dW = i.rand(n_in, Ca), i.rand(n_out, Cb), i.randint(-1, n_in, K, n_out), i.zeros(K, Ca, Cb)
    return (L.pcb_conv_wgrad_ws_bytes(K, n_out, Ca, Cb),
            lambda ws, b: L.pcb_conv_wgrad(A.data_ptr(), Ca, Bm.data_ptr(), Cb, tbl.data_ptr(), n_out, K, n_out, Ca, Cb, dW.data_ptr(), 0, ws, b,
                                           0, _st()),
            _outputs(dW))


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
]
IDS = [f"{f.__name__}{args}".replace(" ", "") for f, args in CASES]


@pytest.mark.parametrize("case,args", CASES, ids=IDS)
def test_short_workspace_is_an_argument_error(case, args):
    q, call, _ = case(*args)
    if q == 0:
        pytest.skip("an unsplit convolution needs no workspace")
    ws = torch.empty(q - 1, dtype=torch.uint8, device=DEV)
    assert call(ws.data_ptr(), q - 1) == 2
    assert b"bad argument" in L.pcb_last_error()


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
    q2, call2, outputs2 = case(*args)
    big = torch.full((max(64 << 20, q + 1),), 0x5A, dtype=torch.uint8, device=DEV)
    _lib.check(call2(big.data_ptr(), big.numel()))
    torch.cuda.synchronize()
    for a, b in zip(exact, outputs2()):
        assert a.tobytes() == b.tobytes()
