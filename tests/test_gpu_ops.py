"""Per-operator parity on the GPU against the fp64 oracle (tolerance: 1e-3 relative, the north-star bar; the split-operand
tensor-core path is expected near 1e-5, the exact SIMT path near 1e-6)."""
import numpy as np
import pytest
import torch

from oracle import loss_cpu
from oracle import me_cpu as OR
from tests.helpers import max_rel_err, rand_coords, rel_err, surface_coords

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _pair(kind, cin, cout, bias=False):
    from pointcontrast_b200 import me
    def gen(M):
        if kind == "k3hyb":
            return M.KernelGenerator(3, 1, 1, region_type=M.RegionType.HYBRID, axis_types=[M.RegionType.HYPERCUBE] * 3, dimension=3)
        if kind == "k3cube":
            return M.KernelGenerator([3, 3, 3], 1, 1, region_type=M.RegionType.HYPERCUBE, dimension=3)
        if kind == "k1":
            return M.KernelGenerator(1, 1, 1, dimension=3)
        return M.KernelGenerator([2, 2, 2], 2, 1, dimension=3)
    stride = 2 if kind in ("down", "up") else 1
    ks = {"k3hyb": 3, "k3cube": [3, 3, 3], "k1": 1}.get(kind, [2, 2, 2])
    def make(M):
        cls = M.MinkowskiConvolutionTranspose if kind == "up" else M.MinkowskiConvolution
        return cls(in_channels=cin, out_channels=cout, kernel_size=ks, stride=stride, dilation=1, has_bias=bias,
                   kernel_generator=gen(M), dimension=3)
    return make(me), make(OR)


CASES = [("k3cube", 3, 32, False), ("k3hyb", 32, 32, False), ("k3hyb", 32, 64, False), ("k3hyb", 128, 96, False),
         ("k3hyb", 96, 96, False), ("k3hyb", 256, 256, False), ("k3hyb", 384, 256, False), ("k3hyb", 192, 128, False),
         ("k1", 96, 32, True), ("k1", 128, 96, False), ("down", 32, 32, False), ("down", 128, 128, False),
         ("up", 256, 128, False), ("up", 96, 96, False)]


@pytest.mark.parametrize("simt", [False, True])
@pytest.mark.parametrize("kind,cin,cout,bias", CASES)
def test_conv_forward_backward(kind, cin, cout, bias, simt):
    from pointcontrast_b200 import me
    if simt and cin * cout > 128 * 96:
        pytest.skip("exact SIMT kernel is only exercised on the smaller shapes")
    rng = np.random.default_rng(cin * 1000 + cout)
    n = 3000 if cin * cout <= 128 * 128 else 1200
    coords = surface_coords(rng, n)
    g = torch.Generator().manual_seed(cin + cout)
    conv, oconv = _pair(kind, cin, cout, bias)
    oconv = oconv.double()
    with torch.no_grad():
        oconv.kernel.copy_(conv.kernel.double())
        if bias:
            oconv.bias.copy_(conv.bias.double())
    conv = conv.cuda()
    # input level: the fine level for k3/k1/down, the strided level for up
    st0 = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    ost0 = OR.SparseTensor(torch.zeros(len(coords), 1, dtype=torch.float64), coords=torch.from_numpy(coords))
    if kind == "up":
        key = st0.coords_man.stride(st0.coords_key, [2, 2, 2]); okey = ost0.coords_man.stride(ost0.coords_key, [2, 2, 2])
    else:
        key, okey = st0.coords_key, ost0.coords_key
    n_in = st0.coords_man.num_rows(key)
    x = torch.randn(n_in, cin, generator=g, dtype=torch.float64)
    xg = x.float().cuda().requires_grad_(True)
    xo = x.clone().requires_grad_(True)
    me.FORCE_SIMT = simt
    try:
        y = conv(me.SparseTensor(xg, coords_key=key, coords_manager=st0.coords_man))
        yo = oconv(OR.SparseTensor(xo, coords_key=okey, coords_manager=ost0.coords_man))
        assert y.F.shape == yo.F.shape and y.coords_key.ts == yo.coords_key.ts
        dy = torch.randn(yo.F.shape, generator=g, dtype=torch.float64)
        y.F.backward(dy.float().cuda())
        yo.F.backward(dy)
    finally:
        me.FORCE_SIMT = False
    assert max_rel_err(y.F, yo.F) < TOL and rel_err(y.F, yo.F) < TOL / 10
    assert max_rel_err(xg.grad, xo.grad) < TOL and rel_err(xg.grad, xo.grad) < TOL / 10
    assert max_rel_err(conv.kernel.grad, oconv.kernel.grad) < TOL and rel_err(conv.kernel.grad, oconv.kernel.grad) < TOL / 10
    if bias:
        assert rel_err(conv.bias.grad, oconv.bias.grad) < TOL / 10


def test_tensor_core_and_simt_paths_agree_tightly():
    from pointcontrast_b200 import me
    rng = np.random.default_rng(11)
    coords = surface_coords(rng, 6000)
    conv, _ = _pair("k3hyb", 96, 96)
    conv = conv.cuda()
    st = me.SparseTensor(torch.randn(len(coords), 96, device="cuda"), coords=torch.from_numpy(coords))
    y_tc = conv(st).F
    me.FORCE_SIMT = True
    try:
        y_simt = conv(st).F
    finally:
        me.FORCE_SIMT = False
    assert max_rel_err(y_tc, y_simt) < 1e-4


@pytest.mark.parametrize("n,C", [(5000, 32), (777, 96), (1, 64), (20000, 256), (3001, 384)])
def test_batchnorm_matches_torch(n, C):
    from pointcontrast_b200 import me
    g = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, C, generator=g, dtype=torch.float64) * 2 + 0.5
    bn = me.MinkowskiBatchNorm(C, momentum=0.05).cuda()
    ref = torch.nn.BatchNorm1d(C, momentum=0.05).double()
    with torch.no_grad():
        w = torch.rand(C, generator=g, dtype=torch.float64) + 0.5; b = torch.randn(C, generator=g, dtype=torch.float64)
        bn.bn.weight.copy_(w.float()); bn.bn.bias.copy_(b.float()); ref.weight.copy_(w); ref.bias.copy_(b)
    coords = torch.cat([torch.zeros(n, 1, dtype=torch.int32), torch.arange(n, dtype=torch.int32)[:, None].repeat(1, 3)], 1)
    xg = x.float().cuda().requires_grad_(True)
    xo = x.clone().requires_grad_(True)
    if n == 1:
        y = bn(me.SparseTensor(xg, coords=coords)).F          # torch refuses n == 1 in training; ours gives beta
        assert torch.allclose(y.cpu().double(), b[None], atol=1e-5)
        return
    y = bn(me.SparseTensor(xg, coords=coords)).F
    yo = ref(xo)
    dy = torch.randn(n, C, generator=g, dtype=torch.float64)
    y.backward(dy.float().cuda()); yo.backward(dy)
    assert max_rel_err(y, yo) < 1e-4 and max_rel_err(xg.grad, xo.grad) < 1e-4
    assert rel_err(bn.bn.weight.grad, ref.weight.grad) < 1e-4 and rel_err(bn.bn.bias.grad, ref.bias.grad) < 1e-4
    assert rel_err(bn.bn.running_mean, ref.running_mean) < 1e-5 and rel_err(bn.bn.running_var, ref.running_var) < 1e-5
    assert int(bn.bn.num_batches_tracked) == 1
    bn.eval(); ref.eval()
    assert max_rel_err(bn(me.SparseTensor(xg.detach(), coords=coords)).F, ref(x)) < 1e-4


@pytest.mark.parametrize("n,T", [(4096, 0.4), (1000, 0.07), (37, 0.4)])
def test_point_nce_loss_and_grads(n, T):
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(n)
    N0, N1 = 3 * n, 3 * n + 11
    F0 = torch.nn.functional.normalize(torch.randn(N0, 32, generator=g, dtype=torch.float64), dim=1)
    F1 = torch.nn.functional.normalize(torch.randn(N1, 32, generator=g, dtype=torch.float64), dim=1)
    q_rows = torch.randperm(N0, generator=g)[:n]
    k_rows = torch.randint(0, N1, (n,), generator=g)          # keys may repeat
    F1[k_rows] = F1[k_rows] * 0.5 + F0[q_rows] * 0.5
    f0o, f1o = F0.clone().requires_grad_(True), F1.clone().requires_grad_(True)
    lo = loss_cpu.point_nce_loss(f0o, f1o, q_rows, k_rows, T)
    lo.backward()
    f0, f1 = F0.float().cuda().requires_grad_(True), F1.float().cuda().requires_grad_(True)
    l = losses.point_nce_loss(f0, f1, q_rows.cuda(), k_rows.cuda(), T)
    l.backward()
    assert abs(float(l) - float(lo)) / abs(float(lo)) < 1e-4
    assert rel_err(f0.grad, f0o.grad) < 1e-4 and rel_err(f1.grad, f1o.grad) < 1e-4


def test_hardest_contrastive_loss_and_grads():
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(5)
    N0, N1, P = 6000, 5500, 20000
    F0 = torch.nn.functional.normalize(torch.randn(N0, 32, generator=g, dtype=torch.float64), dim=1)
    F1 = torch.nn.functional.normalize(torch.randn(N1, 32, generator=g, dtype=torch.float64), dim=1)
    F1[:3000] = torch.nn.functional.normalize(F0[:3000] + 0.3 * torch.randn(3000, 32, generator=g, dtype=torch.float64), dim=1)
    rng = np.random.default_rng(0)
    i0 = np.sort(rng.integers(0, 3000, P))
    pairs = np.unique(np.stack([i0, np.clip(i0 + rng.integers(-2, 3, P), 0, N1 - 1)], 1), axis=0)
    sel0 = rng.choice(N0, 1024, replace=False); sel1 = rng.choice(N1, 1024, replace=False)
    pos_sel = rng.choice(len(pairs), 4096, replace=False)
    f0o, f1o = F0.clone().requires_grad_(True), F1.clone().requires_grad_(True)
    po, no = loss_cpu.hardest_contrastive_loss(f0o, f1o, pairs, sel0, sel1, pos_sel)
    (po + no).backward()
    f0, f1 = F0.float().cuda().requires_grad_(True), F1.float().cuda().requires_grad_(True)
    p, n_ = losses.hardest_contrastive_loss(f0, f1, torch.from_numpy(pairs).cuda(), torch.from_numpy(sel0).cuda(),
                                            torch.from_numpy(sel1).cuda(), torch.from_numpy(pos_sel).cuda())
    (p + n_).backward()
    assert abs(float(p) - float(po)) < 1e-5 and abs(float(n_) - float(no)) < 1e-4
    assert rel_err(f0.grad, f0o.grad) < 1e-3 and rel_err(f1.grad, f1o.grad) < 1e-3


def test_pdist_rowmin_against_torch():
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(9)
    for P, S, D in ((4096, 1024, 32), (100, 3000, 32), (1, 1, 32), (513, 65, 16)):
        A = torch.randn(P, D, generator=g); B = torch.randn(S, D, generator=g)
        mv, am = losses.pdist_rowmin(A.cuda(), B.cuda())
        D2 = torch.sqrt(((A.double()[:, None] - B.double()[None]) ** 2).sum(2) + 1e-7)
        rv, ra = D2.min(1)
        assert torch.allclose(mv.cpu().double(), rv, rtol=1e-5, atol=1e-6)
        picked = D2[torch.arange(P), am.cpu().long()]
        assert torch.allclose(picked, rv, rtol=1e-5, atol=1e-6)      # argmin may differ only between numerical ties


def test_sgd_matches_torch():
    from pointcontrast_b200 import optim as pco
    g = torch.Generator().manual_seed(1)
    shapes = [(27, 32, 64), (64,), (1, 32), (7,)]
    ps = [torch.randn(s, generator=g) for s in shapes]
    ref = [p.clone().requires_grad_(True) for p in ps]
    mine = [torch.nn.Parameter(p.clone().cuda()) for p in ps]
    o_ref = torch.optim.SGD(ref, lr=0.1, momentum=0.8, weight_decay=1e-4)
    o = pco.FlatSGD(mine, lr=0.1, momentum=0.8, weight_decay=1e-4)
    for step in range(3):
        for r, m in zip(ref, mine):
            gr = torch.randn(r.shape, generator=g)
            r.grad = gr.clone(); m.grad.copy_(gr.cuda()) if m.grad is not None else setattr(m, "grad", gr.cuda())
        o_ref.step(); o.step()
        for r, m in zip(ref, mine):
            assert torch.allclose(m.detach().cpu(), r.detach(), rtol=1e-6, atol=1e-7)
    sd = o.state_dict()
    assert sd["param_groups"][0]["momentum"] == 0.8 and len(sd["state"]) == len(shapes)


def _split(x, flags=0):
    from pointcontrast_b200._lib import check, lib, ptr, stream
    n, C = x.shape
    planes = torch.empty(2, n * C, dtype=torch.bfloat16, device="cuda")
    check(lib.pcb_split_rows(ptr(x), C, n, C, planes[0].data_ptr(), planes[1].data_ptr(), C, flags, stream()))
    return planes


@pytest.mark.parametrize("Ca,Cb,tr", [(96, 96, 0), (128, 96, 0), (32, 32, 0), (64, 64, 1), (256, 256, 0), (384, 256, 0),
                                       (192, 128, 1), (96, 32, 0), (256, 128, 1), (32, 96, 0)])
def test_split_operand_wgrad_tcgen05_matches_exact_fp32_kernel(Ca, Cb, tr):
    """Tensor-core weight-gradient on bf16 hi/lo planes (MN-major wgmma operands) vs the exact fp32 SIMT kernel of the library."""
    from pointcontrast_b200 import me
    from pointcontrast_b200._lib import check, lib, ptr, stream
    rng = np.random.default_rng(Ca + Cb)
    coords = surface_coords(rng, 3000 if Ca * Cb <= 128 * 128 else 900)
    st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    kg = me.KernelGenerator(3, 1, 1, region_type=me.RegionType.HYBRID, axis_types=[me.RegionType.HYPERCUBE] * 3, dimension=3)
    plan = st.coords_man.conv_plan(st.coords_key, st.coords_key, kg, False)
    n = plan.n_out
    A = torch.randn(n, Ca, device="cuda"); B = torch.randn(n, Cb, device="cuda")
    K = 27
    shape = (K, Cb, Ca) if tr else (K, Ca, Cb)
    ref = torch.empty(shape, device="cuda"); got = torch.full(shape, 0.5, device="cuda")
    wsb = lib.pcb_conv_wgrad_ws_bytes(K, n, Ca, Cb); ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    check(lib.pcb_conv_wgrad(ptr(A), Ca, ptr(B), Cb, ptr(plan.wg_tbl), plan.wg_tbl.shape[1], K, n, Ca, Cb, ptr(ref), tr, ptr(ws), wsb, 1, stream()))
    As, Bs = _split(A), _split(B)
    wsb = lib.pcb_conv_wgrad_split_ws_bytes(K, n, Ca, Cb); ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    check(lib.pcb_conv_wgrad_split(As[0].data_ptr(), As[1].data_ptr(), Ca, Bs[0].data_ptr(), Bs[1].data_ptr(), Cb, ptr(plan.wg_tbl),
                                   plan.wg_tbl.shape[1], K, n, Ca, Cb, ptr(got), tr, ptr(ws), wsb, 4, stream()))      # accumulate onto 0.5
    torch.cuda.synchronize()
    assert max_rel_err(got - 0.5, ref) < 1e-4          # bf16 hi/lo products (2^-17) vs exact fp32
    # and against fp64
    tbl = plan.wg_tbl.long()
    k = 5
    ok = tbl[k] >= 0
    exact = A.double()[tbl[k][ok]].t() @ B.double()[ok]
    mine = (got[k] - 0.5).double()
    assert max_rel_err(mine.t() if tr else mine, exact) < 1e-4


@pytest.mark.parametrize("cin,cout", [(96, 96), (128, 96), (32, 64), (256, 256), (384, 256)])
def test_split_operand_conv_forward_matches_exact_fp32_kernel(cin, cout):
    """Tensor-core forward / data gradient on bf16 hi/lo planes and pre-tiled weights vs the exact fp32 SIMT kernel of the library."""
    from pointcontrast_b200 import me
    from pointcontrast_b200._lib import check, lib, ptr, stream
    rng = np.random.default_rng(cin + cout)
    coords = surface_coords(rng, 4000 if cin * cout <= 128 * 128 else 1200)
    st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    kg = me.KernelGenerator(3, 1, 1, region_type=me.RegionType.HYBRID, axis_types=[me.RegionType.HYPERCUBE] * 3, dimension=3)
    plan = st.coords_man.conv_plan(st.coords_key, st.coords_key, kg, False)
    n = plan.n_out
    X = torch.randn(n, cin, device="cuda"); W = torch.randn(27, cin, cout, device="cuda") * 0.05
    ref = torch.empty(n, cout, device="cuda")
    check(lib.pcb_conv_forward(ptr(X), cin, ptr(plan.fwd_tbl), plan.fwd_tbl.shape[1], None, 27, n, cin, cout, ptr(W), None, ptr(ref), cout,
                               stream()))
    Xs = _split(X)
    got = torch.full((n, cout), 0.25, device="cuda")
    wsb = lib.pcb_conv_forward_split_ws_bytes(27, n, cin, cout); ws = torch.empty(max(wsb, 256), dtype=torch.uint8, device="cuda")
    ft = torch.empty(lib.pcb_weight_tile_bytes(27, cin, cout, 0), dtype=torch.uint8, device="cuda")
    dt = torch.empty(lib.pcb_weight_tile_bytes(27, cin, cout, 1), dtype=torch.uint8, device="cuda")
    check(lib.pcb_weight_tile(ptr(W), 27, cin, cout, ptr(ft), ptr(dt), 0, stream()))
    check(lib.pcb_conv_forward_split(Xs[0].data_ptr(), Xs[1].data_ptr(), cin, ptr(plan.fwd_tbl), plan.fwd_tbl.shape[1], None, 27, n, cin,
                                     cout, ptr(ft), None, ptr(got), cout, ptr(ws), wsb, 4, stream()))      # accumulate onto 0.25
    torch.cuda.synchronize()
    assert max_rel_err(got - 0.25, ref) < 1e-4          # bf16 hi/lo products (2^-17) vs exact fp32
    # and against fp64, offset by offset
    def fp64(tbl, kmap, A, Wk):
        out = torch.zeros(n, Wk.shape[2], dtype=torch.float64, device="cuda")
        for k in range(27):
            t = tbl[kmap[k] if kmap is not None else k].long()
            ok = t >= 0
            out[ok] += A.double()[t[ok]] @ Wk[k].double()
        return out
    assert max_rel_err(got - 0.25, fp64(plan.fwd_tbl, None, X, W)) < 1e-4
    # data-gradient roles: dX = sum_k dY[tbl[opp k]] W[k]^T through the dgrad tiles vs the exact kernel on the transposed weights
    dY = torch.randn(n, cout, device="cuda")
    opp = plan.dg_kmap
    Wt = W.transpose(1, 2).contiguous()
    ref_dx = torch.empty(n, cin, device="cuda")
    check(lib.pcb_conv_forward(ptr(dY), cout, ptr(plan.dg_tbl), plan.dg_tbl.shape[1], me._c_int_array(opp), 27, n, cout, cin, ptr(Wt), None,
                               ptr(ref_dx), cin, stream()))
    dYs = _split(dY)
    got_dx = torch.empty(n, cin, device="cuda")
    wsb = lib.pcb_conv_forward_split_ws_bytes(27, n, cout, cin); ws = torch.empty(max(wsb, 256), dtype=torch.uint8, device="cuda")
    check(lib.pcb_conv_forward_split(dYs[0].data_ptr(), dYs[1].data_ptr(), cout, ptr(plan.dg_tbl), plan.dg_tbl.shape[1],
                                     me._c_int_array(opp), 27, n, cout, cin, ptr(dt), None, ptr(got_dx), cin, ptr(ws), wsb, 0, stream()))
    torch.cuda.synchronize()
    assert max_rel_err(got_dx, ref_dx) < 1e-4
    assert max_rel_err(got_dx, fp64(plan.dg_tbl, opp, dY, Wt)) < 1e-4


@pytest.mark.parametrize("n0,n1,C", [(5000, 3777, 32), (130, 1, 96), (128, 128, 64), (1, 300, 256)])
def test_segmented_batchnorm_relu_hi_plane_equals_two_batches(n0, n1, C):
    """pcb_bn_*_seg: rows [0,n0) and [n0,n0+n1) normalised as two batches (the two views of a pair stacked in one matrix)
    == torch BatchNorm1d applied to view 0 and then to view 1 (fp64), including the sequential running-stat updates and
    the summed parameter gradients; residual + ReLU folded in as in the fused executor, the backward taking its ReLU mask
    from the bf16 hi plane the apply pass wrote."""
    from pointcontrast_b200 import _lib
    from pointcontrast_b200._lib import check, lib, ptr, stream
    n = n0 + n1
    g = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, C, generator=g, dtype=torch.float64) * 1.5 + 0.3
    res = torch.randn(n, C, generator=g, dtype=torch.float64)
    dy = torch.randn(n, C, generator=g, dtype=torch.float64)
    w = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    b = torch.randn(C, generator=g, dtype=torch.float64)
    ref = torch.nn.BatchNorm1d(C, momentum=0.1).double()
    with torch.no_grad():
        ref.weight.copy_(w); ref.bias.copy_(b)
    xo = x.clone().requires_grad_(True)
    ro = res.clone().requires_grad_(True)
    if n0 > 1 and n1 > 1:
        yo = torch.relu(torch.cat([ref(xo[:n0]), ref(xo[n0:])]) + ro)
        yo.backward(dy)
    dev = torch.device("cuda")
    X, R, DY = x.float().to(dev), res.float().to(dev), dy.float().to(dev)
    W, B = w.float().to(dev), b.float().to(dev)
    mean = torch.empty(2, C, device=dev); invstd = torch.empty(2, C, device=dev)
    rm = torch.zeros(C, device=dev); rv = torch.ones(C, device=dev)
    wsb = lib.pcb_bn_ws_bytes(n, C)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    Y = torch.empty(n, C, device=dev)
    hi = torch.empty(n, C, dtype=torch.bfloat16, device=dev); lo = torch.empty(n, C, dtype=torch.bfloat16, device=dev)
    st = stream()
    check(lib.pcb_bn_stats_seg(ptr(X), C, n, n0, C, 1e-5, 0.1, ptr(mean), ptr(invstd), ptr(rm), ptr(rv), ptr(ws), wsb, st))
    check(lib.pcb_bn_apply_seg(ptr(X), C, n, n0, C, ptr(mean), ptr(invstd), ptr(W), ptr(B), ptr(R), C, 1, ptr(Y), C, ptr(hi), ptr(lo), C, None, None, st))
    for s, (a, e) in enumerate(((0, n0), (n0, n))):
        m = x[a:e].mean(0); v = x[a:e].var(0, unbiased=False)
        assert rel_err(mean[s], m) < 1e-5
        if e - a > 1:       # one row: x - mean == 0 whatever invstd is (E[x^2] - mean^2 cancels to ~1e-7 x^2 next to eps = 1e-5)
            assert rel_err(invstd[s], 1 / torch.sqrt(v + 1e-5)) < 1e-5
        else:
            assert rel_err(invstd[s], 1 / torch.sqrt(v + 1e-5)) < 5e-2
    assert max_rel_err(hi.float() + lo.float(), Y) < 1e-4
    if not (n0 > 1 and n1 > 1):
        return
    assert max_rel_err(Y, yo) < 1e-4
    assert rel_err(rm, ref.running_mean) < 1e-5 and rel_err(rv, ref.running_var) < 1e-5
    dX = torch.empty(n, C, device=dev); dW = torch.zeros(C, device=dev); dB = torch.zeros(C, device=dev)
    gout = torch.empty(n, C, device=dev)
    check(lib.pcb_bn_backward_seg(ptr(DY), C, ptr(X), C, ptr(hi), C, n, n0, C, ptr(mean), ptr(invstd), ptr(W), ptr(dX), C, ptr(dW), ptr(dB), 1,
                                  ptr(gout), C, 1, None, None, 0, ptr(ws), wsb, st))
    assert max_rel_err(dX, xo.grad) < 1e-4 and max_rel_err(gout, ro.grad) < 1e-5
    assert rel_err(dW, ref.weight.grad) < 1e-4 and rel_err(dB, ref.bias.grad) < 1e-4


@pytest.mark.parametrize("n,C", [(5000, 32), (3, 13), (777, 96)])
def test_l2_normalize_matches_torch(n, C):
    """`model/res16unet.py:262-266`: F / ||F||_2 per row (no epsilon), forward and backward, vs torch fp64."""
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, C, generator=g, dtype=torch.float64)
    dy = torch.randn(n, C, generator=g, dtype=torch.float64)
    xo = x.clone().requires_grad_(True)
    yo = xo / torch.norm(xo, p=2, dim=1, keepdim=True)
    yo.backward(dy)
    xg = x.float().cuda().requires_grad_(True)
    y = losses.l2_normalize(xg)
    y.backward(dy.float().cuda())
    assert max_rel_err(y, yo) < 1e-6 and max_rel_err(xg.grad, xo.grad) < 1e-5


@pytest.mark.parametrize("n,D,T", [(2000, 64, 0.4), (300, 32, 0.07)])
def test_point_nce_tensor_core_and_simt_paths_agree(n, D, T, monkeypatch):
    """The fused tensor-core PointInfoNCE (D = 32 / 64) against the oracle AND against the exact-fp32 SIMT kernels of the same
    library (the SIMT side is reached through a width the tiling does not cover)."""
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(n + D)
    F0 = torch.nn.functional.normalize(torch.randn(n, D, generator=g, dtype=torch.float64), dim=1)
    F1 = torch.nn.functional.normalize(0.6 * F0 + 0.4 * torch.randn(n, D, generator=g, dtype=torch.float64), dim=1)
    rows = torch.arange(n)
    f0o, f1o = F0.clone().requires_grad_(True), F1.clone().requires_grad_(True)
    lo = loss_cpu.point_nce_loss(f0o, f1o, rows, rows, T)
    lo.backward()
    f0, f1 = F0.float().cuda().requires_grad_(True), F1.float().cuda().requires_grad_(True)
    l = losses.point_nce_loss(f0, f1, rows.cuda(), rows.cuda(), T)
    l.backward()
    assert abs(float(l) - float(lo)) / abs(float(lo)) < 1e-4
    assert rel_err(f0.grad, f0o.grad) < 1e-4 and rel_err(f1.grad, f1o.grad) < 1e-4
    # SIMT path of the library: pad the features with 4 zero channels (D + 4 is not a tensor-core width; the loss is unchanged)
    pad = torch.zeros(n, 4)
    f0s = torch.cat([F0.float(), pad], 1).cuda().requires_grad_(True)
    f1s = torch.cat([F1.float(), pad], 1).cuda().requires_grad_(True)
    ls = losses.point_nce_loss(f0s, f1s, rows.cuda(), rows.cuda(), T)
    ls.backward()
    assert abs(float(l) - float(ls)) / abs(float(ls)) < 1e-5
    assert rel_err(f0.grad, f0s.grad[:, :D]) < 1e-4 and rel_err(f1.grad, f1s.grad[:, :D]) < 1e-4


@pytest.mark.parametrize("n,C", [(5000, 13), (333, 20), (64, 32)])
def test_cross_entropy_with_ignore_index_matches_torch(n, C):
    """`nn.CrossEntropyLoss(ignore_index=255)` (`downstream/semseg/lib/train.py:68,120`), loss and gradient, vs torch fp64."""
    from pointcontrast_b200 import losses
    g = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, C, generator=g, dtype=torch.float64) * 3
    t = torch.randint(0, C, (n,), generator=g)
    t[torch.rand(n, generator=g) < 0.2] = 255
    xo = x.clone().requires_grad_(True)
    lo = torch.nn.functional.cross_entropy(xo, t, ignore_index=255)
    (lo * 0.5).backward()
    xg = x.float().cuda().requires_grad_(True)
    l = losses.cross_entropy(xg, t.cuda(), 255)
    (l * 0.5).backward()
    assert abs(float(l.detach()) - float(lo.detach())) / abs(float(lo.detach())) < 1e-5
    assert max_rel_err(xg.grad, xo.grad) < 1e-5


def test_sgd_with_dampening_and_poly_lr_match_torch():
    """`downstream/semseg/lib/solvers.py:27-32,50-57`: SGD(momentum 0.9, dampening 0.1, wd 1e-4) under PolyLR(power 0.9)."""
    from pointcontrast_b200 import optim as pco
    g = torch.Generator().manual_seed(3)
    shapes = [(27, 32, 64), (64,), (1, 13)]
    ps = [torch.randn(s, generator=g) for s in shapes]
    ref = [p.clone().requires_grad_(True) for p in ps]
    mine = [torch.nn.Parameter(p.clone().cuda()) for p in ps]
    o_ref = torch.optim.SGD(ref, lr=0.01, momentum=0.9, dampening=0.1, weight_decay=1e-4)
    o = pco.FlatSGD(mine, lr=0.01, momentum=0.9, dampening=0.1, weight_decay=1e-4)
    s_ref = torch.optim.lr_scheduler.LambdaLR(o_ref, lambda s: (1 - s / (10 + 1)) ** 0.9)
    s = pco.PolyLR(o, max_iter=10, power=0.9)
    for step in range(4):
        for r, m in zip(ref, mine):
            gr = torch.randn(r.shape, generator=g)
            r.grad = gr.clone(); m.grad.copy_(gr.cuda())
        o_ref.step(); o.step(); s_ref.step(); s.step()
        assert abs(s.get_last_lr()[0] - s_ref.get_last_lr()[0]) < 1e-12
        for r, m in zip(ref, mine):
            assert torch.allclose(m.detach().cpu(), r.detach(), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("kind", ["sum", "avg", "unpool", "pool_tr", "sum_k3"])
def test_pooling_layers_match_oracle(kind):
    """MinkowskiSumPooling / AvgPooling / PoolingTranspose / AvgUnpooling (SURVEY.md 8f-4) forward and backward vs the oracle's
    restatement on the same kernel maps (fp64)."""
    from pointcontrast_b200 import me
    rng = np.random.default_rng(len(kind))
    coords = surface_coords(rng, 4000)
    C = 24 if kind != "sum_k3" else 6           # 6: not a multiple of 4 (padded internally)
    g = torch.Generator().manual_seed(3)
    cls = {"sum": "MinkowskiSumPooling", "avg": "MinkowskiAvgPooling", "unpool": "MinkowskiAvgUnpooling", "pool_tr": "MinkowskiPoolingTranspose",
           "sum_k3": "MinkowskiSumPooling"}[kind]
    ks, st = ([3, 3, 3], 1) if kind == "sum_k3" else ([2, 2, 2], 2)
    layer, olayer = getattr(me, cls)(kernel_size=ks, stride=st, dimension=3), getattr(OR, cls)(kernel_size=ks, stride=st, dimension=3)
    st0 = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    ost0 = OR.SparseTensor(torch.zeros(len(coords), 1, dtype=torch.float64), coords=torch.from_numpy(coords))
    if kind in ("unpool", "pool_tr"):
        key = st0.coords_man.stride(st0.coords_key, [2, 2, 2]); okey = ost0.coords_man.stride(ost0.coords_key, [2, 2, 2])
    else:
        key, okey = st0.coords_key, ost0.coords_key
    n_in = st0.coords_man.num_rows(key)
    x = torch.randn(n_in, C, generator=g, dtype=torch.float64)
    xg, xo = x.float().cuda().requires_grad_(True), x.clone().requires_grad_(True)
    y = layer(me.SparseTensor(xg, coords_key=key, coords_manager=st0.coords_man))
    yo = olayer(OR.SparseTensor(xo, coords_key=okey, coords_manager=ost0.coords_man))
    assert y.F.shape == yo.F.shape and y.coords_key.ts == yo.coords_key.ts
    dy = torch.randn(yo.F.shape, generator=g, dtype=torch.float64)
    y.F.backward(dy.float().cuda()); yo.F.backward(dy)
    assert max_rel_err(y.F, yo.F) < 1e-5 and max_rel_err(xg.grad, xo.grad) < 1e-5


def test_global_pooling_broadcast_and_instance_norm():
    """Per-instance ops of `downstream/semseg/lib/layers.py:12-90` / `model/modules/common.py:22-23` against plain torch per batch index."""
    from pointcontrast_b200 import me
    rng = np.random.default_rng(2)
    coords = surface_coords(rng, 3000, batches=3)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(len(coords), 16, generator=g, dtype=torch.float64)
    b = torch.from_numpy(coords[:, 0]).long()
    st = me.SparseTensor(x.float().cuda(), coords=torch.from_numpy(coords))
    glob = me.MinkowskiGlobalPooling(dimension=3)(st)
    ref = torch.stack([x[b == i].mean(0) for i in range(3)])
    assert max_rel_err(glob.F, ref) < 1e-5
    added = me.MinkowskiBroadcastAddition(dimension=3)(st, glob)
    assert max_rel_err(added.F, x + ref[b]) < 1e-5
    mul = me.MinkowskiBroadcastMultiplication(dimension=3)(st, glob)
    assert max_rel_err(mul.F, x * ref[b]) < 1e-5
    inorm = me.MinkowskiInstanceNorm(16, D=3).cuda()
    y = inorm(st).F
    refn = torch.empty_like(x)
    for i in range(3):
        xi = x[b == i]
        refn[b == i] = (xi - xi.mean(0)) / torch.sqrt(xi.var(0, unbiased=False) + 1e-6)
    assert max_rel_err(y, refn) < 1e-4


def _host_tile_image(w, fp16):
    """Host restatement of a weight-tile image of the split conv kernel, as int16 words.  w: fp32 [K][Kc][N] (contraction channels x
    tile columns: [K][Cin][Cout] for the forward roles, [K][Cout][Cin] for the data-gradient roles)."""
    w = w.contiguous()
    K, Kc, N = w.shape
    bn = next(b for b in (128, 96, 64, 32) if N % b == 0)
    plane = 4 * ((bn // 8) * 128 + 16)
    k, c, n = np.meshgrid(np.arange(K), np.arange(Kc), np.arange(N), indexing="ij")
    blob = ((k * (Kc // 32) + c // 32) * (N // bn) + n // bn) * 2 * plane
    off = blob + (c % 32 // 8) * (plane // 4) + (n % bn // 8) * 128 + (n % 8) * 16 + (c % 8) * 2
    v, dt = ((w * 1024.0).clamp(-65000.0, 65000.0), torch.float16) if fp16 else (w, torch.bfloat16)
    hi = v.to(dt)
    lo = (v - hi.float()).to(dt)
    img = np.zeros(K * (Kc // 32) * (N // bn) * plane, np.int16)        # 2 * plane bytes per blob; the 16-byte pads stay zero
    img[off // 2] = hi.view(torch.int16).numpy()
    img[(off + plane) // 2] = lo.view(torch.int16).numpy()
    return img


@pytest.mark.parametrize("fp16", [False, True])
def test_weight_tiling_matches_host_layout(fp16):
    """`pcb_weight_tile` (one convolution) and `pcb_weight_tile_batch` (all convolutions of a network in one launch) write bit for bit the
    tile images restated on the host: forward roles (fp16 hi/lo of W * 2^10, or bf16 hi/lo) and data-gradient roles (bf16 hi/lo)."""
    import ctypes
    from pointcontrast_b200._lib import PcbTileDesc, check, lib, ptr, stream
    g = torch.Generator().manual_seed(3)
    shapes = [(27, 96, 96), (8, 32, 64), (1, 128, 256), (27, 384, 256), (27, 32, 32)]
    Ws = [torch.randn(K, ci, co, generator=g) * (0.3 if i else 1e-3) for i, (K, ci, co) in enumerate(shapes)]
    Wd = [W.cuda() for W in Ws]
    flag = 16 if fp16 else 0
    descs = (PcbTileDesc * len(shapes))()
    single, batch, start = [], [], 0
    for i, (W, (K, ci, co)) in enumerate(zip(Wd, shapes)):
        f, d, fb, db = (torch.zeros(lib.pcb_weight_tile_bytes(K, ci, co, r), dtype=torch.uint8, device="cuda") for r in (0, 1, 0, 1))
        check(lib.pcb_weight_tile(ptr(W), K, ci, co, ptr(f), ptr(d), flag, stream()))
        check(lib.pcb_tile_desc_fill(ctypes.byref(descs[i]), ptr(W), K, ci, co, ptr(fb), ptr(db), flag, start))
        start += K * ci * co
        single.append((f, d))
        batch.append((fb, db))
    dev = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    check(lib.pcb_weight_tile_batch(dev.data_ptr(), len(shapes), start, stream()))
    torch.cuda.synchronize()
    for W, sh, s, b in zip(Ws, shapes, single, batch):
        want = (_host_tile_image(W, fp16), _host_tile_image(W.transpose(1, 2), False))
        for role, ref in zip(("forward", "data-gradient"), want):
            for entry, out in (("pcb_weight_tile", s), ("pcb_weight_tile_batch", b)):
                got = out[role != "forward"].cpu().numpy().view(np.int16)
                assert got.shape == ref.shape and np.array_equal(got, ref), (sh, entry, role, int((got != ref).sum()), ref.size)
