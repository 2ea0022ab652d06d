"""The fused training unit (`pcb_unit_forward` / `pcb_unit_backward`, csrc/unit.cu) at every signature the executor issues
(tests/exact_unit.py), held to fp64 bit for bit on exactly representable operands, and to its primitives bit for bit on the operands
the forward pass writes.

  * Backward: dz (both bf16 planes, or the stem's fp32 dz), dW in both weight-gradient orientations, gin through the opposite-offset
    table written and accumulated, gres written and accumulated, dgamma / dbeta on a nonzero base -- against an fp64 reference
    written from the math, on the real tables of a coordinate-manager scene at an offset-split and a direct-mode size.
  * Forward: z against fp64; mean, invstd, the running statistics, out_p and every plane bit-identical to `pcb_bn_stats_seg` and
    `pcb_bn_apply_seg` on the unit's own z; eval mode leaves the running statistics alone.
  * Forward then backward against the same steps issued as primitive calls.
  * Every signature the fused executor issues for Res16UNet14/18/34/34C is in the case matrix.
  * A rejected struct leaves every output as it was.
Operands are framed by NaN (inputs) and sentinels (outputs); the workspace is NaN-poisoned.
"""
import ctypes

import numpy as np
import pytest
import torch

from pointcontrast_b200._lib import CONV_ACCUMULATE, ERR_ARG, PLANES_B_FP16, UNIT_EVAL, UNIT_FP16_FORWARD
from tests import exact_bn as XB
from tests import exact_conv as XC
from tests import exact_unit as XU
from tests.helpers import surface_coords
from tests.test_gpu_conv_exact import _assert_exact, _gather, _kmap_arg, _ref_forward, _ws

pytestmark = pytest.mark.gpu
SENT = -7777.25
SENT16 = 0x5A5A


def _L():
    from pointcontrast_b200 import _lib
    return _lib


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope="module")
def plans():
    """ConvPlans of two coordinate-manager scenes, as tests/test_gpu_conv_exact.py builds them: "split" (every tensor-core shape with
    more than one offset-chunk runs offset-split) and "direct" (at least one CTA per SM for every width the models give each kind)."""
    from pointcontrast_b200 import me
    out = {}
    for size, npts, extent in (("split", 1500, 40), ("direct", 90_000, 70)):
        coords = surface_coords(np.random.default_rng(5), npts, extent=extent)
        st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
        cm, fine = st.coords_man, st.coords_key
        coarse = cm.stride(fine, [2, 2, 2])
        hyb = me.KernelGenerator(3, 1, 1, region_type=me.RegionType.HYBRID, axis_types=[me.RegionType.HYPERCUBE] * 3, dimension=3)
        k8 = me.KernelGenerator([2, 2, 2], 2, 1, dimension=3)
        p27 = cm.conv_plan(fine, fine, hyb, False)
        out[size] = dict(k27=p27, stem=p27, down=cm.conv_plan(fine, coarse, k8, False), up=cm.conv_plan(coarse, fine, k8, True),
                         k1=cm.conv_plan(fine, fine, me.KernelGenerator(1, 1, 1, dimension=3), False))
    return out


def _mode(sig, plan):
    return "direct" if XC.conv_splits(plan.K, plan.n_out, sig.Cin, sig.Cout, _sms()) == 1 else "split"


# ----------------------------------------------------------------------------------------------- one unit's buffers
class _Case:
    """Every buffer of one unit of signature `sig` on `plan`, each a slice of a framed tensor, and the struct pointing at them."""

    def __init__(self, sig, plan, seed):
        L = _L()
        self.sig, self.plan = sig, plan
        self.K, Cin, Cout = plan.K, sig.Cin, sig.Cout
        self.n_in, self.n_out = plan.n_in, plan.n_out
        self.n0 = XU.view_split(self.n_out) if sig.two_views else self.n_out
        self.gen = torch.Generator(device="cuda").manual_seed(seed)
        self.b = {}
        u = self.u = L.PcbUnit()
        u.n_in, u.n_out, u.n0, u.K, u.Cin, u.Cout, u.relu = self.n_in, self.n_out, self.n0, self.K, Cin, Cout, int(sig.relu)
        u.fwd_tbl, u.fwd_stride = plan.fwd_tbl.data_ptr(), plan.fwd_tbl.shape[1]
        u.fwd_kmap = ctypes.cast(plan.c_kmap("fwd_kmap"), ctypes.c_void_p) if plan.fwd_kmap is not None else None
        u.dg_tbl, u.dg_stride = plan.dg_tbl.data_ptr(), plan.dg_tbl.shape[1]
        u.dg_kmap = ctypes.cast(plan.c_kmap("dg_kmap"), ctypes.c_void_p) if plan.dg_kmap is not None else None
        u.wg_tbl, u.wg_stride, u.wg_gather_x = plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], int(plan.wg_gather_x)
        f32, i16 = torch.float32, torch.int16
        if sig.tc:
            planes = ("x_hi", "x_lo", "x_bhi", "x_blo") if sig.fp16 else ("x_hi", "x_lo")
            for k in planes:
                u.x_lds = self._buf(k, self.n_in, Cin, sig.x_str, i16, -1)
            u.dz_ld = self._buf("dz_hi", self.n_out, Cout, True, i16, SENT16, extra=8)
            self._buf("dz_lo", self.n_out, Cout, True, i16, SENT16, extra=8)
        else:
            u.x_ld = self._buf("x_p", self.n_in, Cin, sig.x_str, f32, float("nan"))
            u.dz_ld = self._buf("dz_p", self.n_out, Cout, True, f32, SENT, extra=8)
        u.z_ld = self._buf("z_p", self.n_out, Cout, False, f32, SENT)
        planes = ("out_hi", "out_lo", "out_bhi", "out_blo") if sig.fp16 and not sig.eval else ("out_hi", "out_lo")
        for k in planes:
            u.out_lds = self._buf(k, self.n_out, Cout, sig.out_str, i16, SENT16)
        if sig.out_p:
            u.out_ld = self._buf("out_p", self.n_out, Cout, False, f32, SENT)
        if sig.res:
            u.res_ld = self._buf("res_p", self.n_out, Cout, False, f32, float("nan"))
        u.g_ld = self._buf("g_p", self.n_out, Cout, sig.g_str, f32, float("nan"))
        if sig.gin_mode:
            u.gin_ld = self._buf("gin_p", self.n_in, Cin, sig.gin_str, f32, SENT)
        u.gin_mode = sig.gin_mode
        if sig.gres_mode:
            u.gres_ld = self._buf("gres_p", self.n_out, Cout, sig.gres_str, f32, SENT)
        u.gres_mode = sig.gres_mode
        for k, C in (("mean", 2 * Cout), ("invstd", 2 * Cout), ("gamma", Cout), ("beta", Cout), ("running_mean", Cout), ("running_var", Cout),
                     ("dgamma", Cout), ("dbeta", Cout), ("dW", self.K * Cin * Cout)):
            self._vec(k, C)
        u.eps, u.momentum = XB.EPS, XB.MOMENTUM
        self.W = XC.weights(self.K, Cin, Cout, XC.FP16 if sig.fp16 else XC.BF16, self.gen, "cuda")[0]
        u.W = self.W.data_ptr()
        self.tiles()
        wsb = L.lib.pcb_unit_ws_bytes(self.K, self.n_in, self.n_out, Cin, Cout)
        self.ws = _ws(wsb)
        u.ws, u.ws_bytes = self.ws.data_ptr(), wsb
        u.flags = (UNIT_FP16_FORWARD if sig.fp16 else 0) | (UNIT_EVAL if sig.eval else 0)

    def _buf(self, name, n, C, strided, dtype, fill, c0=8, extra=16):
        """[n + 1, ld] framed by `fill`; the operand is columns [c0, c0 + C) of the first n rows.  Sets the struct's pointer."""
        c0, ld = (c0, c0 + C + extra) if strided else (0, C)
        t = torch.full((n + 1, ld), fill, dtype=dtype, device="cuda")
        self.b[name] = (t, c0, n, C)
        setattr(self.u, name, t.data_ptr() + t.element_size() * c0)
        return ld

    def _vec(self, name, C, pad=8):
        t = torch.full((C + 2 * pad,), SENT, device="cuda")
        self.b[name] = (t, pad, 1, C)
        setattr(self.u, name, t.data_ptr() + 4 * pad)

    def tiles(self):
        L = _L()
        K, Cin, Cout = self.K, self.sig.Cin, self.sig.Cout
        if not self.sig.tc:
            return
        self.ft = torch.empty(L.lib.pcb_weight_tile_bytes(K, Cin, Cout, 0), dtype=torch.uint8, device="cuda")
        self.dt = torch.empty(L.lib.pcb_weight_tile_bytes(K, Cin, Cout, 1), dtype=torch.uint8, device="cuda")
        L.check(L.lib.pcb_weight_tile(self.W.data_ptr(), K, Cin, Cout, self.ft.data_ptr(), self.dt.data_ptr(), PLANES_B_FP16 if self.sig.fp16 else 0,
                                      L.stream()))
        self.u.wt_fwd, self.u.wt_dg = self.ft.data_ptr(), self.dt.data_ptr()

    def view(self, name):
        t, c0, n, C = self.b[name]
        return t[c0:c0 + C] if t.dim() == 1 else t[:n, c0:c0 + C]

    def set(self, name, v):
        dst = self.view(name)
        if dst.dtype == torch.int16 and v.dtype != torch.int16:
            v = v.to(torch.bfloat16 if name in ("x_bhi", "x_blo", "dz_hi", "dz_lo") or not self.sig.fp16 else torch.float16).view(torch.int16)
        dst.copy_(v.reshape(dst.shape))

    def value(self, name, fmt="bf16"):
        v = self.view(name)
        return v.view(torch.bfloat16 if fmt == "bf16" else torch.float16).double() if v.dtype == torch.int16 else v.double()

    def snapshot(self):
        return {k: t.clone() for k, (t, _, _, _) in self.b.items()}

    def assert_frames(self, names, what):
        """Every element outside each output's slice still holds what the frame was filled with."""
        for k in names:
            t, c0, n, C = self.b[k]
            f = t.clone()
            if t.dim() == 1:
                f[c0:c0 + C] = f[0]
            else:
                f[:n, c0:c0 + C] = f[n, 0]
            assert bool((f.view(torch.int32 if f.element_size() == 4 else torch.int16) ==
                         f.view(torch.int32 if f.element_size() == 4 else torch.int16).flatten()[0]).all()), f"{what}: frame of {k} overwritten"

    # -------------------------------------------------------------------------------------------- operands
    def forward_operands(self):
        """x (exact_conv's forward rule in the forward format, plus its bf16 planes under fp16 forward), gamma / beta on the exact_bn
        apply grid, running statistics, residual.  -> fp64 (hi, lo) of x as the forward reads it"""
        sig, g = self.sig, self.gen
        C = sig.Cout
        self.set("gamma", torch.tensor(XB.GAMMA, device="cuda")[torch.randint(0, 5, (C,), generator=g, device="cuda")])
        self.set("beta", torch.randint(-8, 9, (C,), generator=g, device="cuda") / 8.0)
        self.set("running_mean", torch.randint(-64, 65, (C,), generator=g, device="cuda") / 8.0)
        self.set("running_var", torch.randint(1, 65, (C,), generator=g, device="cuda") / 8.0)
        if sig.res:
            self.set("res_p", torch.randint(-16, 17, (self.n_out, C), generator=g, device="cuda") / 8.0)
        if not sig.tc:
            hi, lo = XC.dense_planes(self.n_in, sig.Cin, 0.7, XC.BF16.HI, XC.BF16.LO, g, "cuda")
            self.set("x_p", hi + lo)
            self.W.copy_(XC.weights(self.K, sig.Cin, sig.Cout, XC.BF16, g, "cuda")[1])      # integers: exact_conv's fp32 rule
            return (hi + lo).double(), None
        fmt = XC.FP16 if sig.fp16 else XC.BF16
        hi, lo = XC.capped_planes(self.n_in, sig.Cin, XC.row_cap(fmt, self.K, sig.Cin), fmt.HI, fmt.LO, g, "cuda")
        self.set("x_hi", hi)
        self.set("x_lo", lo)
        if sig.fp16:
            x = hi + lo
            bh = x.to(torch.bfloat16).float()
            self.set("x_bhi", bh)
            self.set("x_blo", x - bh)
        return hi.double(), lo.double()

    def z_reference(self, xh, xl):
        sig, plan = self.sig, self.plan
        if not sig.tc:
            want = torch.zeros(self.n_out, sig.Cout, dtype=torch.float64, device="cuda")
            for k in range(self.K):
                want += _gather(xh.double(), plan.fwd_tbl[k, :self.n_out]) @ self.W[k].double()
            return want
        fmt = XC.FP16 if sig.fp16 else XC.BF16
        wh, wl = XC.split_weights(self.W, fmt)
        y, a = _ref_forward(xh, xl, wh.double(), wl.double(), plan.fwd_tbl, plan.fwd_kmap, self.n_out)
        assert float(a.max()) * fmt.SCALE < XC.LIMIT * fmt.Q
        return y * fmt.SCALE

    def forward(self):
        L = _L()
        L.check(L.lib.pcb_unit_forward(ctypes.byref(self.u), L.stream()))
        torch.cuda.synchronize()

    def backward(self, u=None):
        L = _L()
        L.check(L.lib.pcb_unit_backward(ctypes.byref(u or self.u), L.stream()))
        torch.cuda.synchronize()


def _assert_bits(got, want, what):
    got, want = got.contiguous(), want.contiguous()
    iv = torch.int32 if got.element_size() == 4 else torch.int16
    bad = got.view(iv) != want.view(iv)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} differ; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {want[tuple(i)].item()!r}")


def _cases():
    return XU.training_cases()


def _ids(cases):
    return [s.name() for s in cases]


# ----------------------------------------------------------------------------------------------- a. backward against fp64
def _paired_backward(case):
    """Paired operands into the case's buffers.  -> expected dz (fp64, h and l planes), the masked g, the x values the weight
    gradient reads (hi, lo fp64; fp32 rows for the stem)"""
    sig, g = case.sig, case.gen
    K, Cin, Cout = case.K, sig.Cin, sig.Cout
    row_cap, col_cap = XU.backward_caps(sig, K)
    p = XU.paired_backward(case.n_out, case.n0, Cout, row_cap, col_cap, not sig.tc, "fp16" if sig.fp16 else "bf16",
                           seed=XB.seed_of(str(sig.name())), device="cuda")
    assert XU.bn_sum_terms(p, case.n0) < XU.BN_LIMIT
    for k in ("z", "g"):
        case.set(k + "_p", p[k])
    case.set("mean", p["mean"])
    case.set("invstd", p["invstd"])
    case.set("gamma", p["gamma"])
    case.set("out_hi", p["codes"])
    if sig.fp16:
        case.set("out_bhi", p["bcodes"])
    case.set("dgamma", p["dgamma_base"])
    case.set("dbeta", p["dbeta_base"])
    if sig.gres_mode == 2:
        case.set("gres_p", p["gres_base"])
    if sig.gin_mode == 2:
        case.set("gin_p", XC.bias_values(case.n_in * Cin, XC.BF16, g, "cuda").view(case.n_in, Cin))
    case.set("dW", XC.bias_values(K * Cin * Cout, XC.BF16, g, "cuda"))
    case.W.copy_(XC.weights(K, Cin, Cout, XC.BF16, g, "cuda")[0])
    case.tiles()
    ok = XB.mask_passes(p["codes"]) if sig.relu else torch.ones_like(p["g"], dtype=torch.bool)
    h, l = torch.where(ok, p["h"], 0.0).double(), torch.where(ok, p["l"], 0.0).double()
    gm = torch.where(ok, p["g"], 0.0).double()
    if not sig.tc:
        hi, lo = XC.dense_planes(case.n_in, Cin, 0.7, XC.BF16.HI, XC.BF16.LO, g, "cuda")
        case.set("x_p", hi + lo)
        return h, l, gm, ((hi + lo).double(), None)
    if case.plan.wg_gather_x:
        xh, xl = XC.dense_planes(case.n_in, Cin, XC.WG_A_DENSITY, XC.BF16.HI, XC.BF16.LO, g, "cuda")
    else:
        xh, xl = (t.t() for t in XC.capped_planes(Cin, case.n_in, min(case.n_in, XC.wgrad_col_cap()), XC.BF16.HI, XC.BF16.LO, g, "cuda"))
    if sig.fp16:                       # x_hi / x_lo: the fp16 planes of the same rows (what the forward read); the weight gradient must not
        case.set("x_bhi", xh)
        case.set("x_blo", xl)
        x = xh + xl
        fh = x.half().float()
        case.set("x_hi", fh)
        case.set("x_lo", x - fh)
    else:
        case.set("x_hi", xh)
        case.set("x_lo", xl)
    return h, l, gm, (xh.double(), xl.double())


def _check_backward(case, h, l, gm, x, base, what):
    """dz, dW, gin, gres, dgamma / dbeta against fp64; `base`: the snapshot taken before the call"""
    sig, plan = case.sig, case.plan
    K, Cin, Cout = case.K, sig.Cin, sig.Cout
    if sig.tc:
        _assert_exact(case.value("dz_hi"), h, what + " dz_hi")
        _assert_exact(case.value("dz_lo"), l, what + " dz_lo")
    else:
        _assert_exact(case.value("dz_p"), h, what + " dz_p")
    for k in ("dgamma", "dbeta"):
        t, c0, _, C = case.b[k]
        _assert_bits(case.view(k), base[k][c0:c0 + C], what + " " + k)
    if sig.gres_mode:
        t, c0, n, C = case.b["gres_p"]
        want = gm + (base["gres_p"][:n, c0:c0 + C].double() if sig.gres_mode == 2 else 0)
        _assert_exact(case.value("gres_p"), want, what + " gres")
    # dW[k] = sum over table pairs of x[in]^T dz[out]
    t, c0, _, nW = case.b["dW"]
    want = base["dW"][c0:c0 + nW].double().view(K, Cin, Cout).clone()
    bound = want.abs()
    xh, xl = x
    rows = case.n_out if plan.wg_gather_x else case.n_in
    for k in range(K):
        tb = plan.wg_tbl[k, :rows]
        if not sig.tc:
            gx = _gather(xh, tb)
            want[k] += gx.t() @ h
            bound[k] += gx.abs().t() @ h.abs()
        elif plan.wg_gather_x:
            gh, gl = _gather(xh, tb), _gather(xl, tb)
            want[k] += gl.t() @ h + gh.t() @ l + gh.t() @ h
            bound[k] += gl.abs().t() @ h.abs() + gh.abs().t() @ l.abs() + gh.abs().t() @ h.abs()
        else:
            gh, gl = _gather(h, tb), _gather(l, tb)
            want[k] += (gl.t() @ xh + gh.t() @ xl + gh.t() @ xh).t()
            bound[k] += (gl.abs().t() @ xh.abs() + gh.abs().t() @ xl.abs() + gh.abs().t() @ xh.abs()).t()
    q = XC.EXACT_Q if not sig.tc else XC.WG_Q
    assert float(bound.max()) < XC.LIMIT * q, (what, "dW operands leave the exact range", float(bound.max()))
    _assert_exact(case.view("dW").view(K, Cin, Cout), want, what + " dW")
    if sig.gin_mode:
        wh, wl = XC.split_weights(case.W, XC.BF16)
        y, a = _ref_forward(h, l, wh.double().transpose(1, 2), wl.double().transpose(1, 2), plan.dg_tbl, plan.dg_kmap, case.n_in)
        t, c0, n, C = case.b["gin_p"]
        if sig.gin_mode == 2:
            b0 = base["gin_p"][:n, c0:c0 + C].double()
            y, a = y + b0, a + b0.abs()
        assert float(a.max()) < XC.LIMIT * XC.BF16.Q, (what, "gin operands leave the exact range")
        _assert_exact(case.value("gin_p"), y, what + " gin")
    outs = ["dgamma", "dbeta", "dW"] + (["dz_hi", "dz_lo"] if sig.tc else ["dz_p"]) + ["gin_p"] * (sig.gin_mode > 0) + ["gres_p"] * (sig.gres_mode > 0)
    case.assert_frames(outs, what)


def _unpaired_backward(case, what):
    """exact_bn's operands: dgamma, dbeta and gres exact, summed over both views."""
    sig = case.sig
    n, n0, C = case.n_out, case.n0, sig.Cout
    z, dy, mean, invstd, gamma_, bg, bb, gb = (t.cuda() for t in XU.unpaired_backward(n0, n - n0, C, XB.seed_of(str(what))))
    for k, v in (("z_p", z), ("g_p", dy), ("mean", mean), ("invstd", invstd), ("gamma", gamma_), ("dgamma", bg), ("dbeta", bb)):
        case.set(k, v)
    if sig.gres_mode:
        case.set("gres_p", gb)
    t, c0, _, _ = case.b["out_hi"]
    codes = case.view("out_hi").clone()
    ok = XB.mask_passes(codes) if sig.relu else torch.ones(n, C, dtype=torch.bool, device="cuda")
    case.backward()
    view = (torch.arange(n, device="cuda") >= n0).long()
    xhat = (z.double() - mean.double()[view]) * invstd.double()[view]
    gm = torch.where(ok, dy.double(), 0.0)
    _assert_exact(case.value("dbeta"), bb.double() + gm.sum(0), what + " unpaired dbeta")
    _assert_exact(case.value("dgamma"), bg.double() + (gm * xhat).sum(0), what + " unpaired dgamma")
    if sig.gres_mode:
        _assert_exact(case.value("gres_p"), gm + (gb.double() if sig.gres_mode == 2 else 0), what + " unpaired gres")


@pytest.mark.parametrize("sig", _cases(), ids=_ids(_cases()))
def test_unit_backward_bit_exact(plans, sig):
    """Paired operands at the offset-split and the direct-mode scene size: every backward output against fp64, frames intact; then
    one unpaired call for dgamma, dbeta and gres."""
    for size in ("split", "direct"):
        plan = plans[size][sig.kind]
        case = _Case(sig, plan, seed=XB.seed_of(f"{sig.name()} {size}"))
        what = f"{sig.name()} {size} n_in={case.n_in} n_out={case.n_out} n0={case.n0}"
        h, l, gm, x = _paired_backward(case)
        base = case.snapshot()
        case.backward()
        _check_backward(case, h, l, gm, x, base, what)
        if size == "split":
            _unpaired_backward(case, what)


# ----------------------------------------------------------------------------------------------- b. forward
def _bn_primitives(case, z, stats=None):
    """pcb_bn_stats_seg (unless `stats` = (mean, invstd) is given) and pcb_bn_apply_seg on z, into fresh copies of the case's
    buffers.  -> dict of outputs"""
    L = _L()
    sig, u = case.sig, case.u
    n, n0, C = case.n_out, case.n0, sig.Cout
    o = {k: case.view(k).clone() for k in ("running_mean", "running_var")}
    if stats is None:
        init = case.initial
        o["running_mean"], o["running_var"] = init["running_mean"].clone(), init["running_var"].clone()
        o["mean"], o["invstd"] = torch.full((2 * C,), SENT, device="cuda"), torch.full((2 * C,), SENT, device="cuda")
        wsb = L.lib.pcb_bn_ws_bytes(n, C)
        ws = _ws(wsb)
        L.check(L.lib.pcb_bn_stats_seg(z.data_ptr(), C, n, n0, C, XB.EPS, XB.MOMENTUM, o["mean"].data_ptr(), o["invstd"].data_ptr(),
                                       o["running_mean"].data_ptr(), o["running_var"].data_ptr(), ws.data_ptr(), wsb, L.stream()))
    else:
        o["mean"], o["invstd"] = stats
    ld = case.b["out_hi"][0].shape[1]
    planes = ("out_hi", "out_lo", "out_bhi", "out_blo") if "out_bhi" in case.b else ("out_hi", "out_lo")
    for k in planes:
        o[k] = torch.full((n, ld), SENT16, dtype=torch.int16, device="cuda")
    if sig.out_p:
        o["out_p"] = torch.full((n, C), SENT, device="cuda")
    res = case.view("res_p") if sig.res else None
    c0 = case.b["out_hi"][1]
    pl = lambda k: o[k].data_ptr() + 2 * c0 if k in o else None
    L.check(L.lib.pcb_bn_apply_seg(z.data_ptr(), C, n, n0, C, o["mean"].data_ptr(), o["invstd"].data_ptr(), u.gamma, u.beta,
                                   res.data_ptr() if res is not None else None, res.stride(0) if res is not None else 0,
                                   (1 if sig.relu else 0) | (8 if sig.fp16 else 0), o["out_p"].data_ptr() if sig.out_p else None, C,
                                   pl("out_hi"), pl("out_lo"), ld, pl("out_bhi"), pl("out_blo"), L.stream()))
    torch.cuda.synchronize()
    for k in planes:
        o[k] = o[k][:, c0:c0 + C]
    return o


def _check_forward(case, what):
    xh, xl = case.forward_operands()
    case.initial = {k: case.view(k).clone() for k in ("running_mean", "running_var")}
    case.forward()
    sig = case.sig
    z = case.view("z_p")
    _assert_exact(z, case.z_reference(xh, xl), what + " z")
    nseg = 2 if case.n0 < case.n_out else 1
    C = sig.Cout
    if sig.eval:
        for k in ("running_mean", "running_var"):
            _assert_bits(case.view(k), case.initial[k], what + f" eval leaves {k} untouched")
        _assert_bits(case.view("mean")[:C], case.initial["running_mean"], what + " eval mean")
        rv = case.initial["running_var"].cpu().numpy()
        want = (np.float32(1.0) / np.sqrt(rv + np.float32(XB.EPS))).astype(np.float32)
        _assert_bits(case.view("invstd")[:C].cpu(), torch.from_numpy(want), what + " eval invstd")
        ref = _bn_primitives(case, z.contiguous(), (case.view("mean").clone(), case.view("invstd").clone()))
    else:
        ref = _bn_primitives(case, z.contiguous())
        for k in ("mean", "invstd"):
            _assert_bits(case.view(k)[:nseg * C], ref[k][:nseg * C], what + " " + k)
        for k in ("running_mean", "running_var"):
            _assert_bits(case.view(k), ref[k], what + " " + k)
    for k in ("out_hi", "out_lo", "out_bhi", "out_blo", "out_p"):
        if k in case.b:
            _assert_bits(case.view(k), ref[k], what + " " + k)
    outs = ["z_p", "mean", "invstd", "running_mean", "running_var", "out_hi", "out_lo"] + [k for k in ("out_bhi", "out_blo", "out_p") if k in case.b]
    case.assert_frames(outs, what)
    assert bool((case.b["mean"][0][8 + nseg * C:] == SENT).all()), what + " mean of a view that does not exist written"


_FWD = XU.signatures()


@pytest.mark.parametrize("sig", _FWD, ids=_ids(_FWD))
def test_unit_forward_bit_exact(plans, sig):
    """z against fp64 at both scene sizes; the statistics (fused into the offset-split reduction or a separate pass, or eval's running
    statistics), out_p and every plane bit-identical to the BatchNorm primitives on the unit's own z."""
    for size in ("split", "direct"):
        plan = plans[size][sig.kind]
        case = _Case(sig, plan, seed=XB.seed_of(f"{sig.name()} {size} fwd"))
        if sig.tc:                # one offset-chunk (K = 1, Cin = 32) has nothing to split
            assert _mode(sig, plan) == size or (size == "split" and plan.K * (sig.Cin // XC.BK) < 2), (sig.name(), size, case.n_out)
        _check_forward(case, f"{sig.name()} {size} ({_mode(sig, plan)}) n_out={case.n_out} n0={case.n0}")


# ----------------------------------------------------------------------------------------------- c. forward then backward
@pytest.mark.parametrize("sig", _cases(), ids=_ids(_cases()))
def test_unit_chain_matches_primitives(plans, sig):
    """The backward consumes what the forward wrote; every output is bit-identical to pcb_bn_backward_seg, then the weight gradient
    (pcb_conv_wgrad_split in the executor's orientation, or pcb_conv_wgrad for the stem), then pcb_conv_forward_split on the
    data-gradient tiles, issued one by one into copies of the same buffers."""
    L = _L()
    plan = plans["split"][sig.kind]
    case = _Case(sig, plan, seed=XB.seed_of(f"{sig.name()} chain"))
    case.forward_operands()
    case.forward()
    g = case.gen
    K, Cin, Cout, n, n_in = case.K, sig.Cin, sig.Cout, case.n_out, case.n_in
    case.set("g_p", torch.randint(-8, 9, (n, Cout), generator=g, device="cuda") / 4.0)
    case.set("dgamma", torch.randn(Cout, generator=g, device="cuda"))
    case.set("dbeta", torch.randn(Cout, generator=g, device="cuda"))
    case.set("dW", torch.randn(K * Cin * Cout, generator=g, device="cuda"))
    if sig.gin_mode == 2:
        case.set("gin_p", torch.randn(n_in, Cin, generator=g, device="cuda"))
    if sig.gres_mode == 2:
        case.set("gres_p", torch.randn(n, Cout, generator=g, device="cuda"))
    prim = case.snapshot()
    case.backward()
    u = case.u
    P = lambda k: prim[k].data_ptr() + prim[k].element_size() * case.b[k][1]
    ld = lambda k: prim[k].shape[1]
    wsb = max(L.lib.pcb_bn_ws_bytes(n, Cout), L.lib.pcb_unit_ws_bytes(K, n_in, n, Cin, Cout))
    ws = _ws(wsb)
    st = L.stream()
    tc = sig.tc
    mask = P("out_hi") if sig.relu else None
    L.check(L.lib.pcb_bn_backward_seg(u.g_p, u.g_ld, u.z_p, u.z_ld, mask, u.out_lds, n, case.n0, Cout, u.mean, u.invstd, u.gamma,
                                      None if tc else P("dz_p"), u.dz_ld, P("dgamma"), P("dbeta"), 1,
                                      P("gres_p") if sig.gres_mode else None, u.gres_ld, sig.gres_mode,
                                      P("dz_hi") if tc else None, P("dz_lo") if tc else None, u.dz_ld, ws.data_ptr(), wsb, st))
    if tc:
        xh, xl = (P("x_bhi"), P("x_blo")) if sig.fp16 else (P("x_hi"), P("x_lo"))
        if plan.wg_gather_x:
            args = (xh, xl, u.x_lds, P("dz_hi"), P("dz_lo"), u.dz_ld, plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], K, n, Cin, Cout, P("dW"), 0)
        else:
            args = (P("dz_hi"), P("dz_lo"), u.dz_ld, xh, xl, u.x_lds, plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], K, n_in, Cout, Cin, P("dW"), 1)
        L.check(L.lib.pcb_conv_wgrad_split(*args, ws.data_ptr(), wsb, 4, st))
    else:
        L.check(L.lib.pcb_conv_wgrad(P("x_p"), u.x_ld, P("dz_p"), u.dz_ld, plan.wg_tbl.data_ptr(), plan.wg_tbl.shape[1], K, n, Cin, Cout,
                                     P("dW"), 0, ws.data_ptr(), wsb, 4, st))
    if sig.gin_mode:
        L.check(L.lib.pcb_conv_forward_split(P("dz_hi"), P("dz_lo"), u.dz_ld, plan.dg_tbl.data_ptr(), plan.dg_tbl.shape[1],
                                             _kmap_arg(plan.dg_kmap), K, n_in, Cout, Cin, case.dt.data_ptr(), None, P("gin_p"), u.gin_ld,
                                             ws.data_ptr(), wsb, CONV_ACCUMULATE if sig.gin_mode == 2 else 0, st))
    torch.cuda.synchronize()
    what = sig.name() + " chained"
    for k in ["dgamma", "dbeta", "dW"] + (["dz_hi", "dz_lo"] if tc else ["dz_p"]) + ["gin_p"] * (sig.gin_mode > 0) + ["gres_p"] * (sig.gres_mode > 0):
        _assert_bits(case.b[k][0], prim[k], f"{what}: {k}")
    assert bool(torch.isfinite(case.view("dW")).all()), what


def test_residual_gradient_written_then_accumulated(plans):
    """A BasicBlock's pattern: its second unit writes the residual gradient (gres_mode 1), then its first unit, whose input is that
    residual, accumulates its data gradient into the same buffer (gin_mode 2).  The buffer ends as masked g of the second unit plus the
    fp64 data gradient of the first."""
    plan = plans["split"]["k27"]
    sig2 = XU.Sig("k27", 27, 32, 32, True, True, False, 1, 1, False, False, True, False, False, False, False, False)
    sig1 = sig2._replace(res=False, gres_mode=0, gin_mode=2)
    second, first = _Case(sig2, plan, seed=21), _Case(sig1, plan, seed=22)
    _, _, gm2, _ = _paired_backward(second)
    second.backward()
    h, l, _, _ = _paired_backward(first)
    R = second.b["gres_p"][0]
    first.b["gin_p"] = (R, second.b["gres_p"][1], second.n_out, 32)
    first.u.gin_p, first.u.gin_ld = second.u.gres_p, second.u.gres_ld
    first.backward()
    wh, wl = XC.split_weights(first.W, XC.BF16)
    y, a = _ref_forward(h, l, wh.double().transpose(1, 2), wl.double().transpose(1, 2), plan.dg_tbl, plan.dg_kmap, first.n_in)
    assert float((a + gm2.abs()).max()) < XC.LIMIT * XC.BF16.Q
    _assert_exact(first.value("gin_p"), gm2 + y, "gres written, then gin accumulated")
    first.assert_frames(["gin_p"], "gres then gin")


# ----------------------------------------------------------------------------------------------- d. reach
class _Recorder:
    """fused.lib with pcb_unit_forward / pcb_unit_backward recording the signature of every struct they are given."""

    def __init__(self, lib):
        self._lib, self.fwd, self.bwd = lib, [], []

    def __getattr__(self, k):
        return getattr(self._lib, k)

    @staticmethod
    def sig(u, backward):
        tc = u.Cin % 32 == 0 and u.Cout % 32 == 0
        if not tc:
            kind = "stem"
        elif u.K in (27, 1):
            kind = {27: "k27", 1: "k1"}[u.K]
        elif backward:
            kind = "down" if u.wg_gather_x else "up"
        else:
            kind = "down" if u.n_out < u.n_in else "up"
        s = XU.Sig(kind, u.K, u.Cin, u.Cout, bool(u.relu), bool(u.res_p), bool(u.out_p), u.gres_mode if backward else 0,
                   u.gin_mode if backward else 0, bool(u.flags & UNIT_FP16_FORWARD), bool(u.flags & UNIT_EVAL), u.n0 < u.n_out,
                   (u.x_lds if tc else u.x_ld) != u.Cin, u.out_lds != u.Cout, backward and u.g_ld != u.Cout,
                   backward and u.gin_mode > 0 and u.gin_ld != u.Cin, backward and u.gres_mode > 0 and u.gres_ld != u.Cout)
        return s

    def pcb_unit_forward(self, ref, st):
        self.fwd.append(self.sig(ref._obj, False))
        return self._lib.pcb_unit_forward(ref, st)

    def pcb_unit_backward(self, ref, st):
        self.bwd.append(self.sig(ref._obj, True))
        return self._lib.pcb_unit_backward(ref, st)


@pytest.mark.parametrize("name", XU.MODELS)
def test_every_executor_signature_is_in_the_matrix(monkeypatch, name):
    """forward_pair + backward through the fused executor with me.FWD_FP16 on and off, and one eval forward: every struct handed to
    pcb_unit_forward / pcb_unit_backward has a signature of the case matrix."""
    from pointcontrast_b200 import fused, me, synth
    from pointcontrast_b200.model import load_model
    from tests import refload
    from tests.helpers import det_init
    rec = _Recorder(fused.lib)
    monkeypatch.setattr(fused, "lib", rec)
    batch = synth.collate_pairs([synth.synth_pair(3, scale=0.12)])
    T = {k: torch.from_numpy(batch[k]) for k in ("sinput0_F", "sinput0_C", "sinput1_F", "sinput1_C")}
    net = load_model(name)(3, 32, refload.default_config(), D=3)
    det_init(net, 1)
    net = net.cuda().train()
    matrix = set(XU.signatures())
    for fp16 in (True, False):
        monkeypatch.setattr(me, "FWD_FP16", fp16)
        rec.fwd.clear(), rec.bwd.clear()
        F = net.forward_pair(T["sinput0_F"], T["sinput0_C"], T["sinput1_F"], T["sinput1_C"], torch.device("cuda"))
        (F[0].square().sum() + F[1].sum()).backward()
        torch.cuda.synchronize()
        assert rec.bwd and len(rec.bwd) == len(rec.fwd), (fp16, len(rec.fwd), len(rec.bwd))
        missing = sorted({s.name() for s in rec.bwd if s not in matrix})
        assert not missing, f"{name} fp16={fp16}: signatures outside the case matrix: {missing}"
        assert all(s.fp16 == fp16 and s.two_views for s in rec.bwd)
        assert sorted(rec.bwd) == sorted(s._replace(fp16=fp16) for s in XU.model_units(name))
    monkeypatch.setattr(me, "FWD_FP16", True)
    rec.fwd.clear()
    net.eval()
    with torch.no_grad():
        net(me.SparseTensor(T["sinput0_F"], coords=T["sinput0_C"]).to("cuda"))
    torch.cuda.synchronize()
    assert rec.fwd and all(s.eval for s in rec.fwd)
    missing = sorted({s.name() for s in rec.fwd if s not in matrix})
    assert not missing, f"{name} eval: signatures outside the case matrix: {missing}"


# ----------------------------------------------------------------------------------------------- e. arguments before writes
def _violations_forward(u):
    yield "eval with two views", dict(flags=u.flags | UNIT_EVAL, n0=u.n_out - 1)
    yield "eval without running_mean", dict(flags=u.flags | UNIT_EVAL, n0=u.n_out, running_mean=None)
    yield "eval without running_var", dict(flags=u.flags | UNIT_EVAL, n0=u.n_out, running_var=None)
    yield "fp16 forward without out_bhi", dict(out_bhi=None)
    yield "no x_lo", dict(x_lo=None)
    yield "no weight tiles", dict(wt_fwd=None)
    yield "short workspace", dict(ws_bytes=u.ws_bytes - 1)
    yield "n0 == 0", dict(n0=0)


def _violations_backward(u, stem):
    if stem:
        yield "stem with wg_gather_x == 0", dict(wg_gather_x=0)
        yield "stem with a data gradient", dict(gin_mode=1)
        yield "stem without dz_p", dict(dz_p=None)
        return
    yield "fp16 forward without x_bhi", dict(x_bhi=None)
    yield "fp16 forward without x_blo", dict(x_blo=None)
    yield "gin_mode 2 without gin_p", dict(gin_p=None)
    yield "gin_mode 2 without dg_tbl", dict(dg_tbl=None)
    yield "gin_mode 2 without wt_dg", dict(wt_dg=None)
    yield "no dz_lo", dict(dz_lo=None)
    yield "no dgamma", dict(dgamma=None)
    yield "short workspace", dict(ws_bytes=u.ws_bytes - 1)


def _copy(u, **kw):
    v = _L().PcbUnit.from_buffer_copy(u)
    for k, x in kw.items():
        setattr(v, k, x)
    return v


@pytest.mark.parametrize("stem", (False, True), ids=("k27-fp16", "stem"))
def test_rejected_struct_writes_nothing(plans, stem):
    """A struct that violates exactly one argument check returns PCB_ERR_ARG and leaves z, the out planes, the statistics, dz,
    dgamma, dbeta, dW, gin and gres as they were: a caller that fixes the struct and retries does not accumulate twice."""
    L = _L()
    kind = "stem" if stem else "k27"
    sig = XU.Sig(kind, 27, 3 if stem else 32, 32, True, not stem, False, 0 if stem else 2, 0 if stem else 2, not stem, False, True,
                 False, False, False, False, False)
    case = _Case(sig, plans["split"][kind], seed=31)
    case.forward_operands()
    case.set("g_p", torch.ones(case.n_out, 32, device="cuda"))
    for k in ("z_p", "mean", "invstd"):
        case.set(k, torch.ones_like(case.view(k)))
    cases = [("forward", name, kw) for name, kw in _violations_forward(case.u) if not (stem and name in ("fp16 forward without out_bhi",
                                                                                                             "no x_lo", "no weight tiles"))]
    cases += [("backward", name, kw) for name, kw in _violations_backward(case.u, stem)]
    for fn, name, kw in cases:
        before = case.snapshot()
        v = _copy(case.u, **kw)
        rc = getattr(L.lib, f"pcb_unit_{fn}")(ctypes.byref(v), L.stream())
        torch.cuda.synchronize()
        assert rc == ERR_ARG, (fn, name, rc)
        for k, t in before.items():
            _assert_bits(case.b[k][0], t, f"{fn} rejected ({name}): {k} written")
    # the unchanged struct is accepted by both
    case.forward()
    case.backward()
