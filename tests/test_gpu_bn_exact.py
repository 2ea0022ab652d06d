"""The BatchNorm kernels (`pcb_bn_stats_seg`, `pcb_bn_apply_seg`, `pcb_bn_backward_seg`, `pcb_split_rows`, and the statistics inside
`pcb_unit_forward`) against fp64, element by element, on exactly representable operands (tests/exact_bn.py), at every chunk,
view-boundary and plane-format edge.

Bit-exact: every apply output (fp32 and each 16-bit plane), dgamma / dbeta (also accumulated), the residual gradient in every mode, the
split planes, the mean (fl32 of the fp64 quotient of an exact sum), the fused statistics of the unit against the separate pass, and the
eval-mode statistics.  The rest is held to worst-case bounds derived from the kernels' code; nothing in them is fitted to observed
errors.

Derivation
----------
u = 2^-24, v = 2^-53, gamma_k(u) = k u / (1 - k u).  fl(x op y) = (x op y)(1 + d), |d| <= u; a contracted multiply-add rounds once,
which only removes roundings from the chains counted below.

invstd (bn.cu colstat_kernel, bn_finalize_kernel).  Chunk k of m_k rows has exact shifted sums t1, t2 (exact_bn.py).  Its fp32 M2 is
fl(t2 - fl(fl(t1 t1) / m)): |M2_c - M2_k| <= e_k = gamma_2 t1^2 / m + u (t2 + (1 + gamma_2) t1^2 / m), and 0 when t1 = 0 (then
t2 - 0 is exact); clamping at 0 only moves M2_c toward the true value (M2_k >= 0).  The chunk's sum of x is exact.  The fp64 finalize:
the mean m64 is the fp64 quotient of the exact sum (|m64 - mu| <= v |mu|), the chunk mean c_k one division (or an exact product by
1 / R), d_k = fl(c_k - m64) is within Dd_k = 3 v (|c_k| + |mu|) of c_k - mu, and the M2 sum adds at most ch + 40 roundings of
positive terms (two per term, the lane loop, five shuffle levels).  So
    |M2_fin - M2| <= sum_k e_k + gamma_{ch+40}(v) sum_k (M2_k + e_k + m_k (|d_k| + Dd_k)^2) + sum_k m_k (2 |d_k| Dd_k + Dd_k^2),
var = M2 / rows (one more v), and with DV the resulting bound on |var_c - var|, V = var + eps (eps: the fp32 value, widened),
    |invstd_c - invstd| <= B = Di + 4 v invstd + u (invstd + Di),   Di = DV / (2 (V - DV)^(3/2))
(the fp64 add, sqrt and division, then the fp32 store).  Where every chunk's t1 is zero ("zero-sum" cases) the kernel must also be
within 1 ulp of the fp32 value of invstd.
The running statistics: r <- fl(fl(1 - mom) r + mom s) twice (view 0, then view 1), s the fp32 mean (exact above) or the fp32 unbiased
variance (within Du = DV rows / (rows - 1) + 2 v unb + u (unb + ...)).  Each update adds gamma_2(u)(|a r| + |mom s|) + mom Ds and carries
a = fl(1 - mom) times the previous bound.

dX (bn_bwd_apply_kernel).  g, xhat = (x - mean) invstd, the per-view sums db, dg and G = gamma invstd are exact; inv_n is the host's
fp32 1 / rows.  o = G (g - db inv_n - xhat dg inv_n) in fp32 puts each term through at most four roundings (the products with dg and
inv_n, two subtractions, the final product), so |o_c - o| <= |G| gamma_4(u) (|g| + |db inv_n| + |xhat dg inv_n|).  The fp64 reference
itself is allowed 2^-40 of the magnitudes it sums.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from pointcontrast_b200._lib import BN_RELU, ERR_ARG, PLANES_A_FP16, UNIT_EVAL, UNIT_FP16_FORWARD, UNIT_SEPARATE_STATS
from tests import exact_bn as X
from tests import exact_conv as XC

pytestmark = pytest.mark.gpu

U, V64 = 2.0 ** -24, 2.0 ** -53
REF = 2.0 ** -40
F64 = torch.float64
SENT = -7777.25              # fp32 output sentinel
SENT16 = 0x5A5A              # 16-bit plane sentinel
EPS32 = float(np.float32(X.EPS))
MOM32 = float(np.float32(X.MOMENTUM))
A32 = float(np.float32(1.0) - np.float32(X.MOMENTUM))        # fl32(1 - momentum), as the kernel forms it


def gamma(k, u=U):
    return k * u / (1 - k * u)


def _lib():
    from pointcontrast_b200 import _lib as L
    return L


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# (function, output) -> the element closest to its bound over every case run: (|error| / bound, |error|, bound, case), and the largest
# |error| of any element; printed at the end of the module (pytest -s)
_REPORT = {}


def _note(key, case, got, ref, bound):
    got, ref, bound = (torch.as_tensor(t, dtype=F64).flatten().cpu() for t in (got, ref, bound))
    err = (got - ref).abs()
    ratio = torch.where(err > 0, err / bound, 0.0)
    i = int(ratio.argmax())
    old = _REPORT.get(key, (-1.0, 0.0, 0.0, None, 0.0))
    worst = (float(ratio[i]), float(err[i]), float(bound[i]), case) if float(ratio[i]) > old[0] else old[:4]
    _REPORT[key] = worst + (max(old[4], float(err.max())),)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if _REPORT:
        print(f"\nworst error against its bound on {torch.cuda.get_device_properties(0).name}, {_sms()} SMs")
        for (fn, out), (ratio, err, bound, case, emax) in sorted(_REPORT.items()):
            print(f"  {fn:>10} {out:>13}: |err| {err:.3e} <= bound {bound:.3e} (ratio {ratio:.3f}) at {case}; largest |err| {emax:.3e}")


# ----------------------------------------------------------------------------------------------- buffers
def _in(A, strided, c0=4, extra=12):
    """A ([n, C] fp32 or 16-bit) in an [n, ld] buffer, NaN (fp32) or 0xFFFF codes around it when strided.  -> (buffer, pointer, ld, c0);
    the caller keeps the buffer alive until the kernel has run"""
    n, C = A.shape
    c0, ld = (c0, c0 + C + extra) if strided else (0, C)
    if A.dtype == torch.float32:
        b = torch.full((n, ld), float("nan"), device="cuda")
    else:
        b = torch.full((n, ld), -1, dtype=A.dtype, device="cuda")
    b[:, c0:c0 + C] = A
    return b, b.data_ptr() + b.element_size() * c0, ld, c0


class _Out:
    """[n + 1, ld] output (fp32 or int16 planes) full of the sentinel; the operand is columns [c0, c0 + C) of the first n rows."""

    def __init__(self, n, C, strided, dtype=torch.float32, base=None, c0=8, extra=16):
        self.n, self.C = n, C
        self.c0, self.ld = (c0, c0 + C + extra) if strided else (0, C)
        self.b = torch.full((n + 1, self.ld), SENT if dtype == torch.float32 else SENT16, dtype=dtype, device="cuda")
        if base is not None:
            self.b[:n, self.c0:self.c0 + C] = base
        self.ptr = self.b.data_ptr() + self.b.element_size() * self.c0

    def get(self):
        return self.b[:self.n, self.c0:self.c0 + self.C]

    def assert_padding(self, what):
        pad = self.b.clone()
        pad[:self.n, self.c0:self.c0 + self.C] = pad[self.n, 0]
        assert bool((pad == pad[self.n, 0]).all()) and float(self.b[self.n, 0]) in (SENT, SENT16), f"{what}: padding overwritten"


def _vec(t, pad=8):
    """A 1-D fp32 buffer with `pad` sentinels on each side.  -> (buffer, pointer, slice)"""
    b = torch.full((t.numel() + 2 * pad,), SENT, device="cuda")
    b[pad:pad + t.numel()] = t.flatten()
    return b, b.data_ptr() + 4 * pad, slice(pad, pad + t.numel())


def _vec_padding_ok(b, sl):
    return bool((b[:sl.start] == SENT).all() and (b[sl.stop:] == SENT).all())


def _ws(nbytes):
    return torch.full((max(nbytes, 256),), 255, dtype=torch.uint8, device="cuda")     # 0xFF: NaN as fp32


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16)


def _assert_bits(got, want, what):
    got, want = got.contiguous(), want.contiguous()
    bad = _bits(got) != _bits(want)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} differ; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {want[tuple(i)].item()!r}")


def _assert_within(got, ref, bound, what, key, case):
    err = (got.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} outside the bound; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item()!r}")
    _note(key, case, got, ref, bound)


def split_planes(y, fp16):
    """The expected hi / lo planes of fp32 y: round-to-nearest-even of y (fp16: of y clamped to +-65000) and of the residual."""
    if fp16:
        y = y.clamp(-65000.0, 65000.0)
        hi = y.half()
        return hi.view(torch.int16), (y - hi.float()).half().view(torch.int16)
    hi = y.bfloat16()
    return hi.view(torch.int16), (y - hi.float()).bfloat16().view(torch.int16)


def _ulp32(x):
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


# ----------------------------------------------------------------------------------------------- statistics
def stats_reference(x, n, n0, rm0, rv0):
    """fp64 statistics of x (cuda fp32 [n, C]) view by view and their bounds (see the derivation)."""
    cid, first, size, _ = (t.cuda() for t in X.row_chunks(n, n0))
    xd = x.double()
    C = x.shape[1]
    a = xd - xd[first]
    nch = int(cid.max()) + 1
    t1 = torch.zeros(nch, C, dtype=F64, device="cuda").index_add_(0, cid, a)
    t2 = torch.zeros(nch, C, dtype=F64, device="cuda").index_add_(0, cid, a * a)
    starts = torch.unique(first)
    m = size[starts].double()[:, None]
    pk = xd[starts]
    M2k = t2 - t1 * t1 / m
    q = t1 * t1 / m
    e = torch.where(t1 != 0, gamma(2) * q + U * (t2 + (1 + gamma(2)) * q), 0.0)
    ck = pk + t1 / m
    out = dict(mean=[], V=[], DV=[], rows=[])
    R = X.chunk_rows(n)
    for s, (lo, hi) in enumerate(X.segments(n, n0)):
        rows = hi - lo
        ks = slice(0 if s == 0 else X.chunks_of(n0, R), (X.chunks_of(n0, R) if s == 0 else nch) if n0 < n else nch)
        xs = xd[lo:hi]
        S = xs.sum(0)                                                  # exact: multiples of 2^-3 far below 2^53
        mu = S / rows
        sa = xs - xs[0]
        M2 = (sa * sa).sum(0) - sa.sum(0) ** 2 / rows                 # exact sums; one division, one subtraction
        ref_err = 2 * V64 * (sa * sa).sum(0)
        d = ck[ks] - mu
        Dd = 3 * V64 * (ck[ks].abs() + mu.abs())
        ch = ks.stop - ks.start
        terms = (M2k[ks] + e[ks] + m[ks] * (d.abs() + Dd) ** 2).sum(0)
        DM2 = e[ks].sum(0) + gamma(ch + 40, V64) * terms + (m[ks] * (2 * d.abs() * Dd + Dd * Dd)).sum(0) + ref_err
        var = M2 / rows
        DV = DM2 / rows * (1 + V64) + V64 * var
        out["mean"].append(mu)
        out["V"].append(var)
        out["DV"].append(DV)
        out["rows"].append(rows)
    return out


@pytest.mark.parametrize("case", X.stats_cases(), ids=[c[0] for c in X.stats_cases()])
def test_bn_stats_against_fp64(case):
    L = _lib()
    name, n0, n1, C, offset, pattern = case
    n = n0 + n1
    nn0 = n0 if n1 else n
    seed = X.seed_of(name)
    x = X.stats_operand(n0, n1, C, offset, pattern, seed).cuda()
    strided = C <= 256
    xb, xp, ldx, _ = _in(x, strided)
    gen = torch.Generator().manual_seed(seed + 1)
    rm0 = (torch.randint(-64, 65, (C,), generator=gen).double() / 8).float().cuda()
    rv0 = (torch.randint(1, 65, (C,), generator=gen).double() / 8).float().cuda()
    nseg = len(X.segments(n, nn0))
    mb, mp, msl = _vec(torch.full((2 * C,), SENT))
    ib, ip, isl = _vec(torch.full((2 * C,), SENT))
    rmb, rmp, rmsl = _vec(rm0)
    rvb, rvp, rvsl = _vec(rv0)
    wsb = L.lib.pcb_bn_ws_bytes(n, C)
    ws = _ws(wsb)
    L.check(L.lib.pcb_bn_stats_seg(xp, ldx, n, nn0, C, X.EPS, X.MOMENTUM, mp, ip, rmp, rvp, ws.data_ptr(), wsb, L.stream()))
    torch.cuda.synchronize()
    for b, sl in ((mb, msl), (ib, isl), (rmb, rmsl), (rvb, rvsl)):
        assert _vec_padding_ok(b, sl), name
    mean, invstd = mb[msl].view(2, C), ib[isl].view(2, C)
    assert bool((mean[nseg:] == SENT).all() and (invstd[nseg:] == SENT).all()), (name, "a view that does not exist was written")
    r = stats_reference(x, n, nn0, rm0, rv0)
    rm, rv = rm0.double(), rv0.double()
    Brm, Brv = torch.zeros_like(rm), torch.zeros_like(rv)
    for s in range(nseg):
        mu, var, DV, rows = r["mean"][s], r["V"][s], r["DV"][s], r["rows"][s]
        what = f"{name} view {s}"
        _assert_bits(mean[s], mu.float(), what + " mean")                   # fl32 of the fp64 quotient of the exact sum
        _note(("stats", "mean"), name, mean[s], mu, _ulp32(mu))
        Vt = var + EPS32
        assert bool((DV < Vt).all()), what
        inv = 1 / torch.sqrt(Vt)
        Di = DV / (2 * (Vt - DV) ** 1.5)
        B = Di + 4 * V64 * inv + U * (inv + Di)
        _assert_within(invstd[s], inv, B, what + " invstd", ("stats", "invstd"), name)
        if pattern == "zero-sum":
            _assert_within(invstd[s], inv, _ulp32(inv), what + " invstd (exact chunk M2)", ("stats", "invstd 1 ulp"), name)
        # running statistics, this view after the previous one
        unb = var * rows / (rows - 1) if rows > 1 else var
        Du = (DV * rows / (rows - 1) if rows > 1 else DV) + 2 * V64 * unb
        Du = Du + U * (unb + Du)
        m32 = mu.float().double()
        Brm = A32 * Brm + gamma(2) * (A32 * (rm.abs() + Brm) + MOM32 * m32.abs())
        rm = A32 * rm + MOM32 * m32
        Brv = A32 * Brv + MOM32 * Du + gamma(2) * (A32 * (rv.abs() + Brv) + MOM32 * (unb + Du))
        rv = A32 * rv + MOM32 * unb
    _assert_within(rmb[rmsl], rm, Brm, name + " running_mean", ("stats", "running_mean"), name)
    _assert_within(rvb[rvsl], rv, Brv, name + " running_var", ("stats", "running_var"), name)


# ----------------------------------------------------------------------------------------------- apply
# (fp16 planes, dual bf16 planes, relu, residual, fp32 Y, strided)
APPLY_VARIANTS = ((True, True, True, True, True, True), (False, False, False, False, True, False), (True, True, False, True, False, True),
                  (False, False, True, False, False, True), (True, False, False, False, True, False))


def _apply_call(x, n0, mean, invstd, gamma_, beta, res, v, what):
    """One pcb_bn_apply_seg call with every output framed; returns {name: output} after checking the frames."""
    L = _lib()
    fp16, dual, relu, use_res, use_y, strided = v
    n, C = x.shape
    xb, xp, ldx, _ = _in(x, strided)
    rb, rp, ldr = None, None, 0
    if use_res:
        rb, rp, ldr, _ = _in(res, strided, c0=8, extra=4)
    outs = {}
    Y = _Out(n, C, strided) if use_y else None
    planes = {k: _Out(n, C, strided, torch.int16, c0=4, extra=8) for k in (("hi", "lo", "bhi", "blo") if dual else ("hi", "lo"))}
    mb, ib = mean.flatten().cuda(), invstd.flatten().cuda()
    g, b = gamma_.cuda(), beta.cuda()
    lds = planes["hi"].ld
    rc = L.lib.pcb_bn_apply_seg(xp, ldx, n, n0, C, mb.data_ptr(), ib.data_ptr(), g.data_ptr(), b.data_ptr(), rp, ldr,
                                (BN_RELU if relu else 0) | (PLANES_A_FP16 if fp16 else 0), Y.ptr if Y else None, Y.ld if Y else 0,
                                planes["hi"].ptr, planes["lo"].ptr, lds, planes["bhi"].ptr if dual else None,
                                planes["blo"].ptr if dual else None, L.stream())
    L.check(rc)
    torch.cuda.synchronize()
    if Y:
        Y.assert_padding(what + " Y")
        outs["Y"] = Y.get()
    for k, p in planes.items():
        p.assert_padding(what + " " + k)
        outs[k] = p.get()
    return outs


def _check_apply(x, n0, mean, invstd, gamma_, beta, res, what):
    n, C = x.shape
    view = (torch.arange(n) >= n0).long()
    for vi, v in enumerate(APPLY_VARIANTS):
        fp16, dual, relu, use_res, use_y, strided = v
        y = (x.double() - mean.double()[view]) * invstd.double()[view] * gamma_.double() + beta.double()
        if use_res:
            y = y + res.double()
        if relu:
            y = y.clamp_min(0.0)
        y32 = y.float().cuda()
        assert torch.equal(y32.double(), y.cuda()), (what, "the operands leave the exact range")
        w = f"{what} variant {vi} {v}"
        outs = _apply_call(x.cuda(), n0, mean, invstd, gamma_, beta, res.cuda(), v, w)
        if use_y:
            _assert_bits(outs["Y"], y32, w + " Y")
        hi, lo = split_planes(y32, fp16)
        _assert_bits(outs["hi"], hi, w + " hi")
        _assert_bits(outs["lo"], lo, w + " lo")
        if dual:
            bhi, blo = split_planes(y32, False)
            _assert_bits(outs["bhi"], bhi, w + " dual bf16 hi")
            _assert_bits(outs["blo"], blo, w + " dual bf16 lo")


@pytest.mark.parametrize("case", X.APPLY_CASES, ids=[c[0] for c in X.APPLY_CASES])
def test_bn_apply_bit_exact(case):
    """Exact operands with different statistics per view (the first row of view 1 uses view 1's), then the plane-format edges with
    identity statistics: y = x, so each plane is the rounding of a chosen value (fp16 clamp, subnormals, ties, fp32 extremes)."""
    name, n0, n1, C = case
    n = n0 + n1
    nn0 = n0 if n1 else n
    x, mean, invstd, gamma_, beta, res = X.apply_operands(n0, n1, C, seed=X.seed_of(name))
    _check_apply(x, nn0, mean, invstd, gamma_, beta, res, name)
    if n1:
        view = (torch.arange(n) >= n0).long()
        y0 = (x[n0].double() - mean[0].double()) * invstd[0].double() * gamma_.double()
        y1 = (x[n0].double() - mean[1].double()) * invstd[1].double() * gamma_.double()
        assert bool((y0 != y1).any()) and int(view[n0]) == 1
    px = X.plane_palette(n, C, seed=X.seed_of(name) + 1)
    ones, zeros = torch.ones(2, C), torch.zeros(2, C)
    _check_apply(px, nn0, zeros, ones, ones[0], zeros[0], torch.zeros(n, C), name + " palette")


def test_bn_apply_rejects_a_missing_first_view():
    """n0 == 0 < n would normalise every row with the second view's statistics, which no statistics call writes: an argument error
    before anything is written.  n == 0 stays a no-op."""
    L = _lib()
    n, C = 8, 16
    x = torch.ones(n, C, device="cuda")
    st = torch.ones(2 * C, device="cuda")
    Y = _Out(n, C, False)
    hi, lo = _Out(n, C, False, torch.int16), _Out(n, C, False, torch.int16)
    assert L.lib.pcb_bn_apply_seg(x.data_ptr(), C, n, 0, C, st.data_ptr(), st.data_ptr(), st.data_ptr(), st.data_ptr(), None, 0, 0,
                                  Y.ptr, C, hi.ptr, lo.ptr, C, None, None, L.stream()) == ERR_ARG
    assert b"bad argument" in L.lib.pcb_last_error()
    assert L.lib.pcb_bn_apply_seg(x.data_ptr(), C, 0, 0, C, st.data_ptr(), st.data_ptr(), st.data_ptr(), st.data_ptr(), None, 0, 0,
                                  Y.ptr, C, hi.ptr, lo.ptr, C, None, None, L.stream()) == 0
    torch.cuda.synchronize()
    assert bool((Y.b == SENT).all() and (hi.b == SENT16).all() and (lo.b == SENT16).all())


# ----------------------------------------------------------------------------------------------- backward
# (mask: None / "bf16" / "fp16", gout_mode, gout aliases dY, accumulate, fp32 dX, dX planes, strided)
BACKWARD_VARIANTS = (("bf16", 1, False, 0, True, True, True), ("fp16", 2, False, 1, False, True, True), (None, 0, False, 1, True, False, False),
                     ("fp16", 2, True, 0, True, True, False), ("bf16", 1, True, 1, True, True, True))


def _backward_call(x, dy, codes, n0, mean, invstd, gamma_, bg, bb, gbase, v, what):
    """One pcb_bn_backward_seg call with every output framed.  -> dict of outputs (and of dY when gout aliases it)"""
    L = _lib()
    mask, gmode, alias, acc, use_dx, use_planes, strided = v
    n, C = x.shape
    xb, xp, ldx, _ = _in(x, strided)
    cb, mp, ldm = None, None, 0
    if mask:
        cb, mp, ldm, _ = _in(codes, strided, c0=8, extra=8)
    if alias:
        D = _Out(n, C, strided, base=dy)
        dyp, lddy = D.ptr, D.ld
        gp, ldg = D.ptr, D.ld
    else:
        dyb, dyp, lddy, _ = _in(dy, strided, c0=8, extra=4)
        G = _Out(n, C, strided, base=gbase if gmode == 2 else None) if gmode else None
        gp, ldg = (G.ptr, G.ld) if G else (None, 0)
    dX = _Out(n, C, strided) if use_dx else None
    P = {k: _Out(n, C, strided, torch.int16, c0=4, extra=8) for k in ("hi", "lo")} if use_planes else None
    dgb, dgp, dgsl = _vec(bg if acc else torch.full((C,), SENT))
    dbb, dbp, dbsl = _vec(bb if acc else torch.full((C,), SENT))
    mb, ib, gb = mean.flatten().cuda(), invstd.flatten().cuda(), gamma_.cuda()
    wsb = L.lib.pcb_bn_ws_bytes(n, C)
    ws = _ws(wsb)
    L.check(L.lib.pcb_bn_backward_seg(dyp, lddy, xp, ldx, mp, ldm, n, n0, C, mb.data_ptr(), ib.data_ptr(), gb.data_ptr(),
                                      dX.ptr if dX else None, dX.ld if dX else 0, dgp, dbp, acc, gp, ldg, gmode,
                                      P["hi"].ptr if P else None, P["lo"].ptr if P else None, P["hi"].ld if P else 0,
                                      ws.data_ptr(), wsb, L.stream()))
    torch.cuda.synchronize()
    out = {}
    assert _vec_padding_ok(dgb, dgsl) and _vec_padding_ok(dbb, dbsl), what
    out["dgamma"], out["dbeta"] = dgb[dgsl], dbb[dbsl]
    if dX:
        dX.assert_padding(what + " dX")
        out["dX"] = dX.get()
    if P:
        for k, p in P.items():
            p.assert_padding(what + " d" + k)
            out[k] = p.get()
    if gmode:
        Gb = D if alias else G
        Gb.assert_padding(what + " gout")
        out["gout"] = Gb.get()
    return out


@pytest.mark.parametrize("case", X.BACKWARD_CASES, ids=[c[0] for c in X.BACKWARD_CASES])
def test_bn_backward_against_fp64(case):
    name, n0, n1, C = case
    n = n0 + n1
    nn0 = n0 if n1 else n
    seed = X.seed_of(name)
    x, dy, mean, invstd, gamma_, bg, bb, gbase = X.backward_operands(n0, n1, C, seed)
    assert X.backward_terms(x, dy, mean, invstd, nn0, bg)[0] < 1.0
    xc, dyc = x.cuda(), dy.cuda()
    view = (torch.arange(n, device="cuda") >= nn0).long()
    md, isd = mean.double().cuda(), invstd.double().cuda()
    xhat = (xc.double() - md[view]) * isd[view]
    Gm = gamma_.double().cuda() * isd[view]
    for vi, v in enumerate(BACKWARD_VARIANTS):
        mask, gmode, alias, acc, use_dx, use_planes, strided = v
        w = f"{name} variant {vi} {v}"
        codes = X.mask_codes(n, C, mask, seed + vi).cuda() if mask else None
        ok = X.mask_passes(codes) if mask else torch.ones(n, C, dtype=torch.bool, device="cuda")
        g = torch.where(ok, dyc.double(), 0.0)
        segs = X.segments(n, nn0)
        db = torch.stack([g[a:e].sum(0) for a, e in segs])
        dg = torch.stack([(g * xhat)[a:e].sum(0) for a, e in segs])
        out = _backward_call(xc, dyc, codes, nn0, mean, invstd, gamma_, bg, bb, gbase.cuda(), v, w)
        _assert_bits(out["dbeta"], (db.sum(0) + (bb.double().cuda() if acc else 0)).float(), w + " dbeta")
        _assert_bits(out["dgamma"], (dg.sum(0) + (bg.double().cuda() if acc else 0)).float(), w + " dgamma")
        if gmode:
            base = dyc.double() if alias else gbase.double().cuda()
            _assert_bits(out["gout"], (g + base if gmode == 2 else g).float(), w + " gout")
        inv_n = torch.tensor([float(np.float32(1.0) / np.float32(e - a)) for a, e in segs], dtype=F64, device="cuda")
        T1 = (db * inv_n[:, None])[view]
        T2 = xhat * (dg * inv_n[:, None])[view]
        ref = Gm * (g - T1 - T2)
        mag = Gm.abs() * (g.abs() + T1.abs() + T2.abs())
        bound = gamma(4) * mag + REF * mag
        if use_dx:
            _assert_within(out["dX"], ref, bound, w + " dX", ("backward", "dX"), name)
        if use_planes:
            if use_dx:
                own = out["dX"]
            else:                                   # the same call with dX written (deterministic): its dX is the one split
                own = _backward_call(xc, dyc, codes, nn0, mean, invstd, gamma_, bg, bb, gbase.cuda(),
                                     (mask, 0, False, 0, True, False, strided), w + " (dX)")["dX"]
                _assert_within(own, ref, bound, w + " dX", ("backward", "dX"), name)
            hi, lo = split_planes(own.contiguous(), False)
            _assert_bits(out["hi"], hi, w + " dX hi")
            _assert_bits(out["lo"], lo, w + " dX lo")


# ----------------------------------------------------------------------------------------------- split rows
@pytest.mark.parametrize("fp16", (False, True))
def test_split_rows_bit_exact(fp16):
    L = _lib()
    for n, C in ((1000, 36), (1, 4), (257, 1024)):
        x = X.plane_palette(n, C, seed=n + C).cuda()
        xb, xp, ldx, _ = _in(x, True)
        hi, lo = _Out(n, C, True, torch.int16), _Out(n, C, True, torch.int16)
        L.check(L.lib.pcb_split_rows(xp, ldx, n, C, hi.ptr, lo.ptr, hi.ld, PLANES_A_FP16 if fp16 else 0, L.stream()))
        torch.cuda.synchronize()
        what = f"split_rows n={n} C={C} fp16={fp16}"
        hi.assert_padding(what)
        lo.assert_padding(what)
        eh, el = split_planes(x, fp16)
        _assert_bits(hi.get(), eh, what + " hi")
        _assert_bits(lo.get(), el, what + " lo")
    assert L.lib.pcb_split_rows(None, 4, 0, 4, None, None, 4, 0, L.stream()) == 0


# ----------------------------------------------------------------------------------------------- through pcb_unit_forward


def _unit_forward(n, n0, flags, seed):
    """pcb_unit_forward of one 27-offset 32 -> 32 unit on exact fp16 planes and tiles (tests/exact_conv.py), production flags.
    -> dict of every output after the call"""
    L = _lib()
    K, Cin, Cout = 27, 32, 32
    fmt = XC.FP16
    gen = torch.Generator(device="cuda").manual_seed(seed)
    hi, lo = XC.capped_planes(n, Cin, XC.row_cap(fmt, K, Cin), fmt.HI, fmt.LO, gen, "cuda")
    xh, xl = hi.half().view(torch.int16), lo.half().view(torch.int16)
    W = XC.weights(K, Cin, Cout, fmt, gen, "cuda")[0]
    ft = torch.empty(L.lib.pcb_weight_tile_bytes(K, Cin, Cout, 0), dtype=torch.uint8, device="cuda")
    dt = torch.empty(L.lib.pcb_weight_tile_bytes(K, Cin, Cout, 1), dtype=torch.uint8, device="cuda")
    L.check(L.lib.pcb_weight_tile(W.data_ptr(), K, Cin, Cout, ft.data_ptr(), dt.data_ptr(), 16, L.stream()))
    tbl = torch.randint(0, n, (K, n), generator=gen, device="cuda", dtype=torch.int32)
    tbl[torch.rand(K, n, generator=gen, device="cuda") > 0.4] = -1
    g2 = torch.Generator().manual_seed(seed + 1)
    o = dict(gamma=torch.tensor(X.GAMMA)[torch.randint(0, 5, (Cout,), generator=g2)], beta=(torch.randint(-8, 9, (Cout,), generator=g2) / 8.0),
             running_mean=torch.randint(-64, 65, (Cout,), generator=g2) / 8.0, running_var=torch.randint(1, 65, (Cout,), generator=g2) / 8.0,
             mean=torch.full((2 * Cout,), SENT), invstd=torch.full((2 * Cout,), SENT), z_p=torch.full((n, Cout), SENT),
             out_hi=torch.zeros(n, Cout, dtype=torch.int16), out_lo=torch.zeros(n, Cout, dtype=torch.int16),
             out_bhi=torch.zeros(n, Cout, dtype=torch.int16), out_blo=torch.zeros(n, Cout, dtype=torch.int16))
    o = {k: t.float().cuda() if t.dtype != torch.int16 else t.cuda() for k, t in o.items()}
    u = L.PcbUnit()
    u.n_in = u.n_out = n
    u.n0, u.K, u.Cin, u.Cout, u.relu = n0, K, Cin, Cout, 1
    u.fwd_tbl, u.fwd_stride = tbl.data_ptr(), n
    u.W, u.wt_fwd, u.wt_dg = W.data_ptr(), ft.data_ptr(), dt.data_ptr()
    u.x_hi, u.x_lo, u.x_lds = xh.data_ptr(), xl.data_ptr(), Cin
    for k, t in o.items():
        setattr(u, k, t.data_ptr())
    u.eps, u.momentum = X.EPS, X.MOMENTUM
    u.z_ld = u.out_lds = Cout
    u.flags = flags
    wsb = L.lib.pcb_unit_ws_bytes(K, n, n, Cin, Cout)
    ws = _ws(wsb)
    u.ws, u.ws_bytes = ws.data_ptr(), wsb
    L.check(L.lib.pcb_unit_forward(ctypes.byref(u), L.stream()))
    torch.cuda.synchronize()
    return o


def test_unit_forward_statistics_bit_identical_to_the_separate_pass():
    """On an offset-split level the reduction pass takes the statistics of z (MODE 2); they must be the bits `pcb_bn_stats_seg` computes
    from the z the unit wrote, and the bits of PCB_UNIT_SEPARATE_STATS: every pass loads the same fp32 row sums in the same order.
    PCB_UNIT_EVAL normalises with the running statistics, leaves them untouched, and its invstd is fp32 1 / sqrt(running_var + eps)."""
    L = _lib()
    n, n0 = 300, 170
    assert XC.conv_splits(27, n, 32, 32, _sms()) > 1
    fused = _unit_forward(n, n0, UNIT_FP16_FORWARD, seed=5)
    sep = _unit_forward(n, n0, UNIT_FP16_FORWARD | UNIT_SEPARATE_STATS, seed=5)
    for k in ("z_p", "mean", "invstd", "running_mean", "running_var", "out_hi", "out_lo", "out_bhi", "out_blo"):
        _assert_bits(fused[k], sep[k], f"unit fused vs separate statistics: {k}")
    init = _unit_forward(1, 1, UNIT_FP16_FORWARD | UNIT_EVAL, seed=5)          # the initial running statistics of seed 5, untouched
    z = fused["z_p"]
    assert bool(torch.isfinite(z).all()) and len(torch.unique(z)) > 100
    mean, invstd = torch.full((2 * 32,), SENT, device="cuda"), torch.full((2 * 32,), SENT, device="cuda")
    rm, rv = init["running_mean"].clone(), init["running_var"].clone()
    wsb = L.lib.pcb_bn_ws_bytes(n, 32)
    ws = _ws(wsb)
    L.check(L.lib.pcb_bn_stats_seg(z.data_ptr(), 32, n, n0, 32, X.EPS, X.MOMENTUM, mean.data_ptr(), invstd.data_ptr(), rm.data_ptr(),
                                   rv.data_ptr(), ws.data_ptr(), wsb, L.stream()))
    torch.cuda.synchronize()
    for k, t in (("mean", mean), ("invstd", invstd), ("running_mean", rm), ("running_var", rv)):
        _assert_bits(fused[k], t, f"unit MODE 2 statistics vs pcb_bn_stats_seg on z: {k}")
    ev = _unit_forward(n, n, UNIT_FP16_FORWARD | UNIT_EVAL, seed=5)
    _assert_bits(ev["running_mean"], init["running_mean"], "eval: running_mean untouched")
    _assert_bits(ev["running_var"], init["running_var"], "eval: running_var untouched")
    _assert_bits(ev["mean"][:32], init["running_mean"], "eval mean")
    rvn = init["running_var"].cpu().numpy()
    want = (np.float32(1.0) / np.sqrt(rvn + np.float32(EPS32))).astype(np.float32)
    _assert_bits(ev["invstd"][:32].cpu(), torch.from_numpy(want), "eval invstd")
    assert bool((ev["mean"][32:] == SENT).all() and (ev["invstd"][32:] == SENT).all())
