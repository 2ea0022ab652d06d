"""The small kernels of every training step held to fp64 at their row, tail and degenerate-input edges: the semantic-segmentation
cross-entropy (`pcb_ce_forward_backward`, and the loss `pcb_seg_metrics` reports), the L2 normalisation of the output features
(`pcb_l2norm_forward/backward`), the flat SGD step (`pcb_sgd_step`, and `FlatSGD`'s padding) and the pooling gather-sum
(`pcb_gather_sum`).  Case lists and operands: tests/exact_train_kernels.py.  Every call goes through the C ABI with its outputs full of
NaN, a sentinel one element past each output and a NaN-poisoned workspace: an entry left unwritten, or written out of bounds, fails.

Each kernel is tested bit for bit on exactly representable operands and against fp64 within a worst-case bound on random ones.  The
bounds count the roundings of the kernels' code; nothing in them is fitted to observed errors.

Derivation
----------
u = 2^-24.  fl(x op y) = (x op y)(1 + d), |d| <= u; a contracted multiply-add rounds once, which only removes roundings from the chains
below.  expf is within 2 ulp (relative RHO = 2^-22, absolute 2^-148 for a subnormal result) and exact at 0 and -inf; logf is within
1 ulp (2^-23 |result|); sqrtf and fp32 division are correctly rounded (no fast-math).  lam(x) = -log(1 - x) turns a relative error
into a bound on a logarithm.  gamma_k = k u / (1 - k u).  The fp64 references are allowed REF = 2^-36 of the magnitudes they combine.

Cross-entropy, row i with maximum m (exact: fmaxf), d_j = x_j - m, ls = log sum_j e^(d_j), lse = m + ls.
  Each term expf(fl(x_j - m)) = e^(d_j) f_j with |log f_j| <= u |d_j| + lam(RHO) (0 for x_j = -inf: the term is exactly 0), plus
  2^-148 absolute.  The warp sums its C terms in k = ceil(C / 32) + 4 roundings of positive quantities (a lane's stride after its
  first term, then five butterfly levels), so the sum s_c satisfies
      |log s_c - ls| <= B = log sum_j w_j exp(a_j) + C 2^-147,  a_j = u |d_j| + lam(RHO) + k lam(u),  w_j = softmax_j
  (s >= 1: the maximum's term is 1).  logf adds 2^-23 (ls + B):  |L_c - ls| <= E2 = B + 2^-23 (ls + B).
  lse_c = fl(m + L_c):            E_lse = E2 + u (|lse| + E2)
  rowloss_c = fl(lse_c - x_t):    E_row = E_lse + u (|lse - x_t| + E_lse)
  loss = fl32(fp64 sum / count):  E_loss = E_m + u (|loss| + E_m),  E_m = mean E_row + (n + 64) 2^-53 mean(|rowloss| + E_row).
  Gradient, P = exp(x - lse), q = grad_scale / count (grad_scale: the fp32 argument): p_c = expf(fl(x - lse_c)) has
  |log(p_c / P)| <= b = E_lse + u (|x - lse| + E_lse) + lam(RHO), so |p_c - P| <= dP = P expm1(b) + 2^-148; then one subtraction,
  fl(grad_scale / count) and one product:  |g_c - (P - delta) q| <= q ((|P - delta| + E_h)(1 + u)^2 - |P - delta|),
  E_h = dP + u (|P - delta| + dP).  Rows not counted (target == ignore_index or outside [0, C)) have gradient exactly 0.

L2 normalisation, row of x, ss = sum x^2, inv = 1 / sqrt(ss), y = x inv.
  ss_c: fused multiply-adds of positive terms along a lane's stride, then five butterfly adds: |ss_c / ss - 1| <= gamma_k,
  k = ceil(C / 32) + 5.  inv_c = fl(1 / fl(sqrt(ss_c))): |inv_c / inv - 1| <= r_inv = (1 + u) / ((1 - u) sqrt(1 - gamma_k)) - 1.
  y_c = fl(x inv_c): r_y = (1 + r_inv)(1 + u) - 1 relative.
  Backward, dx = (dy - y (y . dy)) inv: dot_c = fused multiply-adds of y_c dy, k roundings: with S = sum |y dy|,
  |dot_c - y . dy| <= E_dot = r_y S + gamma_k (1 + r_y) S.  h_c = fl(dy - fl(y_c dot_c)) (contracted or not):
  |h_c - h| <= E_h = |y| E_dot + r_y |y| (|dot| + E_dot) + gamma_2 (|dy| + |y| (|dot| + E_dot)(1 + r_y)), and
  dx_c = fl(h_c inv_c):  |dx_c - dx| <= inv ((|h| + E_h)(1 + r_inv)(1 + u) - |h|).
  A row whose fp32 sum of squares is 0 (a zero row, or every square below half the smallest subnormal) or overflows to +inf gets what
  the reference expression F / torch.norm(F, p=2, dim=1, keepdim=True) gives on CUDA fp32, bit for bit (NaN payloads aside): a zero
  row all NaN (0 * inf), an underflowing row +-inf at its nonzero entries and NaN at its zeros, an overflowing row +-0; inv_norm is
  +inf for the first two and 0 for the last.  torch sums the squares in fp32 as the kernel does, except at C = 1, where it takes the
  norm of the single column as |F| and the expression gives +-1; the kernel gives F / sqrt(F^2) there too, with the same edges.

SGD, one step from the kernel's fp32 state (p, g, buf; the scalars lr, momentum, weight_decay, grad_scale and keep =
fp32(1 - dampening) the kernel receives): each statement d = g gs + wd p, b = momentum buf + keep d, p - lr b is at most two products
and a sum, three roundings:  E_d = gamma_3 (|g gs| + |wd p|),  E_b = keep E_d + gamma_3 (|momentum buf| + keep (|d| + E_d))
(E_b = E_d on the first step),  E_p = lr E_b + gamma_3 (|p| + lr (|b| + E_b)).

The gather-sum adds small integers and is exact in any order.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from pointcontrast_b200._lib import check, lib, ptr, stream
from tests import exact_train_kernels as X

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RHO = 2.0 ** -22                     # expf: 2 ulp
LOGF = 2.0 ** -23                    # logf: 1 ulp
REF = 2.0 ** -36                     # the fp64 references
SENT = -7777.25                      # fp32 sentinel one past every output
F64 = torch.float64
NAN = float("nan")


def lam(x):
    return -math.log1p(-x)


def gamma(k):
    return k * U / (1 - k * U)


def _out(n, dtype=torch.float32, fill=NAN, sent=SENT):
    """A [n + 1] device buffer: n entries of `fill`, then the sentinel.  -> (buffer, view of the n entries)"""
    b = torch.full((n + 1,), fill, dtype=dtype, device="cuda")
    b[n] = sent
    return b, b[:n]


def _sent_ok(b, sent=SENT):
    return bool(b[-1] == sent)


def _ws(nbytes):
    return torch.full((max(nbytes, 256),), 0xFF, dtype=torch.uint8, device="cuda")       # every fp32 word a NaN


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bits(got, want, what):
    """Same fp32 bits, or NaN on both sides (NaN payloads are not part of any result)."""
    got, want = got.float(), want.to(got.device).float()
    same = (_bits(got) == _bits(want)) | (torch.isnan(got) & torch.isnan(want))
    if not bool(same.all()):
        i = torch.nonzero(~same)[0].tolist()
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.numel()} differ; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {want[tuple(i)].item()!r}")


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = torch.nonzero(~ok)[0].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} outside the bound; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {ref[tuple(i)].item()!r} +- {bound[tuple(i)].item()!r}")


# ----------------------------------------------------------------------------------------------- cross-entropy
def ce_call(x, t, C, ignore, grad_scale):
    """pcb_ce_forward_backward -> (loss, dlogits [n, C]) with NaN-filled outputs, sentinels and a poisoned workspace."""
    n = t.shape[0]
    xc, tc = x.cuda().contiguous(), t.cuda().contiguous()
    lb, loss = _out(1)
    gb, g = _out(n * C)
    wsb = lib.pcb_ce_ws_bytes(n)
    ws = _ws(wsb)
    check(lib.pcb_ce_forward_backward(ptr(xc), ptr(tc), n, C, int(ignore), float(grad_scale), ptr(lb), ptr(gb), ptr(ws), wsb, stream()))
    torch.cuda.synchronize()
    assert _sent_ok(lb) and _sent_ok(gb), "cross-entropy wrote past an output"
    return loss[0], g.view(n, C)


def seg_metrics_stats(x, t, C, ignore):
    """pcb_seg_metrics from zeroed accumulators -> stats (fp64 [3])."""
    n = t.shape[0]
    xc, tc = x.cuda().contiguous(), t.cuda().contiguous()
    pb, _ = _out(n, torch.int32, fill=-1, sent=-7)
    hist = torch.zeros(C * C + 1, dtype=torch.int64, device="cuda")
    hist[-1] = -7
    sb, stats = _out(3, F64, fill=0.0)
    wsb = lib.pcb_seg_metrics_ws_bytes(n)
    ws = _ws(wsb)
    check(lib.pcb_seg_metrics(ptr(xc), ptr(tc), n, C, int(ignore), ptr(pb), None, ptr(hist), ptr(sb), ptr(ws), wsb, stream()))
    torch.cuda.synchronize()
    assert _sent_ok(pb, -7) and int(hist[-1]) == -7 and _sent_ok(sb), "pcb_seg_metrics wrote past an output"
    return stats.cpu()


def check_seg_metrics_loss(x, t, C, ignore, loss, want_loss, what):
    """stats[0] = loss * n with loss the bits pcb_ce_forward_backward returned, and those the expected bits (NaN: no counted row)."""
    n = t.shape[0]
    stats = seg_metrics_stats(x, t, C, ignore)
    for lv in (float(loss), float(want_loss)):
        want = lv * float(n)
        got = float(stats[0])
        assert (math.isnan(got) and math.isnan(want)) or got == want, (what, "seg_metrics stats[0]", got, want)
    assert float(stats[2]) == float(n), what


def ce_reference(x32, t, C, ignore, grad_scale):
    """fp64 loss, dlogits and their bounds (see the derivation), on the device."""
    x = x32.cuda().double()
    t = t.cuda()
    n = t.shape[0]
    v = X.ce_valid(t, C, ignore)
    tl = t.clamp(0, C - 1)
    rows = torch.arange(n, device="cuda")
    fin = x > -math.inf
    m = x.max(1, keepdim=True).values
    d = x - m
    ls = torch.logsumexp(d, 1, keepdim=True)
    k = -(-C // 32) + 4
    a = torch.where(fin, U * d.abs() + lam(RHO) + k * lam(U), 0.0)
    B = torch.logsumexp(d + a, 1, keepdim=True) - ls + C * 2.0 ** -147
    E2 = B + LOGF * (ls + B)
    lse = m + ls
    E_lse = E2 + U * (lse.abs() + E2) + REF * (m.abs() + ls + 1)
    xt = x[rows, tl][:, None]
    rowloss = (lse - xt)[:, 0]
    E_row = (E_lse + U * ((lse - xt).abs() + E_lse))[:, 0]
    cnt = int(v.sum())
    if cnt:
        loss = float(rowloss[v].mean())
        E_m = float(E_row[v].mean()) + (n + 64) * 2.0 ** -53 * float((rowloss[v].abs() + E_row[v]).mean())
        E_loss = E_m + U * (abs(loss) + E_m) + REF * (1 + abs(loss))
    else:
        loss, E_loss = NAN, NAN
    q = float(np.float32(grad_scale)) / max(cnt, 1)
    P = torch.exp(x - lse)
    b = torch.where(fin, E_lse + U * ((x - lse).abs() + E_lse) + lam(RHO), 0.0)
    dP = torch.where(fin, P * torch.expm1(b) + 2.0 ** -148, 0.0)
    G0 = P.clone()
    G0[rows[v], tl[v]] -= 1
    E_h = dP + U * (G0.abs() + dP)
    G = torch.where(v[:, None], G0 * q, 0.0)
    E_g = torch.where(v[:, None], q * ((G0.abs() + E_h) * (1 + U) ** 2 - G0.abs()) + REF * q * (P + 1), 0.0)
    return loss, E_loss, G, E_g


def _torch_ce(x32, t, C, ignore):
    """torch's fp64 cross-entropy on the same rows, out-of-range targets as ignored (torch raises on them): (loss, dlogits)."""
    x = x32.cuda().double().requires_grad_(True)
    t = t.cuda()
    tt = torch.where(X.ce_valid(t, C, ignore) | (t == ignore), t, torch.full_like(t, ignore))
    loss = torch.nn.functional.cross_entropy(x, tt, ignore_index=ignore)
    loss.backward()
    return float(loss.detach()), x.grad


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


@pytest.mark.parametrize("C", X.CE_C)
def test_ce_bit_exact_on_dominated_rows(C):
    """Integer logits with one dominant entry per row (every other exponential 0): the loss, every gradient entry and pcb_seg_metrics'
    stats[0] exact, at every n, target mix and grad_scale."""
    for n in X.ce_n_list(C):
        for i, mix in enumerate(X.CE_MIXES):
            gs = X.GRAD_SCALES[(i + n) % len(X.GRAD_SCALES)]
            gen = torch.Generator().manual_seed(_seed("ce exact", C, n, mix))
            t = X.ce_targets(mix, n, C, gen)
            ign = X.ce_ignore(mix, C)
            x, jmax = X.ce_dominated(t, C, gen)
            what = f"C={C} n={n} {mix} grad_scale={gs}"
            loss, g = ce_call(x, t, C, ign, gs)
            want_loss, want_g = X.ce_dominated_expected(x, t, jmax, C, ign, gs)
            _assert_bits(loss.reshape(1), torch.tensor([want_loss]), what + " loss")
            _assert_bits(g, want_g.cuda(), what + " dlogits")
            check_seg_metrics_loss(x, t, C, ign, loss, want_loss, what)


@pytest.mark.parametrize("C", X.CE_C)
def test_ce_within_fp64_bound(C):
    """Random logits with -inf entries, |x| up to 10^4, confident and flat rows: loss and gradient within the derived bound of fp64, the
    reference equal to torch's fp64 cross-entropy, pcb_seg_metrics' loss the same bits."""
    for n in X.ce_n_list(C):
        for i, mix in enumerate(X.CE_MIXES):
            gs = X.GRAD_SCALES[(i + n + 1) % len(X.GRAD_SCALES)]
            gen = torch.Generator().manual_seed(_seed("ce fp64", C, n, mix))
            t = X.ce_targets(mix, n, C, gen)
            ign = X.ce_ignore(mix, C)
            x = X.ce_edge_logits(t, C, gen)
            what = f"C={C} n={n} {mix} grad_scale={gs}"
            loss, g = ce_call(x, t, C, ign, gs)
            ref, E_loss, G, E_g = ce_reference(x, t, C, ign, gs)
            tl, tg = _torch_ce(x, t, C, ign)
            if not bool(X.ce_valid(t, C, ign).any()):                   # "all ignored", and single rows that are not counted
                assert math.isnan(float(loss)) and math.isnan(ref) and math.isnan(tl), what
                assert not bool(tg.any()), what
                _assert_bits(g, torch.zeros_like(g), what + " dlogits")
            else:
                assert abs(ref - tl) <= REF * (1 + abs(tl)), (what, ref, tl)
                assert bool(((G - tg * float(np.float32(gs))).abs() <= REF * (1 + tg.abs())).all()), what
                assert abs(float(loss) - ref) <= E_loss, (what, float(loss), ref, E_loss)
                _assert_within(g, G, E_g, what + " dlogits")
            check_seg_metrics_loss(x, t, C, ign, loss, loss, what)


def test_ce_nan_logits_contract():
    """A NaN logit in a counted row makes the loss NaN and that row's gradient NaN, as torch; in a row that is not counted it changes
    nothing (torch's backward gives that row NaN times its zero incoming gradient)."""
    C, n = 13, 9
    gen = torch.Generator().manual_seed(13)
    t = X.ce_targets("valid", n, C, gen)
    t[1] = 255
    t[2] = -1
    x = X.ce_edge_logits(t, C, gen)
    # a NaN in a counted row (row 0) and in two rows that are not counted
    xn = x.clone()
    xn[0, (int(t[0]) + 1) % C] = NAN
    xn[1, 3] = NAN
    xn[2, 0] = NAN
    loss, g = ce_call(xn, t, C, 255, 1.0)
    tl, tg = _torch_ce(xn, t, C, 255)
    assert math.isnan(float(loss)) and math.isnan(tl)
    assert bool(torch.isnan(g[0]).all()) and bool(torch.isnan(tg[0]).all())
    _assert_bits(g[1:3], torch.zeros(2, C, device="cuda"), "rows not counted")
    _, _, G, E_g = ce_reference(x, t, C, 255, 1.0)
    _assert_within(g[3:], G[3:], E_g[3:], "other rows")
    check_seg_metrics_loss(xn, t, C, 255, loss, NAN, "NaN in a counted row")
    # NaN only in rows that are not counted: the loss and gradient of the rest
    xn[0] = x[0]
    loss, g = ce_call(xn, t, C, 255, 1.0)
    ref, E_loss, G, E_g = ce_reference(x, t, C, 255, 1.0)
    tl, _ = _torch_ce(xn, t, C, 255)
    assert abs(float(loss) - ref) <= E_loss and abs(tl - ref) <= REF * (1 + abs(tl)), (float(loss), ref, tl)
    _assert_bits(g[1:3], torch.zeros(2, C, device="cuda"), "rows not counted")
    rows = [0] + list(range(3, n))
    _assert_within(g[rows], G[rows], E_g[rows], "counted rows")
    check_seg_metrics_loss(xn, t, C, 255, loss, loss, "NaN in rows not counted")


# ----------------------------------------------------------------------------------------------- L2 normalisation
def l2_call(x, dy=None):
    """pcb_l2norm_forward (and, with dy, pcb_l2norm_backward on its outputs) -> (y, inv_norm, dx)."""
    n, C = x.shape
    yb, y = _out(n * C)
    ib, inv = _out(n)
    check(lib.pcb_l2norm_forward(ptr(x), n, C, ptr(yb), ptr(ib), stream()))
    dx = None
    if dy is not None:
        db, dx = _out(n * C)
        check(lib.pcb_l2norm_backward(ptr(dy), ptr(yb), ptr(ib), n, C, ptr(db), stream()))
    torch.cuda.synchronize()
    assert _sent_ok(yb) and _sent_ok(ib) and (dy is None or _sent_ok(db)), "L2 normalisation wrote past an output"
    return y.view(n, C), inv, None if dx is None else dx.view(n, C)


@pytest.mark.parametrize("C", X.L2_C)
def test_l2norm_bit_exact_on_power_of_four_rows(C):
    """y, inv_norm and dx exact on rows whose sum of squares is a power of 4, at every n."""
    for n in X.l2_n_list(C):
        gen = torch.Generator(device="cuda").manual_seed(_seed("l2 exact", C, n))
        x, dy = X.l2_exact_rows(n, C, gen)
        y, inv, dx = l2_call(x, dy)
        xd, dyd = x.double(), dy.double()
        ss = (xd * xd).sum(1, keepdim=True)
        mant, ex = torch.frexp(ss)                                  # a power of 4: 0.5 * 2^ex with ex - 1 even
        assert bool((mant == 0.5).all() & ((ex - 1) % 2 == 0).all() & (ss < 2 ** 24).all())
        iv = 1 / ss.sqrt()
        yd = xd * iv
        dxd = (dyd - yd * (yd * dyd).sum(1, keepdim=True)) * iv
        what = f"C={C} n={n}"
        _assert_bits(inv, iv[:, 0], what + " inv_norm")
        _assert_bits(y, yd, what + " y")
        _assert_bits(dx, dxd, what + " dx")


def l2_reference(x, dy):
    """fp64 y, inv_norm, dx and their bounds (see the derivation)."""
    n, C = x.shape
    xd, dyd = x.double(), dy.double()
    k = -(-C // 32) + 5
    gk = gamma(k)
    r_inv = (1 + U) / ((1 - U) * math.sqrt(1 - gk)) - 1 + REF
    r_y = (1 + r_inv) * (1 + U) - 1
    iv = 1 / (xd * xd).sum(1, keepdim=True).sqrt()
    y = xd * iv
    dot = (y * dyd).sum(1, keepdim=True)
    S = (y * dyd).abs().sum(1, keepdim=True)
    E_dot = r_y * S + gk * (1 + r_y) * S + REF * S
    h = dyd - y * dot
    ay = y.abs()
    E_h = ay * E_dot + r_y * ay * (dot.abs() + E_dot) + gamma(2) * (dyd.abs() + ay * (dot.abs() + E_dot) * (1 + r_y))
    dx = h * iv
    E_dx = iv * ((h.abs() + E_h) * (1 + r_inv) * (1 + U) - h.abs())
    return dict(y=y, E_y=r_y * y.abs(), inv=iv[:, 0], E_inv=r_inv * iv[:, 0], dx=dx, E_dx=E_dx)


@pytest.mark.parametrize("C", X.L2_C)
def test_l2norm_within_fp64_bound(C):
    """Random rows of norms from 10^-3 to 10^3, some entries zero: y, inv_norm and dx within the derived bound of fp64."""
    for n in X.l2_n_list(C):
        gen = torch.Generator(device="cuda").manual_seed(_seed("l2 fp64", C, n))
        scale = torch.pow(10.0, torch.rand(n, 1, generator=gen, device="cuda") * 6 - 3)
        x = torch.randn(n, C, generator=gen, device="cuda") * scale
        x[torch.rand(n, C, generator=gen, device="cuda") < 0.1] = 0
        x[:, 0] += (x.abs().sum(1) == 0).float()                    # no zero row here
        dy = torch.randn(n, C, generator=gen, device="cuda")
        y, inv, dx = l2_call(x, dy)
        r = l2_reference(x, dy)
        what = f"C={C} n={n}"
        _assert_within(y, r["y"], r["E_y"], what + " y")
        _assert_within(inv, r["inv"], r["E_inv"], what + " inv_norm")
        _assert_within(dx, r["dx"], r["E_dx"], what + " dx")


@pytest.mark.parametrize("C", (1, 2, 32, 33, 96))
def test_l2norm_degenerate_rows_match_the_reference_expression(C):
    """Zero rows, rows whose squares all underflow and rows whose sum of squares overflows: y and inv_norm bit for bit as
    F / torch.norm(F, p=2, dim=1, keepdim=True) on CUDA fp32 (NaN payloads aside) -- at C = 1 as F / sqrt(F^2), since torch takes the
    norm of a single column as |F|; the ordinary rows beside them within their bound."""
    gen = torch.Generator(device="cuda").manual_seed(C)
    n = 40
    x = torch.randn(n, C, generator=gen, device="cuda")
    kind = torch.arange(n, device="cuda") % 4
    x[kind == 0] = 0
    x[kind == 1] = torch.randn(int((kind == 1).sum()), C, generator=gen, device="cuda").clamp(-3, 3) * 3e-24      # squares < 2^-150
    if C > 1:
        x[kind == 1, 0] = 0
    x[kind == 2, 0] = 3e19                                                                                      # square > FLT_MAX
    if C > 1:
        x[kind == 2, 1] = -2e19
    y, inv, _ = l2_call(x)
    nrm = (x * x).sum(1, keepdim=True).sqrt()
    if C > 1:
        assert torch.equal(torch.norm(x, p=2, dim=1, keepdim=True), nrm)
    else:
        assert torch.equal(torch.norm(x, p=2, dim=1, keepdim=True), x.abs())
    ref = x / nrm
    edge = kind < 3
    assert bool((nrm[kind < 2] == 0).all() & torch.isinf(nrm[kind == 2]).all())
    _assert_bits(y[edge], ref[edge], f"C={C} degenerate rows y")
    _assert_bits(inv[edge], 1 / nrm[edge, 0], f"C={C} degenerate rows inv_norm")
    assert bool(torch.isnan(y[kind == 0]).all() & torch.isinf(inv[kind < 2]).all() & (inv[kind == 2] == 0).all())
    assert bool((y[kind == 2] == 0).all())
    r = l2_reference(x[~edge], torch.zeros_like(x[~edge]))
    _assert_within(y[~edge], r["y"], r["E_y"], f"C={C} ordinary rows")


# ----------------------------------------------------------------------------------------------- SGD
def sgd_call(p, g, b, first, cfg):
    """pcb_sgd_step in place on [n + 1] buffers whose last entry is the sentinel."""
    n = p.numel() - 1
    check(lib.pcb_sgd_step(ptr(p), ptr(g), ptr(b), n, float(cfg["lr"]), float(cfg["momentum"]), float(cfg["weight_decay"]),
                           float(cfg["grad_scale"]), int(first), float(cfg["dampening"]), stream()))
    torch.cuda.synchronize()
    assert _sent_ok(p) and _sent_ok(g) and _sent_ok(b), "pcb_sgd_step wrote past a buffer"


def _sgd_buffers(n, gen, pbound, gbound, grid):
    p, _ = _out(n)
    g, _ = _out(n)
    b, _ = _out(n)                                                  # NaN: the first step must not read it
    if grid:
        p[:n], g[:n] = X.sgd_grid(n, pbound, gen), X.sgd_grid(n, gbound, gen)
    else:
        p[:n] = torch.randn(n, generator=gen, device="cuda") * pbound
        g[:n] = torch.randn(n, generator=gen, device="cuda") * gbound
    return p, g, b


@pytest.mark.parametrize("n", X.SGD_N)
def test_sgd_bit_exact_on_grid_operands(n):
    """Three steps (first = 1, then 0) at every exact setting: p and buf bit for bit as the host restatement, from the state each step
    started from, on every element of the float4 body and of the scalar tail."""
    for ci, cfg in enumerate(X.SGD_EXACT):
        gen = torch.Generator(device="cuda").manual_seed(_seed("sgd exact", n, ci))
        p, g, b = _sgd_buffers(n, gen, 2.0, 1.0, True)
        for step in range(X.STEPS):
            first = step == 0
            p0, b0 = p[:n].clone(), b[:n].clone()
            cands = X.sgd_restate(p0, g[:n], b0, first, **cfg)
            sgd_call(p, g, b, first, cfg)
            match = torch.zeros(n, dtype=torch.bool, device="cuda")
            for pw, bw in cands:
                match |= (_bits(p[:n]) == _bits(pw)) & (_bits(b[:n]) == _bits(bw))
            if not bool(match.all()):
                i = int(torch.nonzero(~match)[0])
                raise AssertionError((n, cfg, step, i, float(p[i]), float(b[i]), [(float(pw[i]), float(bw[i])) for pw, bw in cands]))
            g[:n] = X.sgd_grid(n, 1.0, gen)


@pytest.mark.parametrize("n", X.SGD_N)
def test_sgd_within_fp64_bound(n):
    """Three steps at the trainers' settings on random operands: every element within the per-statement bound of fp64."""
    for ci, cfg in enumerate(X.SGD_REAL):
        gen = torch.Generator(device="cuda").manual_seed(_seed("sgd fp64", n, ci))
        p, g, b = _sgd_buffers(n, gen, 0.1, 0.01, False)
        f32 = lambda v: float(np.float32(v))
        lr, m, wd, gs = f32(cfg["lr"]), f32(cfg["momentum"]), f32(cfg["weight_decay"]), f32(cfg["grad_scale"])
        keep = float(np.float32(1) - np.float32(cfg["dampening"]))
        g3 = gamma(3)
        for step in range(X.STEPS):
            first = step == 0
            pd, gd, bd = p[:n].double(), g[:n].double(), b[:n].double()
            d = gd * gs + pd * wd
            E_d = g3 * ((gd * gs).abs() + (pd * wd).abs())
            if first:
                bw, E_b = d, E_d
            else:
                bw = bd * m + d * keep
                E_b = keep * E_d + g3 * ((bd * m).abs() + keep * (d.abs() + E_d))
            pw = pd - bw * lr
            E_p = lr * E_b + g3 * (pd.abs() + lr * (bw.abs() + E_b))
            sgd_call(p, g, b, first, cfg)
            what = f"n={n} {cfg} step {step}"
            _assert_within(b[:n], bw, E_b + REF * bw.abs(), what + " buf")
            _assert_within(p[:n], pw, E_p + REF * pw.abs(), what + " p")
            g[:n] = torch.randn(n, generator=gen, device="cuda") * 0.01


def test_flat_sgd_padding_stays_zero():
    """FlatSGD over parameters whose sizes are not multiples of 4: the padding of flat_param and flat_buf stays exactly 0 across steps and
    after load_state_dict, and every parameter follows the kernel's restatement."""
    from pointcontrast_b200 import optim
    shapes = [(3,), (5, 2), (7,), (1,), (2, 3, 3), (6,)]
    gen = torch.Generator(device="cuda").manual_seed(5)

    def params():
        return [torch.nn.Parameter((torch.randint(-512, 513, s, generator=gen, device="cuda") / 1024).float()) for s in shapes]

    cfg = X.SGD_EXACT[-1]
    kw = dict(lr=cfg["lr"], momentum=cfg["momentum"], weight_decay=cfg["weight_decay"], dampening=cfg["dampening"])

    def pad_mask(opt):
        m = torch.ones(opt.flat_param.numel(), dtype=torch.bool, device="cuda")
        for p, off in zip(opt.param_groups[0]["params"], opt._offsets):
            m[off:off + p.numel()] = False
        assert bool(m.any())
        return m

    def step(opt, ps):
        for p in ps:
            p.grad.copy_((torch.randint(-512, 513, p.shape, generator=gen, device="cuda") / 1024).float())
        opt.step()
        torch.cuda.synchronize()
        m = pad_mask(opt)
        assert not bool(opt.flat_param[m].any()) and not bool(opt.flat_buf[m].any()), "padding written"

    ps = params()
    opt = optim.FlatSGD(ps, **kw)
    opt.grad_scale = cfg["grad_scale"]
    assert any(p.numel() % 4 for p in ps)
    for _ in range(X.STEPS):
        before = opt.flat_param.clone(), opt.flat_buf.clone(), opt._first
        m = ~pad_mask(opt)
        step(opt, ps)
        cands = X.sgd_restate(before[0], opt.flat_grad, before[1], before[2], **cfg)
        ok = torch.zeros_like(m)
        for pw, bw in cands:
            ok |= (_bits(opt.flat_param) == _bits(pw)) & (_bits(opt.flat_buf) == _bits(bw))
        assert bool(ok[m].all())
    ps2 = params()
    opt2 = optim.FlatSGD(ps2, **kw)
    opt2.load_state_dict(opt.state_dict())
    assert not opt2._first
    m = pad_mask(opt2)
    assert not bool(opt2.flat_buf[m].any()) and not bool(opt2.flat_param[m].any())
    assert torch.equal(opt2.flat_buf[~m], opt.flat_buf[~m])
    step(opt2, ps2)


# ----------------------------------------------------------------------------------------------- gather-sum
def gs_call(Xf, tbl, kmap, K, n_out):
    """pcb_gather_sum on the operand in columns [4, 4 + C) of an ldx = C + 8 buffer (NaN around it) into columns [4, 4 + C) of an
    ldy = C + 12 buffer (NaN inside, the sentinel around it and in one more row), with counts.  -> (Y buffer, cnt buffer)"""
    from tests.test_gpu_conv_exact import _kmap_arg
    n_src, C = Xf.shape
    ldx, ldy = C + X.GS_XPAD, C + X.GS_YPAD
    xb = torch.full((n_src, ldx), NAN, device="cuda")
    xb[:, 4:4 + C] = Xf
    Y = torch.full((n_out + 1, ldy), SENT, device="cuda")
    Y[:n_out, 4:4 + C] = NAN
    cb, _ = _out(n_out)
    check(lib.pcb_gather_sum(xb.data_ptr() + 16, ldx, ptr(tbl), tbl.shape[1], _kmap_arg(kmap), K, n_out, C, Y.data_ptr() + 16, ldy,
                             ptr(cb), stream()))
    torch.cuda.synchronize()
    return Y, cb


def _check_gs(Xf, tbl, kmap, K, n_out, what):
    C = Xf.shape[1]
    Y, cb = gs_call(Xf, tbl, kmap, K, n_out)
    want, cnt = X.gs_restate(Xf, tbl, kmap, K, n_out)
    _assert_bits(Y[:n_out, 4:4 + C], want, what + " Y")
    _assert_bits(cb[:n_out], cnt, what + " cnt")
    frame = Y.clone()
    frame[:n_out, 4:4 + C] = SENT
    assert bool((frame == SENT).all()) and _sent_ok(cb), what + ": wrote outside its output"
    return cnt


@pytest.fixture(scope="module")
def stride2():
    """A stride-2 2x2x2 plan on a surface scene: (forward table, its source rows, transposed data-gradient table and kernel map)."""
    from pointcontrast_b200 import me
    from tests.helpers import surface_coords
    coords = surface_coords(np.random.default_rng(11), 3000)
    st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    cm, fine = st.coords_man, st.coords_key
    coarse = cm.stride(fine, [2, 2, 2])
    p = cm.conv_plan(fine, coarse, me.KernelGenerator([2, 2, 2], 2, 1, dimension=3), False)
    return p, cm.num_rows(fine), cm.num_rows(coarse)


@pytest.mark.parametrize("C", X.GS_C)
def test_gather_sum_bit_exact(C, stride2):
    """Integer features: Y and cnt exact on random tables (K = 1, 8, 27; rows without a neighbour) and on both tables of a stride-2
    plan, the input's padding columns NaN, the output's padding untouched."""
    from tests.test_gpu_conv_exact import _synth_table
    gen = torch.Generator(device="cuda").manual_seed(_seed("gather", C))
    for K in X.GS_K:
        n_out, n_src = 3001, 1500
        tbl = _synth_table(K, n_out, n_src, 0.6, gen)
        kmap = torch.randperm(K, generator=gen, device="cuda").tolist()
        for rows in (1, 9, n_out):
            cnt = _check_gs(X.gs_features(n_src, C, gen), tbl, kmap, K, rows, f"C={C} K={K} n_out={rows}")
        assert bool((cnt == 0).any()), "no row without a neighbour"
    p, nf, nc = stride2
    _check_gs(X.gs_features(nf, C, gen), p.fwd_tbl, p.fwd_kmap, p.K, p.n_out, f"C={C} stride-2 forward")
    cnt = _check_gs(X.gs_features(nc, C, gen), p.dg_tbl, p.dg_kmap, p.K, p.n_in, f"C={C} stride-2 transposed")
    assert bool((cnt == 1).all())


# ----------------------------------------------------------------------------------------------- reach
class _Rec:
    """A module's `lib` recording the calls of the four entry points."""

    def __init__(self, lib, rec):
        self._lib, self.r = lib, rec

    def __getattr__(self, k):
        return getattr(self._lib, k)

    def pcb_ce_forward_backward(self, x, t, n, C, ignore, gs, *a):
        self.r.add(("ce", C, X.ce_n_class(n), ignore, gs))
        return self._lib.pcb_ce_forward_backward(x, t, n, C, ignore, gs, *a)

    def pcb_l2norm_forward(self, x, n, C, *a):
        self.r.add(("l2norm", C, X.ce_n_class(n)))
        return self._lib.pcb_l2norm_forward(x, n, C, *a)

    def pcb_l2norm_backward(self, dy, y, inv, n, C, *a):
        self.r.add(("l2norm bwd", C, X.ce_n_class(n)))
        return self._lib.pcb_l2norm_backward(dy, y, inv, n, C, *a)

    def pcb_sgd_step(self, p, g, b, n, lr, m, wd, gs, first, dampening, st):
        self.r.add(("sgd", n % 4, round(dampening, 6)))
        return self._lib.pcb_sgd_step(p, g, b, n, lr, m, wd, gs, first, dampening, st)

    def pcb_gather_sum(self, x, ldx, tbl, ts, km, K, n, C, *a):
        self.r.add(("gather", C, K))
        return self._lib.pcb_gather_sum(x, ldx, tbl, ts, km, K, n, C, *a)


@pytest.fixture
def record(monkeypatch):
    from pointcontrast_b200 import losses, me, optim
    rec = set()
    for mod in (losses, optim, me):
        monkeypatch.setattr(mod, "lib", _Rec(mod.lib, rec))
    return rec


def _in_matrix(r):
    kind = r[0]
    if kind == "ce":
        return r[1] in X.CE_C and r[2] in {X.ce_n_class(n) for n in X.ce_n_list(r[1])}
    if kind.startswith("l2norm"):
        return r[1] in X.L2_C and r[2] in {X.ce_n_class(n) for n in X.l2_n_list(r[1])}
    if kind == "sgd":
        return r[1] in {n % 4 for n in X.SGD_N}
    return r[1] in X.GS_C and r[2] in X.GS_K


def test_training_steps_call_only_tested_cases(record):
    """One semseg finetune step of Res16UNet34C at 20 and 13 classes and one pretraining step: every call of the four entry points
    falls inside the case lists above."""
    from pointcontrast_b200 import losses, optim, semseg, synth
    from pointcontrast_b200.model import load_model
    from tests import refload
    from tests.helpers import det_init
    sc = synth.synth_scene(0, scale=0.12, voxel=0.05, n_raw=20_000)
    for C in (20, 13):
        mcfg = refload.default_config()
        mcfg["net"]["normalize_feature"] = False
        net = load_model("Res16UNet34C")(3, C, mcfg, D=3)
        det_init(net, 4)
        cfg = refload.Cfg(optimizer=dict(optimizer="SGD", lr=0.01, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=1,
                                         scheduler="PolyLR", max_iter=100, poly_power=0.9), data=dict(ignore_label=255))
        t = np.random.default_rng(C).integers(0, C, len(sc["coords"]))
        t[::7] = 255
        tr = semseg.SegmentationTrainer(net, cfg)
        tr.train_step([(torch.from_numpy(sc["coords"]), torch.from_numpy(sc["feats"]), torch.from_numpy(t))], shift_coords=False)
        torch.cuda.synchronize()
        assert {(r[0], r[1], r[3]) for r in record if r[0] == "ce"} >= {("ce", C, 255)}
        assert ("sgd", 0, 0.1) in record
    batch = synth.collate_pairs([synth.synth_pair(11, scale=0.12)])
    net = load_model("Res16UNet34C")(3, 32, refload.default_config(), D=3)
    det_init(net, 3)
    net = net.cuda().train()
    opt = optim.FlatSGD(net.parameters(), lr=0.1, momentum=0.8, weight_decay=1e-4)
    opt.zero_grad()
    F = net.forward_pair(torch.from_numpy(batch["sinput0_F"]), torch.from_numpy(batch["sinput0_C"]), torch.from_numpy(batch["sinput1_F"]),
                         torch.from_numpy(batch["sinput1_C"]), torch.device("cuda", torch.cuda.current_device()))
    n = min(F[0].shape[0], F[1].shape[0])
    idx = torch.arange(n, device="cuda")
    losses.point_nce_loss(F[0], F[1], idx, idx, 0.4).backward()
    opt.step()
    torch.cuda.synchronize()
    assert {r[:2] for r in record if r[0].startswith("l2norm")} == {("l2norm", 32), ("l2norm bwd", 32)}
    assert ("sgd", 0, 0.0) in record
    out = sorted(r for r in record if not _in_matrix(r))
    assert not out, f"calls outside the case lists: {out}"
