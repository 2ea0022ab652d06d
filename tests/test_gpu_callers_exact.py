"""The convolution and fused-unit kernels held to fp64 bit for bit at what the PointNet++ modules, the VoteNet heads and the one-view
Res16UNet callers issue (tests/exact_callers.py), with the harness and operand rules of tests/test_gpu_conv_exact.py and
tests/test_gpu_unit_exact.py: NaN around inputs, sentinels around outputs, a NaN-poisoned workspace.

  * Units: every signature outside the Res16UNet pair matrix -- K = 1 on the identity table (stride max(n, 65536), not n), one view,
    fp16 forward, the heads' 32 bias columns and column-slice gradients -- at the proposal head's rows (offset-split mode, statistics
    fused into the reduction over one segment) and the voting head's (direct mode); SA1's middle unit once over 2^20 rows; the one-view
    training units of the finetune and detection networks on the coordinate-manager scenes.
  * The direct split-convolution calls of the set-abstraction last layer, the heads' conv3 and the finetune / backbone final layers, and
    the heads' conv3 on their own operands: a bias row of hi = 1, lo = 0, zero-padded output columns, dW accumulated onto a base.
  * The exact fp32 calls of the set-abstraction layer 0 and the finetune final layers; SA1's relative-xyz weight gradient over 2^20 rows.
  * The head epilogue adjoints against a host restatement, bit for bit.
  * Reach: one training step and one eval forward of every caller, recording every struct and call, against exact_callers.
"""
import numpy as np
import pytest
import torch

from pointcontrast_b200._lib import CONV_ACCUMULATE, PLANES_A_FP16, PLANES_B_FP16, PcbStrided
from tests import exact_bn as XB
from tests import exact_callers as XK
from tests import exact_conv as XC
from tests import exact_unit as XU
from tests.test_gpu_conv_exact import (SENT, _assert_exact, _fp32_buffer, _full_operand, _out_buffer, _planes, _ref_forward,
                                       _run_conv_split, _run_wgrad_split, _weights_and_tiles, _ws)
from tests.test_gpu_unit_exact import (_Case, _check_backward, _check_forward, _mode, _paired_backward, _Recorder, _unpaired_backward,
                                       plans)  # noqa: F401  (plans: the coordinate-manager scenes fixture)

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _ident(n):
    from pointcontrast_b200 import pointnet2_modules
    return pointnet2_modules._identity(n, _dev())


class _IdentPlan:
    """The plan a K = 1 unit of the PointNet++ modules and the heads runs on: the identity table for all three roles, no kernel map,
    the weight gradient gathering x."""
    K, wg_gather_x, fwd_kmap, dg_kmap = 1, 1, None, None

    def __init__(self, n):
        self.n_in = self.n_out = n
        self.fwd_tbl = self.dg_tbl = self.wg_tbl = _ident(n)

    def c_kmap(self, name):
        return None


def _plan(plans, sig, size, rows=None):
    if sig.kind == "ident":
        return _IdentPlan(rows or XK.UNIT_ROWS[size])
    return plans[size][sig.kind]


def _is_head(sig):
    return sig.kind == "ident" and sig.out_str


def _with_bias(p, C, one):
    """p [n, C] and the 32 bias columns of the heads: column C holds `one`, the other 31 hold 0."""
    out = torch.cat([p, p.new_zeros(p.shape[0], 32)], 1)
    out[:, C] = one
    return out


def _bias_forward_operands(case):
    """A head unit's forward operands: exact_conv's fp16 rule on the first C columns (one nonzero fewer per row: room for the bias
    entry) and the bias column hi = 1, lo = 0 in both the fp16 and the bf16 planes."""
    base = type(case).forward_operands

    def operands():
        base(case)                                       # gamma, beta, running statistics; x is replaced below
        sig, fmt = case.sig, XC.FP16
        C = sig.Cin - 32
        hi, lo = XC.capped_planes(case.n_in, C, XC.row_cap(fmt, 1, sig.Cin) - 1, fmt.HI, fmt.LO, case.gen, "cuda")
        hi, lo = _with_bias(hi, C, 1.0), _with_bias(lo, C, 0.0)
        case.set("x_hi", hi)
        case.set("x_lo", lo)
        x = hi + lo
        bh = x.to(torch.bfloat16).float()
        case.set("x_bhi", bh)
        case.set("x_blo", x - bh)
        return hi.double(), lo.double()
    case.forward_operands = operands


def _bias_backward_operands(case, x):
    """The weight-gradient operand of a head unit with its bias columns (1, 0, ..., 0): dW's row C is the bias gradient."""
    C = case.sig.Cin - 32
    xh, xl = (t.float().clone() for t in x)
    xh[:, C:], xl[:, C:] = 0.0, 0.0
    xh[:, C] = 1.0
    case.set("x_bhi", xh)
    case.set("x_blo", xl)
    v = xh + xl
    fh = v.half().float()
    case.set("x_hi", fh)
    case.set("x_lo", v - fh)
    return xh.double(), xl.double()


# ----------------------------------------------------------------------------------------------- units
_SIGS, _TRAIN = XK.unit_signatures(), XK.training_signatures()


@pytest.mark.parametrize("sig", _SIGS, ids=[s.name() for s in _SIGS])
def test_caller_unit_forward_bit_exact(plans, sig):
    """z against fp64; the statistics (one segment, fused into the offset-split reduction or a separate pass, or eval's running
    statistics), out_p and every plane bit-identical to the BatchNorm primitives; both kernel modes."""
    for size in ("split", "direct"):
        plan = _plan(plans, sig, size)
        case = _Case(sig, plan, seed=XB.seed_of(f"{sig.name()} {size} caller fwd"))
        assert case.n0 == case.n_out
        if _is_head(sig):
            _bias_forward_operands(case)
        assert _mode(sig, plan) == size or (size == "split" and plan.K * (sig.Cin // XC.BK) < 2) or not sig.tc, (sig.name(), size)
        _check_forward(case, f"{sig.name()} {size} ({_mode(sig, plan)}) n_out={case.n_out} stride={plan.fwd_tbl.shape[1]}")


def _check_unit_backward(sig, plan, size, unpaired):
    case = _Case(sig, plan, seed=XB.seed_of(f"{sig.name()} {size} caller bwd"))
    what = f"{sig.name()} {size} n={case.n_out} stride={plan.fwd_tbl.shape[1]}"
    h, l, gm, x = _paired_backward(case)
    if _is_head(sig):
        x = _bias_backward_operands(case, x)
    base = case.snapshot()
    case.backward()
    _check_backward(case, h, l, gm, x, base, what)
    if unpaired:
        _unpaired_backward(case, what)


@pytest.mark.parametrize("sig", _TRAIN, ids=[s.name() for s in _TRAIN])
def test_caller_unit_backward_bit_exact(plans, sig):
    """dz, dW (the heads' bias row included), gin written or accumulated, dgamma / dbeta against fp64 at both sizes; then one unpaired
    call for the one-segment BatchNorm sums."""
    for size in ("split", "direct"):
        _check_unit_backward(sig, _plan(plans, sig, size), size, size == "split")


def test_sa1_middle_unit_over_2_20_rows():
    """SA1's 64 -> 64 unit at B = 8: 2^20 rows, forward and backward, once."""
    sig = XK.BIG_UNIT
    plan = _IdentPlan(XK.SA1_ROWS)
    assert XK.conv_mode(1, XK.SA1_ROWS, 64, 64, _sms()) == "direct"
    case = _Case(sig, plan, seed=XB.seed_of("sa1 2^20 fwd"))
    _check_forward(case, f"{sig.name()} n={XK.SA1_ROWS}")
    del case
    _check_unit_backward(sig, plan, "2^20", False)
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------- split convolutions
def _split_id(c):
    K, Ck, N, role, fmt, strided, acc = c
    return f"{Ck}x{N}-{role}-{fmt}" + "-strided" * strided + "-acc" * acc


@pytest.mark.parametrize("ci,case", list(enumerate(XK.split_cases())), ids=[_split_id(c) for c in XK.split_cases()])
def test_caller_split_conv_bit_exact(ci, case):
    """Each direct split-kernel call of the callers on the identity table at 1, 129, the proposal head's and the voting head's rows:
    offset-split and direct mode as the tile rules give them; the forward role with and without a bias."""
    K, Ck, N, role, fname, strided, acc = case
    gen = torch.Generator(device="cuda").manual_seed(3000 + ci)
    if role != "wgrad":
        fmt = XC.FMTS[fname]
        Cin, Cout = (Ck, N) if role == "fwd" else (N, Ck)
        ft, dt, wh, wl = _weights_and_tiles(K, Cin, Cout, fmt, gen)
        tiles = ft if role == "fwd" else dt
        if role == "dgrad":
            wh, wl = wh.transpose(1, 2).contiguous(), wl.transpose(1, 2).contiguous()
    modes = set()
    for i, n in enumerate(XK.SPLIT_ROWS):
        tbl = _ident(n)
        what = f"{_split_id(case)} rows={n} stride={tbl.shape[1]}"
        if role == "wgrad":
            _run_wgrad_split(K, Ck, N, 0, tbl, n, n, strided, acc, gen, what)
            continue
        bias = XC.bias_values(N, fmt, gen, "cuda") if role == "fwd" and i % 2 else None
        base = XC.bias_values(n * N, fmt, gen, "cuda").view(n, N) if acc else None
        nsplit = _run_conv_split(fmt, K, Ck, N, tiles, wh, wl, tbl, n, None, n, strided, bias, base, gen, what)
        mode = "direct" if nsplit == 1 else "split"
        assert mode == XK.conv_mode(K, n, Ck, N, _sms()), what
        modes.add(mode)
    assert role == "wgrad" or modes == {"split", "direct"}, (case, modes)


_CONV3 = sorted({(c[1], c[2]) for c in XK.split_cases() if c[3] == "fwd" and XK.head_padding(c[1], c[2])})


@pytest.mark.parametrize("Ck,N", _CONV3, ids=[f"{a}x{b}" for a, b in _CONV3])
def test_head_conv3_bias_row_and_padded_columns(Ck, N):
    """A head's conv3 on its own operands: the input's bias column (hi = 1, lo = 0, then 31 zero columns), weights whose padded output
    columns are 0 -- z must hold exactly 0 there -- and the weight gradient of a dz whose padded columns are 0, accumulated onto a
    nonzero base: dW - base must be exactly 0 in those columns and in the 31 zero input rows."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    C, X = XK.head_padding(Ck, N)
    gen = torch.Generator(device="cuda").manual_seed(Ck * 1000 + N)
    f = XC.FP16
    W = XC.weights(1, Ck, N, f, gen, "cuda")[0]
    W[:, C + 1:, :] = 0.0
    W[:, :, X:] = 0.0
    ft = torch.empty(lib.pcb_weight_tile_bytes(1, Ck, N, 0), dtype=torch.uint8, device="cuda")
    dt = torch.empty(lib.pcb_weight_tile_bytes(1, Ck, N, 1), dtype=torch.uint8, device="cuda")
    check(lib.pcb_weight_tile(ptr(W), 1, Ck, N, ptr(ft), ptr(dt), PLANES_B_FP16, stream()))
    wh, wl = (t.double() for t in XC.split_weights(W, f))
    for n in (XK.PROPOSAL_ROWS, XK.VOTE_ROWS):
        tbl = _ident(n)
        what = f"conv3 {Ck}x{N} (X={X}) rows={n}"
        hi, lo = XC.capped_planes(n, C, XC.row_cap(f, 1, Ck) - 1, f.HI, f.LO, gen, "cuda")
        hi, lo = _with_bias(hi, C, 1.0), _with_bias(lo, C, 0.0)
        xh, xl, _, _ = _planes(hi, lo, f.dtype, False)
        Y, _, _ = _out_buffer(n, N, False)
        wsb = lib.pcb_conv_forward_split_ws_bytes(1, n, Ck, N)
        ws = _ws(wsb)
        check(lib.pcb_conv_forward_split(ptr(xh), ptr(xl), Ck, ptr(tbl), tbl.shape[1], None, 1, n, Ck, N, ptr(ft), None, ptr(Y), N, ptr(ws),
                                         wsb, PLANES_A_FP16 | PLANES_B_FP16, stream()))
        y, a = _ref_forward(hi.double(), lo.double(), wh, wl, tbl, None, n)
        assert float(a.max()) * f.SCALE < XC.LIMIT * f.Q, what
        _assert_exact(Y[:n], y * f.SCALE, what + " z")
        assert bool((Y[:n, X:] == 0).all()), what + ": padded z columns not 0"
        # weight gradient: A = the activation's bf16 planes with the bias columns, B = dz with zero padded columns
        b = XC.BF16
        Ah, Al = XC.dense_planes(n, C, XC.WG_A_DENSITY, b.HI, b.LO, gen, "cuda")
        Ah, Al = _with_bias(Ah, C, 1.0), _with_bias(Al, C, 0.0)
        Bh, Bl = (p.t() for p in XC.capped_planes(N, n, min(n, XC.wgrad_col_cap()), b.HI, b.LO, gen, "cuda"))
        Bh, Bl = Bh.contiguous(), Bl.contiguous()
        Bh[:, X:], Bl[:, X:] = 0.0, 0.0
        ah, al = Ah.to(torch.bfloat16), Al.to(torch.bfloat16)
        bh, bl = Bh.to(torch.bfloat16), Bl.to(torch.bfloat16)
        base = XC.bias_values(Ck * N, b, gen, "cuda").view(Ck, N)
        buf = torch.full((Ck * N + 128,), SENT, device="cuda")
        buf[64:64 + Ck * N] = base.reshape(-1)
        wsb = lib.pcb_conv_wgrad_split_ws_bytes(1, n, Ck, N)
        ws = _ws(wsb)
        check(lib.pcb_conv_wgrad_split(ptr(ah), ptr(al), Ck, ptr(bh), ptr(bl), N, ptr(tbl), tbl.shape[1], 1, n, Ck, N, buf.data_ptr() + 4 * 64,
                                       0, ptr(ws), wsb, CONV_ACCUMULATE, stream()))
        Ad, Ald, Bd, Bld = Ah.double(), Al.double(), Bh.double(), Bl.double()
        want = base.double() + Ald.t() @ Bd + Ad.t() @ Bld + Ad.t() @ Bd
        bound = base.double().abs() + Ald.abs().t() @ Bd.abs() + Ad.abs().t() @ Bld.abs() + Ad.abs().t() @ Bd.abs()
        assert float(bound.max()) < XC.LIMIT * XC.WG_Q, what
        dW = buf[64:64 + Ck * N].view(Ck, N)
        _assert_exact(dW, want, what + " dW")
        assert bool((dW[:, X:] == base[:, X:]).all() and (dW[C + 1:] == base[C + 1:]).all()), what + ": padded dW not 0"
        assert bool((buf[:64] == SENT).all() and (buf[64 + Ck * N:] == SENT).all()), what + ": memory around dW overwritten"


# ----------------------------------------------------------------------------------------------- exact fp32 kernels
@pytest.mark.parametrize("K,Cin,Cout", XK.exact_forward_cases())
def test_caller_exact_fp32_forward_bit_exact(K, Cin, Cout):
    """pcb_conv_forward on the identity table: set-abstraction layer 0 (Cin = 1, the 3-column relative-xyz data gradient, feature
    columns) and the finetune final layers, at 1, 129 and 4097 rows; column slices and bias alternate."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    gen = torch.Generator(device="cuda").manual_seed(K + Cin * 7 + Cout)
    W = XC.weights(K, Cin, Cout, XC.BF16, gen, "cuda")[1].contiguous()
    for i, n in enumerate(XK.EXACT_ROWS):
        tbl = _ident(n)
        Xf = _full_operand(n, Cin, gen)
        strided, use_bias = i > 0, i != 1
        xb, c0, ldx = _fp32_buffer(Xf, strided)
        Y, y0, ldy = _out_buffer(n, Cout, strided)
        bias = XC.bias_values(Cout, XC.BF16, gen, "cuda") if use_bias else None
        check(lib.pcb_conv_forward(xb.data_ptr() + 4 * c0, ldx, ptr(tbl), tbl.shape[1], None, K, n, Cin, Cout, ptr(W), ptr(bias),
                                   Y.data_ptr() + 4 * y0, ldy, stream()))
        want, bound = Xf.double() @ W[0].double(), Xf.double().abs() @ W[0].double().abs()
        if bias is not None:
            want, bound = want + bias.double(), bound + bias.double().abs()
        what = f"K={K} {Cin}x{Cout} n={n} strided={strided} bias={use_bias}"
        assert float(bound.max()) < XC.LIMIT * XC.EXACT_Q, what
        _assert_exact(Y[:n, y0:y0 + Cout], want, what)
        pad = Y.clone()
        pad[:n, y0:y0 + Cout] = SENT
        assert bool((pad == SENT).all()), what + ": output padding overwritten"


def _exact_wgrad(K, Ca, Cb, tr, flags, n, strided, gen, what):
    from pointcontrast_b200._lib import check, lib, ptr, stream
    tbl = _ident(n)
    Af = _full_operand(n, Ca, gen)
    B = XC.capped_planes(Cb, n, min(n, XC.exact_wgrad_col_cap()), XC.BF16.HI, XC.BF16.LO, gen, "cuda")[0].t().contiguous()
    shape = (K, Cb, Ca) if tr else (K, Ca, Cb)
    nW = K * Ca * Cb
    ab, a0, lda = _fp32_buffer(Af, strided)
    bb, b0, ldb = _fp32_buffer(B, strided, c0=8, extra=13)
    buf = torch.full((nW + 128,), SENT, device="cuda")
    base = XC.bias_values(nW, XC.BF16, gen, "cuda").view(shape) if flags & 4 else None
    if base is not None:
        buf[64:64 + nW] = base.reshape(-1)
    wsb = lib.pcb_conv_wgrad_ws_bytes(K, n, Ca, Cb)
    ws = _ws(wsb)
    check(lib.pcb_conv_wgrad(ab.data_ptr() + 4 * a0, lda, bb.data_ptr() + 4 * b0, ldb, ptr(tbl), tbl.shape[1], K, n, Ca, Cb,
                             buf.data_ptr() + 4 * 64, tr, ptr(ws), wsb, flags, stream()))
    d, e = Af.double().t() @ B.double(), Af.double().abs().t() @ B.double().abs()
    want, bound = (d.t(), e.t()) if tr else (d, e)
    want, bound = want.reshape(shape), bound.reshape(shape)
    if base is not None:
        want, bound = want + base.double(), bound + base.double().abs()
    assert float(bound.max()) < XC.LIMIT * XC.EXACT_Q, what
    _assert_exact(buf[64:64 + nW].view(shape), want, what)
    assert bool((buf[:64] == SENT).all() and (buf[64 + nW:] == SENT).all()), f"{what}: memory around dW overwritten"


@pytest.mark.parametrize("K,Ca,Cb,tr,flags", XK.exact_wgrad_cases())
def test_caller_exact_fp32_wgrad_bit_exact(K, Ca, Cb, tr, flags):
    """pcb_conv_wgrad on the identity table: layer 0's relative-xyz (Ca = 3) and feature-column weight gradients (transposed output)
    and the finetune final layers (accumulated), at 1, 129 and 4097 rows."""
    gen = torch.Generator(device="cuda").manual_seed(K + Ca * 7 + Cb + tr + flags)
    for i, n in enumerate(XK.EXACT_ROWS):
        _exact_wgrad(K, Ca, Cb, tr, flags, n, i > 0, gen, f"K={K} {Ca}x{Cb} tr={tr} flags={flags} n={n}")


def test_sa1_relative_xyz_wgrad_over_2_20_rows():
    """SA1's relative-xyz weight gradient (Ca = 3, transposed output) at B = 8: 2^20 rows, once."""
    gen = torch.Generator(device="cuda").manual_seed(20)
    _exact_wgrad(*XK.BIG_EXACT_WGRAD, XK.SA1_ROWS, False, gen, f"{XK.BIG_EXACT_WGRAD} n={XK.SA1_ROWS}")


# ----------------------------------------------------------------------------------------------- epilogue adjoints
def _split_bf16(v):
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def _assert_bits16(got_i16, want_bf16, what):
    assert bool((got_i16 == want_bf16.view(torch.int16)).all()), what


def _strided_arg(t):
    from pointcontrast_b200 import det_heads
    return det_heads._strided(t)


@pytest.mark.parametrize("V", XK.VOTE_FACTORS)
@pytest.mark.parametrize("absent", ("none", "xyz", "features"))
def test_vote_epilogue_grad_bit_exact(V, absent):
    """pcb_vote_epilogue_grad on strided gradients (d_vote_features channel-major as the caller's view gives them, d_vote_xyz a column
    slice) or an absent one: dz hi / lo are bf16 round-to-nearest-even of the gradient and of its residual, the padding columns 0;
    d_seed_features and d_seed_xyz the fp32 sums over v in ascending order, nothing written beyond them."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    B, S, C = 2, 37, XK.SEED_DIM
    W, cpad = 3 + C, -(-(3 + C) * V // 32) * 32
    ldz = cpad + 8
    gen = torch.Generator(device="cuda").manual_seed(V * 10 + len(absent))
    gx = torch.randn(B, S * V, 7, generator=gen, device="cuda")[:, :, 2:5]
    gf = torch.randn(B, C, S * V, generator=gen, device="cuda").transpose(1, 2)
    gx = None if absent == "xyz" else gx
    gf = None if absent == "features" else gf
    n = B * S
    dz = torch.full((2, n + 1, ldz), 0x5A5A, dtype=torch.int16, device="cuda")
    dsf = torch.full((n + 1, C + 32), SENT, device="cuda")
    dsx = torch.full((B * S * 3 + 16,), SENT, device="cuda")
    check(lib.pcb_vote_epilogue_grad(_strided_arg(gx), _strided_arg(gf), B, S, V, C, dz[0].data_ptr(), dz[1].data_ptr(), ldz, cpad,
                                     dsf.data_ptr(), C + 32, dsx.data_ptr(), stream()))
    torch.cuda.synchronize()
    zx = torch.zeros(B, S * V, 3, device="cuda") if gx is None else gx
    zf = torch.zeros(B, S * V, C, device="cuda") if gf is None else gf
    v = torch.zeros(n, cpad, device="cuda")
    per = torch.cat([zx, zf], 2).reshape(B, S, V, W)
    v[:, :V * W] = per.reshape(n, V * W)
    hi, lo = _split_bf16(v)
    what = f"V={V} absent={absent}"
    _assert_bits16(dz[0, :n, :cpad], hi, what + " dz_hi")
    _assert_bits16(dz[1, :n, :cpad], lo, what + " dz_lo")
    assert bool((dz[:, :n, cpad:] == 0x5A5A).all() and (dz[:, n] == 0x5A5A).all()), what + ": dz frame written"
    assert bool((v[:, V * W:] == 0).all())
    sf, sx = torch.zeros(n, C, device="cuda"), torch.zeros(n, 3, device="cuda")
    for k in range(V):                          # ascending v, fp32 adds
        sf = sf + zf.reshape(B, S, V, C)[:, :, k].reshape(n, C)
        sx = sx + zx.reshape(B, S, V, 3)[:, :, k].reshape(n, 3)
    assert bool((dsf[:n, :C].view(torch.int32) == sf.view(torch.int32)).all()), what + " d_seed_features"
    assert bool((dsf[:n, C:] == SENT).all() and (dsf[n] == SENT).all()), what + ": d_seed_features frame written"
    assert bool((dsx[:n * 3].view(torch.int32) == sx.reshape(-1).view(torch.int32)).all()), what + " d_seed_xyz"
    assert bool((dsx[n * 3:] == SENT).all()), what + ": d_seed_xyz frame written"


@pytest.mark.parametrize("dataset", XK.DATASETS)
def test_proposal_epilogue_grad_bit_exact(dataset):
    """pcb_proposal_epilogue_grad on the nine end_point gradients -- strided views of one [B, K, Xpad] buffer as decode_scores'
    outputs are views of z, contiguous ones, and an absent one -- in both output forms: bf16 hi / lo planes (the head) and fp32 dz
    (stand-alone decode_scores).  Every column is the gradient of the view that reads it, plus unit x heading_residuals' / mean_size x
    size_residuals' on the residual columns (fp32 multiply, then add); padding 0; d_aggregated_vote_xyz the center gradient."""
    from pointcontrast_b200 import det_heads
    from pointcontrast_b200._lib import check, lib, stream
    NC, NH, NS = XK.DATASETS[dataset]
    B, K = 2, 37
    dec = det_heads._Decode(NC, NH, NS, np.linspace(0.25, 3.0, 3 * NS, dtype=np.float32).reshape(NS, 3))
    X, Xpad = dec.X, -(-dec.X // 32) * 32
    gen = torch.Generator(device="cuda").manual_seed(NH * 100 + NS)
    r = lambda *s: torch.randn(*s, generator=gen, device="cuda")
    zg = r(B, K, Xpad)                                   # the views read their columns of one wider buffer
    s0, c0 = 5 + 2 * NH, 5 + 2 * NH + 4 * NS
    grads = [zg[:, :, 0:2], r(B, K, 3), zg[:, :, 5:5 + NH], None, r(B, NH, K).transpose(1, 2), zg[:, :, s0:s0 + NS],
             zg[:, :, s0 + NS:c0].view(B, K, NS, 3), r(B, K, NS, 3), zg[:, :, c0:X]]
    if dataset == "sunrgbd":
        grads[3], grads[1] = r(B, K, NH), None           # the other head gives heading_residuals_normalized and no center gradient
    z = lambda i, *s: torch.zeros(B, K, *s, device="cuda") if grads[i] is None else grads[i]
    unit = torch.tensor(dec.unit, dtype=torch.float32, device="cuda")
    ms = torch.from_numpy(dec.ms).cuda()
    want = torch.zeros(B, K, Xpad, device="cuda")
    want[:, :, 0:2] = z(0, 2)
    want[:, :, 2:5] = z(1, 3)
    want[:, :, 5:5 + NH] = z(2, NH)
    want[:, :, 5 + NH:s0] = z(3, NH) + z(4, NH) * unit
    want[:, :, s0:s0 + NS] = z(5, NS)
    want[:, :, s0 + NS:c0] = (z(6, NS, 3) + z(7, NS, 3) * ms).reshape(B, K, 3 * NS)
    want[:, :, c0:X] = z(8, NC)
    want = want.reshape(B * K, Xpad)
    for planes in (True, False):
        what = f"{dataset} planes={planes}"
        d_agg = torch.full((B * K * 3 + 16,), SENT, device="cuda")
        ldz = Xpad + 8
        arr = (PcbStrided * 9)()
        for i, g in enumerate(grads):
            if g is not None:
                arr[i] = PcbStrided(g.data_ptr(), *(list(g.stride()) + [0] * (4 - g.dim())))
        if planes:
            dz = torch.full((2, B * K + 1, ldz), 0x5A5A, dtype=torch.int16, device="cuda")
            args = (dz[0].data_ptr(), dz[1].data_ptr(), None)
        else:
            dz = torch.full((B * K + 1, ldz), SENT, device="cuda")
            args = (None, None, dz.data_ptr())
        check(lib.pcb_proposal_epilogue_grad(arr, B, K, NH, NS, NC, dec.unit, dec.ms.ctypes.data, *args, ldz, Xpad, d_agg.data_ptr(),
                                             stream()))
        torch.cuda.synchronize()
        n = B * K
        if planes:
            hi, lo = _split_bf16(want)
            _assert_bits16(dz[0, :n, :Xpad], hi, what + " dz_hi")
            _assert_bits16(dz[1, :n, :Xpad], lo, what + " dz_lo")
            assert bool((dz[:, :n, Xpad:] == 0x5A5A).all() and (dz[:, n] == 0x5A5A).all()), what + ": dz frame written"
        else:
            assert bool((dz[:n, :Xpad].view(torch.int32) == want.view(torch.int32)).all()), what + " dz"
            assert bool((dz[:n, Xpad:] == SENT).all() and (dz[n] == SENT).all()), what + ": dz frame written"
        assert bool((want[:, X:] == 0).all())
        assert bool((d_agg[:n * 3].view(torch.int32) == z(1, 3).reshape(-1).contiguous().view(torch.int32)).all()), what + " d_agg"
        assert bool((d_agg[n * 3:] == SENT).all()), what + ": d_aggregated_vote_xyz frame written"


# ----------------------------------------------------------------------------------------------- reach
class _CallRecorder(_Recorder):
    """A module's `lib` recording every unit struct (kind "ident" on pointnet2_modules' identity table) and every convolution call of
    exact_callers' four kinds into one shared Calls-like record."""

    def __init__(self, lib, rec):
        super().__init__(lib)
        self.r = rec

    def _ident_sig(self, u, backward):
        from pointcontrast_b200 import pointnet2_modules
        s = self.sig(u, backward)
        t = pointnet2_modules._IDENT.get(torch.cuda.current_device())
        return s._replace(kind="ident") if t is not None and u.fwd_tbl == t.data_ptr() else s

    def pcb_unit_forward(self, ref, st):
        s = self._ident_sig(ref._obj, False)
        self.r["fwd_eval" if s.eval else "fwd"].add(s)
        return self._lib.pcb_unit_forward(ref, st)

    def pcb_unit_backward(self, ref, st):
        self.r["bwd"].add(self._ident_sig(ref._obj, True))
        return self._lib.pcb_unit_backward(ref, st)

    def _split(self, K, Ck, N, lds, ldy, flags):
        fp16 = bool(flags & PLANES_A_FP16)
        self.r["split"].add((K, Ck, N, "fwd" if fp16 else "dgrad", "fp16" if fp16 else "bf16", lds != Ck or ldy != N,
                             bool(flags & CONV_ACCUMULATE)))

    def pcb_conv_forward_split(self, xh, xl, lds, tbl, ts, km, K, n, Ck, N, tiles, bias, y, ldy, ws, wsb, flags, st):
        self._split(K, Ck, N, lds, ldy, flags)
        return self._lib.pcb_conv_forward_split(xh, xl, lds, tbl, ts, km, K, n, Ck, N, tiles, bias, y, ldy, ws, wsb, flags, st)

    def pcb_conv_forward_split_ordered(self, xh, xl, lds, tbl, ts, km, K, perm, n, Ck, N, tiles, bias, y, ldy, ws, wsb, flags, st):
        self._split(K, Ck, N, lds, ldy, flags)
        return self._lib.pcb_conv_forward_split_ordered(xh, xl, lds, tbl, ts, km, K, perm, n, Ck, N, tiles, bias, y, ldy, ws, wsb, flags, st)

    def pcb_conv_wgrad_split(self, ah, al, lda, bh, bl, ldb, tbl, ts, K, n, Ca, Cb, dw, tr, ws, wsb, flags, st):
        self.r["split"].add((K, Ca, Cb, "wgrad", "bf16", lda != Ca or ldb != Cb, bool(flags & CONV_ACCUMULATE)))
        return self._lib.pcb_conv_wgrad_split(ah, al, lda, bh, bl, ldb, tbl, ts, K, n, Ca, Cb, dw, tr, ws, wsb, flags, st)

    def pcb_conv_forward(self, x, ldx, tbl, ts, km, K, n, Cin, Cout, w, bias, y, ldy, st):
        self.r["exact_fwd"].add((K, Cin, Cout))
        return self._lib.pcb_conv_forward(x, ldx, tbl, ts, km, K, n, Cin, Cout, w, bias, y, ldy, st)

    def pcb_conv_wgrad(self, a, lda, b, ldb, tbl, ts, K, n, Ca, Cb, dw, tr, ws, wsb, flags, st):
        self.r["exact_wgrad"].add((K, Ca, Cb, tr, flags))
        return self._lib.pcb_conv_wgrad(a, lda, b, ldb, tbl, ts, K, n, Ca, Cb, dw, tr, ws, wsb, flags, st)


@pytest.fixture
def record(monkeypatch):
    """Patch `lib` in every module that issues the recorded calls (each binds its own); returns the record."""
    from pointcontrast_b200 import det_heads, fused, me, pointnet2_modules
    rec = {k: set() for k in ("fwd", "fwd_eval", "bwd", "split", "exact_fwd", "exact_wgrad")}
    for mod in (fused, pointnet2_modules, det_heads, me):
        monkeypatch.setattr(mod, "lib", _CallRecorder(mod.lib, rec))
    monkeypatch.setattr(me, "FWD_FP16", True)
    return rec


def _cloud(gen, B, N):
    return torch.rand(B, N, 3, generator=gen, device="cuda") * 4.0


def _run_caller(caller, train, gen):
    """One small training step (forward + backward of a random projection of every output) or one eval forward of a caller."""
    from pointcontrast_b200 import det_heads, me, pointnet2_modules
    kind, _, arg = caller.partition(":")
    torch.manual_seed(7)
    grad = torch.enable_grad() if train else torch.no_grad()
    with grad:
        if kind == "sa":
            npoint, radius, nsample, mlp = XK.SA[arg]
            m = pointnet2_modules.PointnetSAModuleVotes(npoint=npoint, radius=radius, nsample=nsample, mlp=list(mlp), use_xyz=True,
                                                        normalize_xyz=True).cuda().train(train)
            xyz = _cloud(gen, 1, max(2 * npoint, 1024)).requires_grad_(train)
            f = torch.randn(1, mlp[0], xyz.shape[1], generator=gen, device="cuda").requires_grad_(train) if mlp[0] else None
            outs = m(xyz, f)[:2]
        elif kind == "fp":
            m = pointnet2_modules.PointnetFPModule(mlp=list(XK.FP)).cuda().train(train)
            unknown, known = _cloud(gen, 1, 512), _cloud(gen, 1, 256)
            uf = torch.randn(1, XK.FP[0] - 256, 512, generator=gen, device="cuda").requires_grad_(train)
            kf = torch.randn(1, 256, 256, generator=gen, device="cuda").requires_grad_(train)
            outs = [m(unknown, known, uf, kf)]
        elif kind == "vote":
            m = det_heads.VotingModule(int(arg), XK.SEED_DIM).cuda().train(train)
            xyz = _cloud(gen, 2, 64).requires_grad_(train)
            f = torch.randn(2, XK.SEED_DIM, 64, generator=gen, device="cuda").requires_grad_(train)
            outs = list(m(xyz, f))
        elif kind == "proposal":
            NC, NH, NS = XK.DATASETS[arg]
            m = det_heads.ProposalModule(NC, NH, NS, np.ones((NS, 3), dtype=np.float32), XK.NUM_PROPOSAL, "vote_fps",
                                         seed_feat_dim=XK.SEED_DIM).cuda().train(train)
            xyz = _cloud(gen, 2, 2 * XK.NUM_PROPOSAL).requires_grad_(train)
            f = torch.randn(2, XK.SEED_DIM, xyz.shape[1], generator=gen, device="cuda").requires_grad_(train)
            ep = m(xyz, f, {})
            outs = [ep[k] for k in det_heads.DECODE]
        else:
            from tests.helpers import surface_coords
            net = _res16unet(int(arg)).train(train)
            coords = torch.from_numpy(surface_coords(np.random.default_rng(3), 1500))
            st = me.SparseTensor(torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(1)), coords=coords).to("cuda")
            outs = [net(st).F]
        if train:
            loss = sum((o * torch.randn(o.shape, generator=gen, device="cuda")).sum() for o in outs)
            loss.backward()
    torch.cuda.synchronize()


def _res16unet(out):
    from pointcontrast_b200 import detection
    from pointcontrast_b200.model import load_model
    from tests.helpers import det_init
    from tests.refload import default_config
    net = detection.SparseConvBackbone(3, out).net if out == XK.BACKBONE_OUT else load_model("Res16UNet34C")(3, out, default_config(), D=3)
    det_init(net, 1)
    return net.cuda()


@pytest.mark.parametrize("caller", XK.CALLERS)
def test_every_caller_call_is_restated_and_in_the_matrix(record, caller):
    """One training step and one eval forward of the caller: every unit struct and convolution call it issues is a case of the bit-exact
    suites, and the recorded set equals what exact_callers restates -- so the restatement is neither incomplete nor stale."""
    gen = torch.Generator(device="cuda").manual_seed(XB.seed_of(caller))
    _run_caller(caller, True, gen)
    train = {k: set(v) for k, v in record.items()}
    for v in record.values():
        v.clear()
    _run_caller(caller, False, gen)
    ev = record
    matrix_units = set(XU.signatures()) | set(XK.unit_signatures())
    fwd_matrix = {XU.forward_part(s) for s in matrix_units}
    got = train["bwd"] | ev["fwd_eval"]
    missing = sorted(s.name() for s in got if s not in matrix_units) + sorted(s.name() for s in train["fwd"] if s not in fwd_matrix)
    assert not missing, f"{caller}: unit signatures outside the case matrix: {missing}"
    assert not ev["fwd"] and not ev["bwd"] and not train["fwd_eval"], caller
    for k, cases in (("split", set(XK.split_cases())), ("exact_fwd", set(XK.exact_forward_cases())),
                     ("exact_wgrad", set(XK.exact_wgrad_cases()))):
        out = sorted((train[k] | ev[k]) - cases)
        assert not out, f"{caller}: {k} calls outside the case lists: {out}"
    want_t, want_e = XK.caller_calls(caller, True), XK.caller_calls(caller, False)
    assert train["bwd"] == set(want_t.units), (caller, sorted(s.name() for s in train["bwd"] ^ set(want_t.units)))
    assert train["fwd"] == {XU.forward_part(s) for s in want_t.units}, caller
    assert ev["fwd_eval"] == set(want_e.units), (caller, sorted(s.name() for s in ev["fwd_eval"] ^ set(want_e.units)))
    for k in ("split", "exact_fwd", "exact_wgrad"):
        assert train[k] == set(getattr(want_t, k)), (caller, k, sorted(train[k] ^ set(getattr(want_t, k))))
        assert ev[k] == set(getattr(want_e, k)), (caller, "eval", k, sorted(ev[k] ^ set(getattr(want_e, k))))

