"""The sparse-convolution kernels held to an fp64 reference BIT FOR BIT, on operands that make every kernel exact (tests/exact_conv.py):
each product is a multiple of one quantum q and each output's terms sum, in absolute value, to less than 2^20 q, so no summation order
can round.  A misplaced, missing or duplicated term, a wrong plane, a skipped split or an unwritten row then changes the result, where a
norm-relative tolerance on random data lets through errors of a low-order term.

Covered: `pcb_conv_forward_split` (forward and data-gradient roles, bf16 and fp16 operands) at every convolution shape of Res16UNet14/18/34/34C
and at extra widths, so that every column tile runs with one and with several blocks; offset-split and direct mode; coordinate-manager and
synthetic tables, rows without neighbours, tiles with one or no offset (empty z-slices), table padding holding valid row indices; the
three kinds of kernel map; column slices of wider buffers (NaN around the input slice, a sentinel around the output); bias and
accumulation.  `pcb_conv_wgrad_split` at every last-M-block size, both output layouts, empty row splits, accumulation and no rows.  The exact
fp32 kernels (`pcb_conv_forward`, `pcb_conv_wgrad`, `pcb_gather_sum`) on the same tables.  And the fused executor on Res16UNet14, whose
decoder widths (384, 320, 288) no other model test runs.
"""
import numpy as np
import pytest
import torch

from tests import exact_conv as X
from tests.helpers import surface_coords

pytestmark = pytest.mark.gpu
SENT = -7777.25          # output-padding sentinel


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope="module")
def scene():
    """Neighbour tables of one surface scene from the coordinate manager: hybrid 3x3x3, stride-2 2x2x2 (down and up) and 1x1x1."""
    from pointcontrast_b200 import me
    coords = surface_coords(np.random.default_rng(5), 3000)
    st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    cm, fine = st.coords_man, st.coords_key
    coarse = cm.stride(fine, [2, 2, 2])
    hyb = me.KernelGenerator(3, 1, 1, region_type=me.RegionType.HYBRID, axis_types=[me.RegionType.HYPERCUBE] * 3, dimension=3)
    p27 = cm.conv_plan(fine, fine, hyb, False)
    p8 = cm.conv_plan(fine, coarse, me.KernelGenerator([2, 2, 2], 2, 1, dimension=3), False)
    p1 = cm.conv_plan(fine, fine, me.KernelGenerator(1, 1, 1, dimension=3), False)
    nf, nc = cm.num_rows(fine), cm.num_rows(coarse)
    assert min(nf, nc) > max(X.SPLIT_ROWS + X.WGRAD_ROWS)
    # (kind, role) -> (table, rows its entries index, kernel map); a transposed convolution's forward role is the down-convolution's
    # data-gradient role and vice versa
    fwd = {("k27", "fwd"): (p27.fwd_tbl, nf, None), ("k27", "dgrad"): (p27.dg_tbl, nf, p27.dg_kmap),
           ("down", "fwd"): (p8.fwd_tbl, nf, None), ("down", "dgrad"): (p8.dg_tbl, nc, None),
           ("up", "fwd"): (p8.dg_tbl, nc, None), ("up", "dgrad"): (p8.fwd_tbl, nf, None),
           ("k1", "fwd"): (p1.fwd_tbl, nf, None), ("k1", "dgrad"): (p1.dg_tbl, nf, p1.dg_kmap)}
    return dict(fwd=fwd, wg={27: (p27.wg_tbl, nf), 8: (p8.wg_tbl, nf), 1: (p1.wg_tbl, nf)})


def _synth_table(K, n_out, n_src, density, gen, pad=45):
    """Random table [K, n_out + pad]: an entry present with probability `density`, every 7th row without any neighbour, and valid row
    indices in the padding beyond n_out (a kernel that read them would change its result)."""
    t = torch.randint(0, n_src, (K, n_out + pad), generator=gen, device="cuda", dtype=torch.int32)
    drop = torch.rand(K, n_out, generator=gen, device="cuda") >= density
    drop[:, ::7] = True
    t[:, :n_out][drop] = -1
    return t


def _gather(A, t):
    """Rows t of A (fp64), zero where t < 0."""
    Z = torch.cat([A, A.new_zeros(1, A.shape[1])])
    return Z[torch.where(t >= 0, t.long(), A.shape[0])]


def _planes(hi, lo, dtype, strided, c0=8, extra=24):
    """The planes as `dtype` in [n, ld] buffers; strided: the operand in columns [c0, c0 + C) and NaN around it.  -> (hi, lo, c0, ld)"""
    n, C = hi.shape
    c0, ld = (c0, C + extra) if strided else (0, C)
    out = []
    for p in (hi, lo):
        b = torch.full((n, ld), float("nan"), dtype=dtype, device="cuda")
        b[:, c0:c0 + C] = p.to(dtype)
        out.append(b)
    return out[0], out[1], c0, ld


def _out_buffer(n, N, strided, base=None):
    """[n + 1, ld] fp32 filled with the sentinel (one row past the output, columns around the slice), the slice holding `base`."""
    y0, ld = (4, (N + 15) // 4 * 4) if strided else (0, N)
    Y = torch.full((n + 1, ld), SENT, device="cuda")
    if base is not None:
        Y[:n, y0:y0 + N] = base
    return Y, y0, ld


def _assert_exact(got, want, what):
    got = got.double()
    bad = got != want
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} values differ; first at {i}: got {got[tuple(i)].item()!r}, "
                             f"want {want[tuple(i)].item()!r}")


def _assert_padding(Y, n, y0, N, what):
    pad = Y.clone()
    pad[:n, y0:y0 + N] = SENT
    assert bool((pad == SENT).all()), f"{what}: output padding overwritten"


def _ws(nbytes):
    # every byte 0xFF (a NaN as fp32): a partial tile the kernel leaves unwritten poisons the reduction
    return torch.full((max(nbytes, 256),), 255, dtype=torch.uint8, device="cuda")


def _kmap_arg(kmap):
    from pointcontrast_b200 import me
    return me._c_int_array(kmap) if kmap is not None else None


def _ref_forward(xh, xl, wh, wl, tbl, kmap, n_out):
    """sum_k hi.hi + lo.hi + hi.lo of the gathered rows in fp64 (exact on these operands), and the same sum over absolute values."""
    y = torch.zeros(n_out, wh.shape[2], dtype=torch.float64, device="cuda")
    a = torch.zeros_like(y)
    for k in range(wh.shape[0]):
        t = tbl[kmap[k] if kmap is not None else k, :n_out]
        gh, gl = _gather(xh, t), _gather(xl, t)
        y += gh @ wh[k] + gl @ wh[k] + gh @ wl[k]
        a += gh.abs() @ wh[k].abs() + gl.abs() @ wh[k].abs() + gh.abs() @ wl[k].abs()
    return y, a


def _run_conv_split(fmt, K, Ck, N, tiles, wh, wl, tbl, n_src, kmap, n_out, strided, bias, base, gen, what):
    """One pcb_conv_forward_split call on fresh capped planes, checked bit for bit.  Returns the number of offset splits it ran."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    hi, lo = X.capped_planes(n_src, Ck, X.row_cap(fmt, K, Ck), fmt.HI, fmt.LO, gen, "cuda")
    xh, xl, c0, lds = _planes(hi, lo, fmt.dtype, strided)
    Y, y0, ldy = _out_buffer(n_out, N, strided, base)
    wsb = lib.pcb_conv_forward_split_ws_bytes(K, n_out, Ck, N)
    ws = _ws(wsb)
    flags = fmt.flags | (4 if base is not None else 0)
    check(lib.pcb_conv_forward_split(xh.data_ptr() + 2 * c0, xl.data_ptr() + 2 * c0, lds, ptr(tbl), tbl.shape[1], _kmap_arg(kmap), K, n_out,
                                     Ck, N, ptr(tiles), ptr(bias), Y.data_ptr() + 4 * y0, ldy, ptr(ws), wsb, flags, stream()))
    nsplit = X.conv_splits(K, n_out, Ck, N, _sms())
    assert wsb == (X.ws_align(4 * nsplit * n_out * N) if nsplit > 1 else 0), (what, wsb, nsplit)
    y, a = _ref_forward(hi.double(), lo.double(), wh, wl, tbl, kmap, n_out)
    want, bound = y * fmt.SCALE, a * fmt.SCALE
    for extra in (bias[None] if bias is not None else None, base):
        if extra is not None:
            want, bound = want + extra.double(), bound + extra.double().abs()
    assert float(bound.max()) < X.LIMIT * fmt.Q, (what, "operands leave the exact range", float(bound.max()))
    _assert_exact(Y[:n_out, y0:y0 + N], want, what)
    _assert_padding(Y, n_out, y0, N, what)
    return nsplit


def _weights_and_tiles(K, Cin, Cout, fmt, gen):
    """W, its forward / data-gradient tiles, and the hi/lo split the tiles must hold (fp64, kernel units, [K][Cin][Cout])."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    W = X.weights(K, Cin, Cout, fmt, gen, "cuda")[0]
    ft = torch.empty(lib.pcb_weight_tile_bytes(K, Cin, Cout, 0), dtype=torch.uint8, device="cuda")
    dt = torch.empty(lib.pcb_weight_tile_bytes(K, Cin, Cout, 1), dtype=torch.uint8, device="cuda")
    check(lib.pcb_weight_tile(ptr(W), K, Cin, Cout, ptr(ft), ptr(dt), 16 if fmt is X.FP16 else 0, stream()))
    wh, wl = X.split_weights(W, fmt)
    return ft, dt, wh.double(), wl.double()


def _case_id(c):
    kind, K, Cin, Cout, role, fmt = c
    return f"{kind}-{Cin}x{Cout}-{role}-{fmt}"


@pytest.mark.parametrize("ci,case", list(enumerate(X.forward_cases())), ids=[_case_id(c) for c in X.forward_cases()])
def test_split_conv_bit_exact(scene, ci, case):
    """Every shape and role at 1, 127, 128 and 129 output rows on the coordinate manager's table (offset-split mode where the rule
    splits) and at one direct-mode row count on a synthetic table (density from sparse to full, a random kernel map on every third
    shape); column slices, bias and accumulation as `exact_conv.forward_variants` assigns them."""
    kind, K, Cin, Cout, role, fname = case
    fmt = X.FMTS[fname]
    Ck, N = X.contraction(case)
    gen = torch.Generator(device="cuda").manual_seed(1000 + ci)
    ft, dt, wh, wl = _weights_and_tiles(K, Cin, Cout, fmt, gen)
    tiles = ft if role == "fwd" else dt
    if role == "dgrad":
        wh, wl = wh.transpose(1, 2).contiguous(), wl.transpose(1, 2).contiguous()
    for rows, strided, use_bias, acc in X.forward_variants(ci):
        if rows == "direct":
            n_out, n_src = X.direct_rows(N, _sms()), 4099
            tbl = _synth_table(K, n_out, n_src, (0.05, 0.4, 0.8, 1.0)[ci % 4], gen)
            kmap = torch.randperm(K, generator=gen, device="cuda").tolist() if ci % 3 == 0 else None
        else:
            (tbl, n_src, kmap), n_out = scene["fwd"][(kind, role)], rows
        bias = X.bias_values(N, fmt, gen, "cuda") if use_bias else None
        base = X.bias_values(n_out * N, fmt, gen, "cuda").view(n_out, N) if acc else None
        what = f"{_case_id(case)} rows={n_out} strided={strided} bias={use_bias} accumulate={acc} kmap={'perm' if kmap else 'none'}"
        nsplit = _run_conv_split(fmt, K, Ck, N, tiles, wh, wl, tbl, n_src, kmap, n_out, strided, bias, base, gen, what)
        if rows == "direct":
            assert nsplit == 1, what


@pytest.mark.parametrize("K,Ck,N,fname", [(27, 32, 32, "bf16"), (27, 256, 96, "bf16"), (8, 64, 320, "fp16"), (27, 768, 160, "bf16"),
                                           (1, 128, 128, "bf16"), (27, 96, 192, "fp16")])
def test_split_conv_empty_offsets_and_tiles(K, Ck, N, fname):
    """Offset-split mode on row tiles with a single offset, with no neighbour at all, with every neighbour present, sparse, and a
    5-row last tile: the z-slices that find nothing to do must still write zero partials."""
    fmt = X.FMTS[fname]
    gen = torch.Generator(device="cuda").manual_seed(K * 7 + Ck + N)
    ft, _, wh, wl = _weights_and_tiles(K, Ck, N, fmt, gen)
    n_out, n_src = 4 * X.BM + 5, 777
    tbl = _synth_table(K, n_out, n_src, 0.5, gen)
    tbl[:, :128] = -1
    tbl[K // 2, :128] = torch.randint(-1, n_src, (128,), generator=gen, device="cuda", dtype=torch.int32)
    tbl[:, 128:256] = -1
    tbl[:, 256:384] = torch.randint(0, n_src, (K, 128), generator=gen, device="cuda", dtype=torch.int32)
    tbl[:, 384:512][torch.rand(K, 128, generator=gen, device="cuda") > 0.05] = -1
    kmap = torch.randperm(K, generator=gen, device="cuda").tolist()
    nsplit = X.conv_splits(K, n_out, Ck, N, _sms())
    assert nsplit > 1                           # the no-neighbour tile leaves every one of its z-slices empty
    bias = X.bias_values(N, fmt, gen, "cuda")
    base = X.bias_values(n_out * N, fmt, gen, "cuda").view(n_out, N)
    for strided, b, acc in ((False, None, None), (True, bias, base)):
        _run_conv_split(fmt, K, Ck, N, ft, wh, wl, tbl, n_src, kmap, n_out, strided, b, acc, gen,
                        f"K={K} {Ck}x{N} {fname} nsplit={nsplit} strided={strided}")


# ----------------------------------------------------------------------------------------------- weight gradient
def _run_wgrad_split(K, Ca, Cb, tr, tbl, n_src, n, strided, acc, gen, what):
    """One pcb_conv_wgrad_split call, checked bit for bit with the sentinel around dW.  Returns the number of row splits it ran."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    f = X.BF16
    Ah, Al = X.dense_planes(n_src, Ca, X.WG_A_DENSITY, f.HI, f.LO, gen, "cuda")
    Bh, Bl = (p.t() for p in X.capped_planes(Cb, n, min(n, X.wgrad_col_cap()), f.HI, f.LO, gen, "cuda"))
    ah, al, a0, lda = _planes(Ah, Al, f.dtype, strided, c0=16, extra=40)
    bh, bl, b0, ldb = _planes(torch.cat([Bh, Bh[:1]]), torch.cat([Bl, Bl[:1]]), f.dtype, strided, c0=8, extra=24)
    bh[n], bl[n] = float("nan"), float("nan")             # the row past n
    shape = (K, Cb, Ca) if tr else (K, Ca, Cb)
    nW = K * Ca * Cb
    buf = torch.full((nW + 128,), SENT, device="cuda")
    base = X.bias_values(nW, f, gen, "cuda").view(shape) if acc else None
    if acc:
        buf[64:64 + nW] = base.reshape(-1)
    wsb = lib.pcb_conv_wgrad_split_ws_bytes(K, n, Ca, Cb)
    ws = _ws(wsb)
    check(lib.pcb_conv_wgrad_split(ah.data_ptr() + 2 * a0, al.data_ptr() + 2 * a0, lda, bh.data_ptr() + 2 * b0, bl.data_ptr() + 2 * b0, ldb,
                                   ptr(tbl), tbl.shape[1], K, n, Ca, Cb, buf.data_ptr() + 4 * 64, tr, ptr(ws), wsb, 4 if acc else 0, stream()))
    splits = wsb // (4 * nW)
    assert wsb == 4 * nW * splits and splits == X.wgrad_splits(K, n, Ca, Cb, _sms()), (what, wsb)
    want = torch.empty(shape, dtype=torch.float64, device="cuda")
    bound = torch.empty_like(want)
    Ahd, Ald, Bhd, Bld = Ah.double(), Al.double(), Bh.double(), Bl.double()
    for k in range(K):
        t = tbl[k, :n]
        gh, gl = _gather(Ahd, t), _gather(Ald, t)
        d = gl.t() @ Bhd + gh.t() @ Bld + gh.t() @ Bhd
        e = gl.abs().t() @ Bhd.abs() + gh.abs().t() @ Bld.abs() + gh.abs().t() @ Bhd.abs()
        want[k], bound[k] = (d.t(), e.t()) if tr else (d, e)
    if acc:
        want, bound = want + base.double(), bound + base.double().abs()
    assert float(bound.max()) < X.LIMIT * X.WG_Q, (what, "operands leave the exact range", float(bound.max()))
    _assert_exact(buf[64:64 + nW].view(shape), want, what)
    assert bool((buf[:64] == SENT).all() and (buf[64 + nW:] == SENT).all()), f"{what}: memory around dW overwritten"
    return splits


@pytest.mark.parametrize("case", X.wgrad_cases(), ids=[f"K{K}-{Ca}x{Cb}-tr{tr}" for K, Ca, Cb, tr in X.wgrad_cases()])
def test_split_wgrad_bit_exact(scene, case):
    """Every weight-gradient shape of the models and the extra widths (last M block of 32 / 64 / 96 / 128 rows, alone and after full
    blocks) at 1, 15, 16, 17 and 257 rows of the coordinate manager's table; column slices and accumulation alternate."""
    K, Ca, Cb, tr = case
    tbl, n_src = scene["wg"][K]
    gen = torch.Generator(device="cuda").manual_seed(K * 1000 + Ca + 7 * Cb + tr)
    for i, n in enumerate(X.WGRAD_ROWS):
        _run_wgrad_split(K, Ca, Cb, tr, tbl, n_src, n, i % 2 == 1, i in (2, 3), gen,
                         f"K={K} {Ca}x{Cb} tr={tr} n={n} strided={i % 2 == 1} accumulate={i in (2, 3)}")


def test_split_wgrad_empty_row_splits():
    """K = 1, 128 x 128 over 6200 rows: rows per split round up to 16 while the split count is capped, so the last splits have no rows
    (18 of 96 with 48 or more SMs) and must still write zero partials."""
    K, Ca, Cb, tr, n = X.BIG_WGRAD
    gen = torch.Generator(device="cuda").manual_seed(6200)
    tbl = _synth_table(K, n, n, 0.9, gen)
    for strided, acc in ((False, False), (True, True)):
        splits = _run_wgrad_split(K, Ca, Cb, tr, tbl, n, n, strided, acc, gen, f"n={n} strided={strided} accumulate={acc}")
        empty = X.wgrad_empty_splits(n, splits)
        assert empty > 0, (splits, X.wgrad_rows_per_split(n, splits))


def test_wgrad_with_no_rows_zeroes_or_keeps_dw():
    """n = 0: the weight gradient is zero (written) or nothing (accumulated), on the split and the exact entry points."""
    from pointcontrast_b200._lib import check, lib, stream
    K, Ca, Cb = 8, 64, 96
    pl = torch.zeros(64, 128, dtype=torch.bfloat16, device="cuda")
    tbl = torch.full((K, 16), -1, dtype=torch.int32, device="cuda")
    f32 = torch.zeros(64, 128, device="cuda")
    ws = _ws(0)
    for acc in (0, 4):
        for split in (True, False):
            buf = torch.full((K * Ca * Cb + 128,), SENT, device="cuda")
            dw = buf.data_ptr() + 4 * 64
            if split:
                check(lib.pcb_conv_wgrad_split(pl.data_ptr(), pl.data_ptr(), 128, pl.data_ptr(), pl.data_ptr(), 128, tbl.data_ptr(), 16, K, 0,
                                               Ca, Cb, dw, 0, ws.data_ptr(), ws.numel(), acc, stream()))
            else:
                check(lib.pcb_conv_wgrad(f32.data_ptr(), 128, f32.data_ptr(), 128, tbl.data_ptr(), 16, K, 0, Ca, Cb, dw, 0, ws.data_ptr(),
                                         ws.numel(), acc, stream()))
            inner = buf[64:64 + K * Ca * Cb]
            assert bool((inner == (SENT if acc else 0.0)).all()), (split, acc)
            assert bool((buf[:64] == SENT).all() and (buf[64 + K * Ca * Cb:] == SENT).all()), (split, acc)


# ----------------------------------------------------------------------------------------------- exact fp32 kernels
def _full_operand(n, C, gen):
    """fp32 rows hi + lo (multiples of 2^-8, |x| <= 2 + 2^-8)."""
    hi, lo = X.dense_planes(n, C, 0.7, X.BF16.HI, X.BF16.LO, gen, "cuda")
    return hi + lo


def _fp32_buffer(A, strided, c0=4, extra=9):
    """A in an [n, ld] fp32 buffer, NaN around it when strided.  -> (buffer, c0, ld)"""
    n, C = A.shape
    c0, ld = (c0, C + extra) if strided else (0, C)
    b = torch.full((n, ld), float("nan"), device="cuda")
    b[:, c0:c0 + C] = A
    return b, c0, ld


def _exact_tables(scene, kind, K, gen):
    """(table, source rows, kernel map, row counts) for an exact-kernel case."""
    if kind == "synth":
        n_src = 1500
        return _synth_table(K, 3001, n_src, 0.6, gen), n_src, torch.randperm(K, generator=gen, device="cuda").tolist(), (1, 129, 3001)
    tbl, n_src, kmap = scene["fwd"][(kind, "fwd")]
    return tbl, n_src, kmap, (1, 129, tbl.shape[1])


@pytest.mark.parametrize("kind,K,Cin,Cout", X.EXACT_FORWARD)
def test_exact_fp32_forward_bit_exact(scene, kind, K, Cin, Cout):
    """pcb_conv_forward: the 3 -> 32 stem kernel and the generic SIMT kernel (Cin = 3 -> 64, the 13 / 20 class final layers)."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    gen = torch.Generator(device="cuda").manual_seed(K + Cin + Cout)
    W = X.weights(K, Cin, Cout, X.BF16, gen, "cuda")[1].contiguous()            # the integer part: products stay on the 2^-8 grid
    tbl, n_src, kmap, rows = _exact_tables(scene, kind, K, gen)
    Xf = _full_operand(n_src, Cin, gen)
    for i, n in enumerate(rows):
        strided, use_bias = i > 0, i != 1
        xb, c0, ldx = _fp32_buffer(Xf, strided)
        Y, y0, ldy = _out_buffer(n, Cout, strided)
        bias = X.bias_values(Cout, X.BF16, gen, "cuda") if use_bias else None
        check(lib.pcb_conv_forward(xb.data_ptr() + 4 * c0, ldx, ptr(tbl), tbl.shape[1], _kmap_arg(kmap), K, n, Cin, Cout, ptr(W), ptr(bias),
                                   Y.data_ptr() + 4 * y0, ldy, stream()))
        want = torch.zeros(n, Cout, dtype=torch.float64, device="cuda")
        bound = torch.zeros_like(want)
        for k in range(K):
            g = _gather(Xf.double(), tbl[kmap[k] if kmap is not None else k, :n])
            want += g @ W[k].double()
            bound += g.abs() @ W[k].double().abs()
        if bias is not None:
            want, bound = want + bias.double(), bound + bias.double().abs()
        what = f"{kind} K={K} {Cin}x{Cout} n={n} strided={strided} bias={use_bias}"
        assert float(bound.max()) < X.LIMIT * X.EXACT_Q, what
        _assert_exact(Y[:n, y0:y0 + Cout], want, what)
        _assert_padding(Y, n, y0, Cout, what)


@pytest.mark.parametrize("K,Ca,Cb,tr,flags", X.EXACT_WGRAD)
def test_exact_fp32_wgrad_bit_exact(scene, K, Ca, Cb, tr, flags):
    """pcb_conv_wgrad: the stem kernel (3 x 32, not transposed), the generic kernel (PCB_CONV_FORCE_SIMT, transpose_out, other
    widths), with and without accumulation, at 1, 129 and all rows of the coordinate manager's table."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    gen = torch.Generator(device="cuda").manual_seed(K + Ca + Cb + tr + flags)
    tbl, n_src = scene["wg"][K]
    Af = _full_operand(n_src, Ca, gen)
    shape = (K, Cb, Ca) if tr else (K, Ca, Cb)
    nW = K * Ca * Cb
    for i, n in enumerate((1, 129, tbl.shape[1])):
        m = min(n, X.exact_wgrad_col_cap())
        B = X.capped_planes(Cb, n, m, X.BF16.HI, X.BF16.LO, gen, "cuda")[0].t().contiguous()       # integers, <= m nonzeros per column
        strided = i > 0
        ab, a0, lda = _fp32_buffer(Af, strided)
        bb, b0, ldb = _fp32_buffer(B, strided, c0=8, extra=13)
        buf = torch.full((nW + 128,), SENT, device="cuda")
        base = X.bias_values(nW, X.BF16, gen, "cuda").view(shape) if flags & 4 else None
        if base is not None:
            buf[64:64 + nW] = base.reshape(-1)
        wsb = lib.pcb_conv_wgrad_ws_bytes(K, n, Ca, Cb)
        ws = _ws(wsb)
        check(lib.pcb_conv_wgrad(ab.data_ptr() + 4 * a0, lda, bb.data_ptr() + 4 * b0, ldb, ptr(tbl), tbl.shape[1], K, n, Ca, Cb,
                                 buf.data_ptr() + 4 * 64, tr, ptr(ws), wsb, flags, stream()))
        want = torch.empty(shape, dtype=torch.float64, device="cuda")
        bound = torch.empty_like(want)
        for k in range(K):
            g = _gather(Af.double(), tbl[k, :n])
            d, e = g.t() @ B.double(), g.abs().t() @ B.double().abs()
            want[k], bound[k] = (d.t(), e.t()) if tr else (d, e)
        if base is not None:
            want, bound = want + base.double(), bound + base.double().abs()
        what = f"K={K} {Ca}x{Cb} tr={tr} flags={flags} n={n} strided={strided}"
        assert float(bound.max()) < X.LIMIT * X.EXACT_Q, what
        _assert_exact(buf[64:64 + nW].view(shape), want, what)
        assert bool((buf[:64] == SENT).all() and (buf[64 + nW:] == SENT).all()), f"{what}: memory around dW overwritten"


@pytest.mark.parametrize("kind,K", [("k27", 27), ("down", 8), ("up", 8), ("synth", 27)])
def test_gather_sum_bit_exact_with_counts(scene, kind, K):
    """pcb_gather_sum: the row sums over a table, in column slices, and the neighbour counts."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    gen = torch.Generator(device="cuda").manual_seed(K + len(kind))
    if kind == "synth":
        n_src = 1500
        tbl, kmap, rows = _synth_table(K, 3001, n_src, 0.6, gen), torch.randperm(K, generator=gen, device="cuda").tolist(), (1, 129, 3001)
    else:
        tbl, n_src, kmap = scene["fwd"][(kind, "fwd")]
        rows = (1, 129, tbl.shape[1])
    C = 24
    Xf = _full_operand(n_src, C, gen)
    for i, n in enumerate(rows):
        strided = i > 0
        xb, c0, ldx = _fp32_buffer(Xf, strided, c0=4, extra=8)
        Y, y0, ldy = _out_buffer(n, C, strided)
        cnt = torch.full((n + 1,), SENT, device="cuda")
        check(lib.pcb_gather_sum(xb.data_ptr() + 4 * c0, ldx, ptr(tbl), tbl.shape[1], _kmap_arg(kmap), K, n, C, Y.data_ptr() + 4 * y0, ldy,
                                 ptr(cnt), stream()))
        want = torch.zeros(n, C, dtype=torch.float64, device="cuda")
        present = torch.zeros(n, dtype=torch.float64, device="cuda")
        for k in range(K):
            t = tbl[kmap[k] if kmap is not None else k, :n]
            want += _gather(Xf.double(), t)
            present += (t >= 0).double()
        what = f"{kind} K={K} n={n} strided={strided}"
        _assert_exact(Y[:n, y0:y0 + C], want, what)
        _assert_padding(Y, n, y0, C, what)
        _assert_exact(cnt[:n], present, what + " counts")
        assert float(cnt[n]) == SENT, what


# ----------------------------------------------------------------------------------------------- Res16UNet14 through the fused executor
def test_res16unet14_fused_pair_matches_fp64_oracle():
    """Res16UNet14 (base planes: decoder concatenations of 384, 320, 288 and 288 channels) through the fused executor's stacked pass,
    against the fp64 oracle: per-point features to 1e-3, as Res16UNet34C in tests/test_gpu_model.py."""
    from oracle import me_cpu as OR
    from pointcontrast_b200 import synth
    from pointcontrast_b200.model import load_model
    from tests import refload
    from tests.helpers import det_init, max_rel_err, model_backend
    batch = synth.collate_pairs([synth.synth_pair(3, scale=0.12)])
    net = load_model("Res16UNet14")(3, 32, refload.default_config(), D=3)
    det_init(net, 1)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    net = net.cuda().train()
    T = {k: torch.from_numpy(batch[k]) for k in ("sinput0_F", "sinput0_C", "sinput1_F", "sinput1_C")}
    F = net.forward_pair(T["sinput0_F"], T["sinput0_C"], T["sinput1_F"], T["sinput1_C"], torch.device("cuda"))
    assert "_fused_runner" in net.__dict__
    with model_backend(OR) as mod:
        onet = mod.Res16UNet14(3, 32, refload.default_config(), D=3).double()
        onet.load_state_dict({k: v.double() if v.dtype.is_floating_point else v for k, v in state.items()})
        onet.train()
        Fo = [onet(OR.SparseTensor(T[f"sinput{v}_F"].double(), coords=T[f"sinput{v}_C"])).F for v in "01"]
    for v in (0, 1):
        assert max_rel_err(F[v], Fo[v]) < 1e-3, v


def test_res16unet14_fused_executor_matches_modular_path():
    """The fused executor against the per-module path on Res16UNet14 (bf16 operands on both sides): features to 1e-5, every parameter
    gradient to 2e-4, as for Res16UNet34C."""
    from tests.test_gpu_model import check_fused_matches_modular
    check_fused_matches_modular("Res16UNet14")
