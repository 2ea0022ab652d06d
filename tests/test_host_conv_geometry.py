"""Host checks of the bit-exact convolution tests (tests/test_gpu_conv_exact.py, operands and rules in tests/exact_conv.py): the case
matrix reaches every tile geometry the library's tile rules produce for the Res16UNet models, and the operand generators stay on the
grid that makes the kernels exact, for every case the GPU file builds."""
import pytest
import torch

from tests import exact_conv as X

H100_SMS = 132          # H100 SXM; the rules below are also evaluated on other SM counts where the claim does not depend on it


def test_model_widths_come_from_the_models():
    """The decoder concatenations of the base-plane models (384, 320, 288) and of Res16UNet34C (192, 128) reach the matrix."""
    shapes = X.conv_shapes()
    for name in X.MODELS:
        for c in X.model_convs(name):
            if c[2] % 32 == 0 and c[3] % 32 == 0:
                assert c in shapes, (name, c)
    for name, widths in (("Res16UNet14", (384, 320, 288)), ("Res16UNet18", (384, 320, 288)), ("Res16UNet34", (384, 320, 288)),
                         ("Res16UNet34C", (384, 192, 128))):
        cins = {c[2] for c in X.model_convs(name) if c[1] == 27}
        assert set(widths) <= cins, (name, sorted(cins))
    assert ("k27", 27, 3, 32) in X.model_convs("Res16UNet14")            # the stem: exact fp32 kernels
    assert max(c[2] for c in shapes) == 768 and 768 // X.BK == 24


def test_every_column_tile_runs_with_one_and_with_several_blocks():
    seen = {}
    for case in X.forward_cases():
        N = X.contraction(case)[1]
        seen.setdefault(X.pick_tile(N), set()).add(min(X.col_blocks(N), 2))
    assert seen == {b: {1, 2} for b in (32, 64, 96, 128)}, seen
    for fmt in ("bf16", "fp16"):         # in both operand formats
        tiles = {(X.pick_tile(X.contraction(c)[1]), X.col_blocks(X.contraction(c)[1]) > 1) for c in X.forward_cases() if c[5] == fmt}
        assert tiles == {(b, m) for b in (32, 64, 96, 128) for m in (False, True)}, fmt
    roles = {(c[4], c[5]) for c in X.forward_cases()}
    assert roles == {("fwd", "bf16"), ("fwd", "fp16"), ("dgrad", "bf16")}
    assert {c[1] for c in X.forward_cases()} == {1, 8, 27} and {c[0] for c in X.forward_cases()} == {"k27", "down", "up", "k1"}


@pytest.mark.parametrize("sms", [H100_SMS, 114, 78])
def test_forward_rows_reach_both_modes_with_bias_and_accumulation(sms):
    """Direct mode at the direct row count, offset-split mode at 1..129 rows whenever the rule can split (more than one step), and
    bias / accumulation each in both modes."""
    flags = set()
    for ci, case in enumerate(X.forward_cases()):
        _, K, _, _, _, _ = case
        Ck, N = X.contraction(case)
        for rows, strided, bias, acc in X.forward_variants(ci):
            n = X.direct_rows(N, sms) if rows == "direct" else rows
            assert rows != "direct" or n % X.BM != 0
            nsplit = X.conv_splits(K, n, Ck, N, sms)
            if rows == "direct":
                assert nsplit == 1, (case, n)
            elif K * Ck // X.BK >= 2:
                assert nsplit > 1, (case, n)
            mode = "direct" if nsplit == 1 else "split"
            flags |= {(mode, "bias")} if bias else set()
            flags |= {(mode, "accumulate")} if acc else set()
            flags |= {(mode, "strided")} if strided else set()
    assert flags == {(m, f) for m in ("direct", "split") for f in ("bias", "accumulate", "strided")}


def test_every_last_m_block_size_runs_alone_and_after_full_blocks():
    seen = set()
    for K, Ca, Cb, tr in X.wgrad_cases():
        nb, last = X.m_blocks(Ca)
        seen.add((last, nb > 1))
    assert seen == {(r, m) for r in (32, 64, 96, 128) for m in (False, True)}, sorted(seen)
    assert {c[0] for c in X.wgrad_cases()} == {1, 8, 27} and {c[3] for c in X.wgrad_cases()} == {0, 1}
    assert {c[2] for c in X.wgrad_cases()} >= {32, 64, 96, 128, 160, 224, 256, 416}


def test_big_weight_gradient_has_empty_row_splits():
    """K = 1, 128 x 128, 6200 rows: 96 splits of 80 rows on an H100 SXM, the last 18 empty (and empty splits on any count >= 48 SMs)."""
    K, Ca, Cb, tr, n = X.BIG_WGRAD
    s = X.wgrad_splits(K, n, Ca, Cb, H100_SMS)
    assert (s, X.wgrad_rows_per_split(n, s), X.wgrad_empty_splits(n, s)) == (96, 80, 18)
    for sms in range(48, 200):
        assert X.wgrad_empty_splits(n, X.wgrad_splits(K, n, Ca, Cb, sms)) > 0, sms
    # the small row counts: one step, a partial step, whole steps
    assert {n % 16 for n in X.WGRAD_ROWS} == {0, 1, 15} and min(X.WGRAD_ROWS) == 1


def test_empty_offset_tiles_run_split():
    """The shapes of test_split_conv_empty_offsets_and_tiles (4 x 128 + 5 rows) run offset-split on an H100 SXM, and a one-offset tile
    of a 32-channel contraction has fewer steps than z-slices."""
    assert X.conv_splits(27, 4 * X.BM + 5, 32, 32, H100_SMS) > 32 // X.BK
    for K, Ck, N in ((27, 256, 96), (8, 64, 320), (27, 768, 160), (1, 128, 128), (27, 96, 192)):
        assert X.conv_splits(K, 4 * X.BM + 5, Ck, N, H100_SMS) > 1, (K, Ck, N)


def _on(values, allowed):
    return bool(torch.isin(values, torch.tensor(sorted(allowed))).all())


@pytest.mark.parametrize("fname", ["bf16", "fp16"])
def test_weight_split_is_the_intended_one(fname):
    """W = (a + b WB) SCALE splits, under the tiles' restated rounding, into exactly hi = a and lo = b WB (kernel units); the fp32
    weights of the exact kernels (the integer part a) have no residual."""
    fmt = X.FMTS[fname]
    gen = torch.Generator().manual_seed(1)
    W, a, b = X.weights(27, 64, 96, fmt, gen)
    assert _on(a, {0.0} | {s * v for v in fmt.WA for s in (1, -1)}) and _on(b, {0.0, fmt.WB, -fmt.WB})
    assert bool((a != 0).any()) and bool((b != 0).any()) and bool((a == 0).any())
    hi, lo = X.split_weights(W, fmt)
    assert torch.equal(hi, a) and torch.equal(lo, b)
    # the same split as tests/test_gpu_ops.py::_host_tile_image (bf16 / fp16 of W or W 2^10, then of the residual)
    v = W * 1024.0 if fmt is X.FP16 else W
    assert torch.equal(v.to(fmt.dtype).float(), a) and torch.equal((v - v.to(fmt.dtype).float()).to(fmt.dtype).float(), b)
    ah, al = X.split_weights(a, X.BF16)
    assert torch.equal(ah, a) and not bool(al.any())


@pytest.mark.parametrize("ci,case", list(enumerate(X.forward_cases())))
def test_forward_operands_are_exact(ci, case):
    """Every forward case: planes on the grid, at most row_cap nonzeros per row, and the table-free bound -- K gathered rows times the
    largest weight, plus |bias| and |base| -- below 2^20 Q."""
    kind, K, Cin, Cout, role, fname = case
    fmt = X.FMTS[fname]
    Ck, _ = X.contraction(case)
    m = X.row_cap(fmt, K, Ck)
    assert X.forward_bound(fmt, K, m) < X.LIMIT * fmt.Q
    assert m == Ck or X.forward_bound(fmt, K, m + 1) >= X.LIMIT * fmt.Q          # as dense as the bound allows
    hi, lo = X.capped_planes(200, Ck, m, fmt.HI, fmt.LO, torch.Generator().manual_seed(ci))
    assert _on(hi, {0.0} | {s * v for v in fmt.HI for s in (1, -1)}) and _on(lo, {0.0, fmt.LO, -fmt.LO})
    assert int((hi != 0).sum(1).max()) <= m and int((lo != 0).sum(1).max()) <= m and bool((hi != 0).any())
    assert torch.equal(hi.to(fmt.dtype).float(), hi) and torch.equal(lo.to(fmt.dtype).float(), lo)
    # every product and the bias / base values lie on the Q grid
    for v in [h * w for h in fmt.HI for w in fmt.WA] + [fmt.LO * w for w in fmt.WA] + [h * fmt.WB for h in fmt.HI] + list(X.BIAS):
        assert v * fmt.SCALE / fmt.Q == int(v * fmt.SCALE / fmt.Q), (v, fmt.name)


@pytest.mark.parametrize("case", X.wgrad_cases() + (X.BIG_WGRAD[:4],))
def test_wgrad_operands_are_exact(case):
    """Weight gradient: B holds at most wgrad_col_cap nonzeros per column, so any table over any number of rows stays exact."""
    K, Ca, Cb, tr = case
    m = X.wgrad_col_cap()
    assert X.wgrad_bound(m) < X.LIMIT * X.WG_Q <= X.wgrad_bound(m + 1)
    f = X.BF16
    gen = torch.Generator().manual_seed(Ca + Cb)
    n = 2000
    B = X.capped_planes(Cb, n, min(n, m), f.HI, f.LO, gen)
    assert all(int((p != 0).sum(1).max()) <= m for p in B)
    A = X.dense_planes(300, Ca, X.WG_A_DENSITY, f.HI, f.LO, gen)
    for h, l in (A, B):
        assert _on(h, {0.0, 1.0, -1.0, 2.0, -2.0}) and _on(l, {0.0, f.LO, -f.LO})
    for v in (f.LO * 1, f.HI[0] * f.HI[0]) + X.BIAS:
        assert v / X.WG_Q == int(v / X.WG_Q)


def test_exact_fp32_operands_are_exact():
    for kind, K, Cin, Cout in X.EXACT_FORWARD:
        assert X.exact_forward_bound(K, Cin) < X.LIMIT * X.EXACT_Q, (kind, K, Cin, Cout)
    m = X.exact_wgrad_col_cap()
    assert X.exact_wgrad_bound(m) < X.LIMIT * X.EXACT_Q <= X.exact_wgrad_bound(m + 1)
    hi, lo = X.dense_planes(100, 3, 0.7, X.BF16.HI, X.BF16.LO, torch.Generator().manual_seed(0))
    full = hi + lo
    assert torch.equal(full - hi, lo) and bool((full * 256 == (full * 256).round()).all())
    # the exact kernels cover the stem (3 -> 32), the generic forward at 3 -> 64 and the class counts of the final layer
    assert {(c[2], c[3]) for c in X.EXACT_FORWARD} >= {(3, 32), (3, 64), (96, 13), (256, 20)}
    assert {(c[1], c[2], c[3], c[4]) for c in X.EXACT_WGRAD} >= {(3, 32, 0, 0), (3, 32, 0, 1), (3, 32, 1, 0)}
    assert {c[0] for c in X.EXACT_FORWARD} >= {"k27", "down", "k1", "synth"}
