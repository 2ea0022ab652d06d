"""Host checks of tests/exact_unit.py (no GPU): the case matrix holds every unit of the models, and every generated backward operand
obeys the exactness rule stated in that module."""
import pytest
import torch

from tests import exact_bn as XB
from tests import exact_conv as XC
from tests import exact_unit as XU


@pytest.mark.parametrize("name", XU.MODELS)
def test_matrix_holds_every_unit_of_the_model(name):
    units = XU.model_units(name)
    matrix = set(XU.signatures())
    for s in units:
        for fp16 in (False, True):
            assert s._replace(fp16=fp16) in matrix, s.name()
        assert XU.forward_part(s)._replace(fp16=True, eval=True, two_views=False) in matrix, s.name()
    kinds = {s.kind for s in units}
    assert kinds == {"stem", "k27", "down", "up", "k1"}, kinds


def test_executor_wiring_restated():
    """Hand-checked units of Res16UNet34C: the stem writes into the last 32 columns of the final concatenation and wants no input
    gradient; the first down-convolution accumulates into that slice; a block's second unit writes the residual gradient; the up
    convolutions write column slices; every gradient mode and slice flag the executor uses occurs."""
    u = XU.model_units("Res16UNet34C")
    stem, down1 = u[0], u[1]
    assert (stem.kind, stem.Cin, stem.gin_mode, stem.out_str, stem.g_str, stem.x_str) == ("stem", 3, 0, True, True, False)
    assert (down1.kind, down1.gin_mode, down1.x_str, down1.gin_str) == ("down", 2, True, True)
    seconds = [s for s in u if s.res]
    assert seconds and all(s.gres_mode == 1 and s.relu for s in seconds)
    assert all(s.out_str and s.gin_mode == 1 for s in u if s.kind == "up")
    assert {s.gin_mode for s in u} == {0, 1, 2} and any(s.out_p for s in u) and any(not s.relu for s in u)
    assert all(s.two_views and not s.fp16 and not s.eval for s in u)


def test_view_split_cuts_inside_a_chunk():
    for n in (1, 2, 3, 1500, 6144, 90_001):
        n0 = XU.view_split(n)
        assert 1 <= n0 <= n
        if n > 2:
            assert n0 < n and n0 % XB.chunk_rows(n) != 0, n


def test_dz_values_split_into_both_bf16_planes():
    for h, l in XU.DZ_VALUES:
        for s in (1.0, -1.0):
            v = torch.tensor([s * (h + l)], dtype=torch.float32)
            hi = v.to(torch.bfloat16).float()
            lo = (v - hi).to(torch.bfloat16).float()
            assert float(hi) == s * h and float(lo) == s * l and l != 0


def _case(kind, K, Cin, Cout, fp16):
    return XU.Sig(kind, K, Cin, Cout, True, False, False, 0, 1, fp16, False, True, False, False, False, False, False)


@pytest.mark.parametrize("n,sig", [(1499, _case("k27", 27, 32, 32, False)), (20_000, _case("down", 8, 64, 128, True)),
                                   (60_001, _case("up", 8, 256, 128, False)), (3001, _case("k1", 1, 384, 256, False)),
                                   (30_000, _case("stem", 27, 3, 32, False))])
def test_paired_operands_obey_the_rule(n, sig):
    n0 = XU.view_split(n)
    row_cap, col_cap = XU.backward_caps(sig, sig.K)
    p = XU.paired_backward(n, n0, sig.Cout, row_cap, col_cap, not sig.tc, "fp16" if sig.fp16 else "bf16", seed=n)
    g, z = p["g"], p["z"]
    # pairing: rows 2i, 2i + 1 of each view share z and codes, g is opposite; an odd last row has g = 0
    first, second, alone = XU.pair_partner(n, n0)
    assert bool((z == z[first]).all() and (p["codes"] == p["codes"][first]).all())
    assert bool((g[second] == -g[first[second]]).all() and (g[alone] == 0).all())
    for a, e in XB.segments(n, n0):
        assert bool((g[a:e].double().sum(0) == 0).all())
    # gamma * invstd is a signed power of two, the same in both views; mean on the grid; |z - mean| <= D_MAX 2^-3
    c = p["gamma"] * p["invstd"]
    assert bool((c.abs().log2() == c.abs().log2().round()).all() and (c[0] == c[1]).all())
    assert bool(((p["mean"] / XU.Q).frac() == 0).all())
    view = (torch.arange(n) >= n0).long()
    assert bool(((z - p["mean"][view]).abs() <= XU.D_MAX * XU.Q).all())
    # dz = c g is v = h + l with the intended bf16 split (integers for the stem)
    v = (g * c[0]).float()
    assert bool((v == p["h"] + p["l"]).all())
    hi = v.to(torch.bfloat16).float()
    if sig.tc:
        assert bool((hi == p["h"]).all() and ((v - hi).to(torch.bfloat16).float() == p["l"]).all())
        both = (p["h"] != 0) & (p["l"] != 0)
        assert bool((both == (v != 0)).all()) and int(both.sum()) > 0.05 * n * min(row_cap, sig.Cout) / sig.Cout * sig.Cout / 2
    else:
        assert bool((v == v.round()).all() and (p["l"] == 0).all())
    # caps: rows for the data gradient, columns for the weight gradient and the BatchNorm sums
    assert XU.row_nonzeros(g) <= row_cap and XU.col_nonzeros(g) <= col_cap
    assert XU.bn_sum_terms(p, n0) < XU.BN_LIMIT
    want_col = XC.exact_wgrad_col_cap() if not sig.tc else XC.wgrad_col_cap() if sig.kind != "up" else XU.BN_COL_CAP
    assert col_cap == min(want_col, XU.BN_COL_CAP)
    # mask codes: positive, +-0, negative and subnormal codes; out_bhi differs in sign / zero pattern
    ok = XB.mask_passes(p["codes"])
    assert 0.2 < float(ok.float().mean()) < 0.8
    assert bool((XB.mask_passes(p["bcodes"]) != ok).any())
    codes = p["codes"].to(torch.int32) & 0xFFFF
    assert {0x0000, 0x8000, 0x0001}.issubset(set(codes.unique().tolist()))


def test_unpaired_operands_are_exact_bn_operands():
    for n0, n1, C in ((1499, 0, 32), (750, 749, 256)):
        x, dy, mean, invstd, _, bg, _, _ = XU.unpaired_backward(n0, n1, C, seed=n0)
        assert XB.backward_terms(x, dy, mean, invstd, n0 if n1 else n0 + n1, bg)[0] < 1.0
