"""Host checks of tests/exact_callers.py (no GPU): every new case keeps its operands in the exact range at the rows it runs, each row
count runs the kernel mode it is meant to, and the identity table's stride differs from the rows it serves."""
import pytest

from tests import exact_callers as XK
from tests import exact_conv as XC
from tests import exact_unit as XU


def test_callers_are_restated():
    """The restatement reaches every caller: identity-table units of the modules and heads, the one-view Res16UNet units, the heads'
    bias-column units, the 2^20-row cases, and the widths the issue of each caller names."""
    sigs = set(XK.unit_signatures())
    assert XK.BIG_UNIT in sigs
    assert {s.kind for s in sigs} == {"ident", "stem", "k27", "down", "up", "k1"}
    assert all(not s.two_views and s.fp16 for s in sigs)
    heads = [s for s in sigs if s.kind == "ident" and s.out_str]
    assert {(s.Cin, s.Cout) for s in heads} == {(288, 256), (160, 128)} and all(s.g_str or s.eval for s in heads)
    assert {s.gin_mode for s in heads if not s.eval} == {1, 2}
    split = set(XK.split_cases())
    assert {(1, 288, 544, "fwd", "fp16", False, False), (1, 160, 128, "fwd", "fp16", False, False),
            (1, 160, 96, "wgrad", "bf16", False, True), (1, 96, 256, "fwd", "fp16", False, False)} <= split
    assert {(1, 1, 64), (1, 64, 3), (1, 96, 20)} <= set(XK.exact_forward_cases())
    assert XK.BIG_EXACT_WGRAD in XK.exact_wgrad_cases()
    assert XK.SA1_ROWS == 2 ** 20


def test_head_padding():
    assert XK.head_padding(288, 288) == (256, 259) and XK.head_padding(288, 544) == (256, 518)
    assert XK.head_padding(160, 128) == (128, 97) and XK.head_padding(160, 96) == (128, 79)
    assert XK.head_padding(128, 256) is None
    # the voting head at V = 2 runs 17 column tiles of 32; its weight gradient's last M block has 32 rows
    assert XC.pick_tile(544) == 32 and XC.col_blocks(544) == 17
    assert XC.m_blocks(288) == (3, 32) and XC.m_blocks(160) == (2, 32)


def test_rows_run_the_intended_modes():
    """The proposal head's rows split every caller shape (statistics fused into the reduction), the voting head's and 2^20 run direct."""
    for s in XK.unit_signatures():
        if s.kind == "ident":
            assert XK.conv_mode(1, XK.PROPOSAL_ROWS, s.Cin, s.Cout) == "split", s.name()
            assert XK.conv_mode(1, XK.VOTE_ROWS, s.Cin, s.Cout) == "direct", s.name()
    assert XK.conv_mode(1, XK.SA1_ROWS, 64, 64) == "direct"
    for K, Ck, N, role, *_ in XK.split_cases():
        if role != "wgrad":
            # 544 columns (17 tiles) at 512 rows already fill half the SMs: the 1- and 129-row calls split
            assert {XK.conv_mode(K, n, Ck, N) for n in XK.SPLIT_ROWS} == {"split", "direct"}, (Ck, N)
            assert XK.conv_mode(K, XK.VOTE_ROWS, Ck, N) == "direct"


def test_identity_stride_differs_from_rows():
    """pointnet2_modules._identity's table is at least 65536 long: the proposal head's 512 rows read it with stride 65536."""
    stride = lambda n: max(n, 1 << 16)
    assert stride(XK.PROPOSAL_ROWS) != XK.PROPOSAL_ROWS and stride(XK.SA1_ROWS) == XK.SA1_ROWS


@pytest.mark.parametrize("n", (XK.PROPOSAL_ROWS, XK.VOTE_ROWS, XK.SA1_ROWS))
def test_unit_operands_stay_exact(n):
    """Forward (with the heads' bias entry), the paired backward's BatchNorm sums and column caps at every row count a unit runs."""
    for s in XK.training_signatures():
        if s.kind != "ident" or (n == XK.SA1_ROWS and s != XK.BIG_UNIT):
            continue
        fmt = XC.FP16
        m = XC.row_cap(fmt, 1, s.Cin) - (1 if s.out_str else 0)
        assert XC.forward_bound(fmt, 1, m + (1 if s.out_str else 0)) < XC.LIMIT * fmt.Q, s.name()
        row_cap, col_cap = XU.backward_caps(s, 1)
        assert col_cap * XU.BN_TERM < XU.BN_LIMIT and XC.wgrad_bound(col_cap) < XC.LIMIT * XC.WG_Q
        if n <= XK.VOTE_ROWS:
            p = XU.paired_backward(n, n, s.Cout, row_cap, col_cap, False, "fp16", seed=n + s.Cin)
            assert XU.bn_sum_terms(p, n) < XU.BN_LIMIT
            assert XU.col_nonzeros(p["g"]) <= col_cap and XU.row_nonzeros(p["g"]) <= row_cap


def test_exact_fp32_operands_stay_exact():
    for K, Cin, Cout in XK.exact_forward_cases():
        assert XC.exact_forward_bound(K, Cin) < XC.LIMIT * XC.EXACT_Q
    assert XC.exact_wgrad_bound(XC.exact_wgrad_col_cap()) < XC.LIMIT * XC.EXACT_Q
