"""Host checks of the exact BatchNorm tests (tests/test_gpu_bn_exact.py, operands and rules in tests/exact_bn.py): the restated chunk
rules, the geometry the case matrix reaches, and that every generated operand obeys the exactness rule."""
import pytest
import torch

from tests import exact_bn as X


def test_chunk_rule_restated():
    """Hand-checked values of bn.cu chunk_rows / chunk_geometry and of the finalize loop split."""
    assert X.chunk_rows(1) == 16 and X.chunk_rows(6144) == 16 and X.chunk_rows(12799) == 16 and X.chunk_rows(12800) == 32
    assert X.chunk_geometry(6144, 6144, 32)[:3] == (16, 384, 384)
    assert X.chunk_geometry(6145, 6145, 32)[:3] == (16, 385, 385)
    assert X.chunk_rows(393_727) == 512 and X.chunk_rows(393_728) == 1024 and X.chunk_rows(10 ** 8) == 1024
    assert X.chunk_rows(100_000) == 256
    # two views round up separately: 6144 | 6145 rows at R = 16 -> 384 + 385 chunks
    assert X.chunk_geometry(12289, 6144, 4)[:3] == (16, 769, 384)
    assert X.lanes(4) == (1, 256, 256) and X.lanes(1024) == (256, 1, 256) and X.lanes(12) == (3, 85, 255) and X.lanes(20) == (5, 51, 255)
    assert X.lanes(96) == (24, 10, 240)
    assert X.chunk_geometry(10, 10, 96)[4] == 10 * 2 * 96 * 4
    assert [X.finalize_pass(k) for k in (0, 383, 384, 415, 416, 447, 448)] == [0, 0, 1, 1, 2, 2, 3]


def test_row_chunks_never_straddle_the_view_boundary():
    for n0, n1 in ((6144, 6145), (1, 5000), (431, 0), (17, 1)):
        n = n0 + n1
        cid, first, size, j = X.row_chunks(n, n0 if n1 else n)
        R, chunks, chunks0, _, _ = X.chunk_geometry(n, n0 if n1 else n, 4)
        assert int(cid.max()) + 1 == chunks and bool((size <= R).all()) and bool((j < size).all())
        view = torch.arange(n) >= n0
        assert bool((view == (first >= n0)).all()) and bool(((cid >= chunks0) == view).all() if n1 else True)


def test_case_matrix_reaches_every_geometry():
    seen = set()
    for _, n0, n1, C, _, _ in X.stats_cases():
        seen |= X.reaches(n0, n1, C)
    want = {"R 16", "R 1024", "R between", "rp 1", "rp 256", "threads not a multiple of 32", "one view", "two views", "n0 % R == 0",
            "n0 % R != 0", "< 384 chunks", "384 chunks", "385 chunks", "> 416 chunks", "one-row view", "one-row last chunk"}
    for v in (0, 1):
        want |= {f"view {v}: < 384 chunks", f"view {v}: 384 chunks", f"view {v}: 385 chunks", f"view {v}: > 416 chunks",
                 f"view {v}: one-row view", f"view {v}: one-row last chunk"}
    assert seen >= want, sorted(want - seen)
    # the backward pass: more than 384 + 32 chunks in each view, and a view at exactly 384 / 385
    bw = set().union(*(X.reaches(n0, n1, C) for _, n0, n1, C in X.BACKWARD_CASES))
    assert bw >= {"view 0: > 416 chunks", "view 1: > 416 chunks", "view 0: 385 chunks", "view 1: 384 chunks", "rp 1"}, sorted(bw)


def test_every_model_batchnorm_width_is_a_case():
    widths = {C for name in X.MODELS for C in X.model_bn_widths(name)}
    assert widths == set(X.bn_widths()) and 32 in widths and len(widths) >= 5
    assert {C for _, _, _, C, _, _ in X.stats_cases()} >= widths


@pytest.mark.parametrize("case", X.stats_cases(), ids=[c[0] for c in X.stats_cases()])
def test_every_statistics_operand_is_exact(case):
    name, n0, n1, C, offset, pattern = case
    x = X.stats_operand(n0, n1, C, offset, pattern, seed=X.seed_of(name))
    n = n0 + n1
    assert x.shape == (n, C) and x.dtype == torch.float32
    worst, on_grid = X.stats_terms(x, n0 if n1 else n)
    assert on_grid and worst < 1.0, (name, worst)
    assert float((x.double() - offset).abs().max()) <= X.SPREAD
    if pattern == "zero-sum":
        assert not bool(X.chunk_shifted_sums(x, n0 if n1 else n).any())
    assert len(torch.unique(x[:, 0])) > min(n, 4) - 1


@pytest.mark.parametrize("case", X.BACKWARD_CASES, ids=[c[0] for c in X.BACKWARD_CASES])
def test_every_backward_operand_is_exact(case):
    name, n0, n1, C = case
    x, dy, mean, invstd, gamma, bg, bb, gb = X.backward_operands(n0, n1, C, seed=n0 + C)
    n = n0 + n1
    for base in (bg, bb):
        worst, on_grid = X.backward_terms(x, dy, mean, invstd, n0, base)
        assert on_grid and worst < 1.0, (name, worst)
    assert float(dy.abs().sum(0).max()) + float(bb.abs().max()) < X.LIMIT * X.G_Q
    assert bool((dy != 0).any(1).sum() > min(n, 1000) * X.backward_density(n) * 0.5)


def test_apply_operands_are_exact():
    """y = (x - mean) invstd gamma + beta + residual on the apply operands needs few bits: it is exact in fp32 in any evaluation order."""
    for _, n0, n1, C in X.APPLY_CASES:
        x, mean, invstd, gamma, beta, res = (t.double() for t in X.apply_operands(n0, n1, C, seed=C))
        view = (torch.arange(n0 + n1) >= n0).long()
        t = (x - mean[view]) * invstd[view] * gamma
        y = t + beta + res
        for v in (t, t + beta, y):
            assert bool((v / 2.0 ** -6 == (v / 2.0 ** -6).round()).all()) and float(v.abs().max()) < 2.0 ** 17


def test_mask_codes_cover_the_contract():
    for fmt in ("bf16", "fp16"):
        c = X.mask_codes(64, 32, fmt, seed=1).to(torch.int32) & 0xFFFF
        for code in (0x0000, 0x8000, 0x0001, 0x8001):
            assert bool((c == code).any()), (fmt, code)
        ok = X.mask_passes(X.mask_codes(64, 32, fmt, seed=1))
        assert not bool(ok[c == 0x8000].any()) and not bool(ok[c == 0].any()) and bool(ok[c == 1].all())
        assert not bool(ok[c >= 0x8000].any()) and bool(ok[(c > 0) & (c < 0x8000)].all())
