"""`pcb_conv_wgrad_split` where the weight-gradient kernel's pipeline and offset stacking have edges, held bit for bit to the fp64
reference of tests/test_gpu_conv_exact.py on its exactly representable operands: row splits long enough to wrap the slot ring three
times at every (A channel tile, B channel tile) instantiation, offset groups cut short by K, splits that end inside a 32-row stage, both
output layouts, and two calls on the same (not exactly representable) inputs giving the same bits.
"""
import pytest
import torch

from tests import exact_conv as X
from tests.test_gpu_conv_exact import _run_wgrad_split, _sms, _synth_table

pytestmark = pytest.mark.gpu

TILES = (32, 64, 96, 128)
STAGE_ROWS = 32


def _offsets_per_cta(cb):
    """conv_wgmma.cu wg::Smem::GK: offsets stacked along M so that GK * cb fills whole M64 slices of both consumer warpgroups."""
    return 2 if cb % 64 == 0 else 4


def _ring_slots(cb, tn):
    """conv_wgmma.cu wg::Smem::NS: 32-row stages of the B and stacked A hi/lo planes, as many as fit in 227 KB."""
    stage = 4 * STAGE_ROWS * (tn + _offsets_per_cta(cb) * cb)
    return (227 * 1024 - 16) // (stage + 16)


def _rows_wrapping(K, Ca, Cb, wraps):
    """A row count (not a multiple of 16) whose row splits each hold at least `wraps` rounds of the ring, and whose rows per split end
    16 rows into a stage."""
    need = wraps * _ring_slots(X.pick_tile(Ca), X.pick_tile(Cb)) * STAGE_ROWS
    n = need
    while True:
        s = X.wgrad_splits(K, n, Ca, Cb, _sms())
        rps = X.wgrad_rows_per_split(n, s)
        if rps >= need and rps % STAGE_ROWS == 16 and n % 16:
            return n
        n += 7


@pytest.mark.parametrize("cb", TILES)
@pytest.mark.parametrize("tn", TILES)
def test_wgrad_ring_wraps_bit_exact(cb, tn):
    """K = 27 (a partial last offset group for GK = 4 and 2) at Ca = cb, Cb = tn: every split wraps the ring three times and ends
    mid-stage, the last one mid-k16-step; both output layouts."""
    K = 27
    n = _rows_wrapping(K, cb, tn, 3)
    gen = torch.Generator(device="cuda").manual_seed(100 * cb + tn)
    tbl = _synth_table(K, n, n, 0.5, gen)
    for tr in (0, 1):
        _run_wgrad_split(K, cb, tn, tr, tbl, n, n, tr == 1, tr == 1, gen, f"K={K} {cb}x{tn} tr={tr} n={n}")


@pytest.mark.parametrize("K", (1, 3, 5, 8))
@pytest.mark.parametrize("Ca,Cb", ((32, 96), (64, 32), (96, 128), (128, 64), (192, 128), (224, 96)))
def test_wgrad_partial_offset_groups_bit_exact(K, Ca, Cb):
    """K below, between and at multiples of the offsets per CTA, with several A channel blocks (192 = 96 x 2, 224 = 32 x 7)."""
    n = _rows_wrapping(K, Ca, Cb, 1)
    gen = torch.Generator(device="cuda").manual_seed(K * 7919 + Ca + Cb)
    tbl = _synth_table(K, n, n, 0.6, gen)
    for tr in (0, 1):
        _run_wgrad_split(K, Ca, Cb, tr, tbl, n, n, tr == 0, tr == 0, gen, f"K={K} {Ca}x{Cb} tr={tr} n={n}")


@pytest.mark.parametrize("Ca,Cb", ((96, 96), (32, 32), (128, 128)))
def test_wgrad_repeatable(Ca, Cb):
    """Two calls on the same random bf16 planes (sums that round) return the same bits."""
    from pointcontrast_b200._lib import check, lib, ptr, stream
    K = 27
    n = _rows_wrapping(K, Ca, Cb, 3)
    gen = torch.Generator(device="cuda").manual_seed(Ca * 31 + Cb)
    tbl = _synth_table(K, n, n, 0.5, gen)
    A = torch.randn(n, Ca, generator=gen, device="cuda")
    B = torch.randn(n, Cb, generator=gen, device="cuda")
    ah = A.bfloat16(); al = (A - ah.float()).bfloat16()
    bh = B.bfloat16(); bl = (B - bh.float()).bfloat16()
    wsb = lib.pcb_conv_wgrad_split_ws_bytes(K, n, Ca, Cb)
    out = []
    for _ in range(2):
        ws = torch.full((max(wsb, 256),), 255, dtype=torch.uint8, device="cuda")
        dw = torch.empty(K, Ca, Cb, device="cuda")
        check(lib.pcb_conv_wgrad_split(ah.data_ptr(), al.data_ptr(), Ca, bh.data_ptr(), bl.data_ptr(), Cb, ptr(tbl), tbl.shape[1], K, n,
                                       Ca, Cb, dw.data_ptr(), 0, ptr(ws), wsb, 0, stream()))
        out.append(dw)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out[0]).all())
    assert torch.equal(out[0], out[1])
