"""Tile orders of the sparse-convolution kernel (`pcb_conv_tile_order`, `pcb_conv_forward_split_ordered`).

The order is checked against a numpy recount from the same table: a stable sort of the rows by (row / window, neighbour mask), every
128-row tile inside one window, the same bytes on every build, and the offsets each tile stages.  The ordered convolution is held to
the identity order bit for bit at every tile geometry the executor issues (tests/exact_conv.py: BN 128 / 96 / 64 / 32, forward and data
gradient, bf16 and fp16 operands, bias and accumulation, offset-split and direct mode with a tail tile): on exactly representable
operands against the fp64 sum, and in direct mode also on random operands, where only the same per-row summation order gives the same
bits."""
import numpy as np
import pytest
import torch

from pointcontrast_b200 import _lib
from tests import exact_conv as X

BM = 128


def _order(tbl, n, window):
    from pointcontrast_b200._lib import check, lib, ptr, stream
    ws = torch.empty(lib.pcb_conv_tile_order_ws_bytes(n), dtype=torch.uint8, device="cuda")
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    check(lib.pcb_conv_tile_order(ptr(tbl), tbl.shape[1], tbl.shape[0], n, window, ptr(perm), ptr(ws), ws.numel(), stream()))
    return perm


def _np_order(tbl, n, window):
    """(perm, mask per row): the stable sort of rows [0, n) of the table by (row // window, mask)."""
    t = tbl[:, :n].cpu().numpy()
    mask = ((t >= 0).astype(np.int64) << np.arange(t.shape[0])[:, None]).sum(0)
    key = ((np.arange(n) // window) << 32) | mask
    return np.argsort(key, kind="stable"), mask


def offsets_per_tile(mask, order):
    """Kernel offsets each 128-row tile stages: the popcount of the OR of its rows' masks."""
    m = np.concatenate([mask[order], np.zeros(-len(order) % BM, np.int64)]).reshape(-1, BM)
    u = np.bitwise_or.reduce(m, axis=1)
    return np.array([bin(int(v)).count("1") for v in u])


def test_tile_order_rejects_bad_arguments():
    """Window not a multiple of 128, too many offsets, a table narrower than n_out: PCB_ERR_ARG before the device is touched."""
    L = _lib.lib
    n = 1000
    wsb = L.pcb_conv_tile_order_ws_bytes(n)
    assert wsb > 0
    fake = 1 << 20          # never dereferenced: the checks return first
    assert L.pcb_conv_tile_order(fake, n, 27, n, 1000, fake, fake, wsb, None) == _lib.ERR_ARG
    assert L.pcb_conv_tile_order(fake, n, 28, n, 1024, fake, fake, wsb, None) == _lib.ERR_ARG
    assert L.pcb_conv_tile_order(fake, n - 1, 27, n, 1024, fake, fake, wsb, None) == _lib.ERR_ARG
    assert L.pcb_conv_tile_order(None, n, 27, 0, 1024, None, None, 0, None) == _lib.OK


@pytest.fixture(scope="module")
def scene():
    """Neighbour tables of a surface scene large enough for direct-mode launches on both levels: hybrid 3x3x3 (fine rows), stride-2
    2x2x2 down (coarse rows) and up (fine rows); (table, source rows, data-gradient kmap) per (kind, role) as the executor uses them."""
    from pointcontrast_b200 import me
    from tests.helpers import surface_coords
    coords = surface_coords(np.random.default_rng(11), 160_000, extent=120)
    st = me.SparseTensor(torch.zeros(len(coords), 1, device="cuda"), coords=torch.from_numpy(coords))
    cm, fine = st.coords_man, st.coords_key
    coarse = cm.stride(fine, [2, 2, 2])
    hyb = me.KernelGenerator(3, 1, 1, region_type=me.RegionType.HYBRID, axis_types=[me.RegionType.HYPERCUBE] * 3, dimension=3)
    p27 = cm.conv_plan(fine, fine, hyb, False)
    p8 = cm.conv_plan(fine, coarse, me.KernelGenerator([2, 2, 2], 2, 1, dimension=3), False)
    nf, nc = cm.num_rows(fine), cm.num_rows(coarse)
    return {("k27", "fwd"): (p27.fwd_tbl, nf, None), ("k27", "dgrad"): (p27.dg_tbl, nf, p27.dg_kmap),
            ("down", "fwd"): (p8.fwd_tbl, nf, None), ("down", "dgrad"): (p8.dg_tbl, nc, None),
            ("up", "fwd"): (p8.dg_tbl, nc, None), ("up", "dgrad"): (p8.fwd_tbl, nf, None)}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["k27", "down", "up"])
def test_tile_order_matches_numpy_recount(scene, kind):
    """perm is the stable (window, mask) sort, a permutation whose tiles stay inside one window, the same bytes on every build; the
    offsets per tile equal the numpy recount and never exceed the identity order's."""
    from pointcontrast_b200 import me
    tbl = scene[(kind, "fwd")][0]
    n_full = tbl.shape[1]
    for n in (n_full, n_full - 77):                     # all rows; a prefix of a wider table (stride > n_out) with a tail tile
        for window in (128, 1024, me.TILE_ORDER_WINDOW, -(-n // BM) * BM):
            what = f"{kind} n={n} window={window}"
            perm = _order(tbl, n, window)
            want, mask = _np_order(tbl, n, window)
            got = perm.cpu().numpy()
            assert np.array_equal(np.sort(got), np.arange(n)), what
            assert np.array_equal(got, want), what
            # position i holds a row of window i // window; windows are whole tiles, so every tile stays inside one window
            assert np.array_equal(got // window, np.arange(n) // window), what
            ordered, ident = offsets_per_tile(mask, got), offsets_per_tile(mask, np.arange(n))
            assert np.array_equal(ordered, offsets_per_tile(mask, want)), what
            if window >= 1024:
                assert ordered.sum() < ident.sum(), what


def _ws(nbytes):
    return torch.full((max(nbytes, 256),), 255, dtype=torch.uint8, device="cuda")


def _conv(fmt, K, Ck, N, tiles, xh, xl, tbl, kmap, perm, n_out, bias, base):
    from pointcontrast_b200._lib import check, lib, ptr, stream
    from tests.test_gpu_conv_exact import _kmap_arg
    Y = torch.zeros(n_out + 1, N, device="cuda") if base is None else torch.cat([base, base.new_zeros(1, N)])
    wsb = lib.pcb_conv_forward_split_ws_bytes(K, n_out, Ck, N)
    ws = _ws(wsb)
    flags = fmt.flags | (_lib.CONV_ACCUMULATE if base is not None else 0)
    check(lib.pcb_conv_forward_split_ordered(xh.data_ptr(), xl.data_ptr(), Ck, ptr(tbl), tbl.shape[1], _kmap_arg(kmap), K, ptr(perm), n_out,
                                             Ck, N, ptr(tiles), ptr(bias), Y.data_ptr(), N, ptr(ws), wsb, flags, stream()))
    assert bool((Y[n_out] == 0).all()), "row past n_out written"
    return Y[:n_out]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _case_id(c):
    kind, K, Cin, Cout, role, fmt = c
    return f"{kind}-{Cin}x{Cout}-{role}-{fmt}"


CASES = [(ci, c) for ci, c in enumerate(X.forward_cases()) if c[0] != "k1"]        # a 1-offset kernel has nothing to reorder


@pytest.mark.gpu
@pytest.mark.parametrize("ci,case", CASES, ids=[_case_id(c) for _, c in CASES])
def test_ordered_conv_bit_identical_to_identity(scene, ci, case):
    """Every shape and role, on the coordinate manager's table in the executor's tile order: offset-split mode (1, 127, 128, 129 rows)
    and direct mode (a tail tile) on exact operands against fp64, and direct mode on random operands against the identity order."""
    from pointcontrast_b200 import me
    from tests.test_gpu_conv_exact import _assert_exact, _ref_forward, _weights_and_tiles
    kind, K, Cin, Cout, role, fname = case
    fmt = X.FMTS[fname]
    Ck, N = X.contraction(case)
    gen = torch.Generator(device="cuda").manual_seed(5000 + ci)
    ft, dt, wh, wl = _weights_and_tiles(K, Cin, Cout, fmt, gen)
    tiles = ft if role == "fwd" else dt
    if role == "dgrad":
        wh, wl = wh.transpose(1, 2).contiguous(), wl.transpose(1, 2).contiguous()
    tbl, n_src, kmap = scene[(kind, role)]
    direct = X.direct_rows(N, _sms())
    assert direct <= tbl.shape[1] and direct % BM
    for n_out, use_bias, acc in ((1, False, False), (127, True, False), (128, False, True), (129, True, True),
                                 (direct, ci % 2 == 0, ci % 2 == 1)):
        what = f"{_case_id(case)} rows={n_out} bias={use_bias} accumulate={acc}"
        perm = _order(tbl, n_out, me.TILE_ORDER_WINDOW)
        hi, lo = X.capped_planes(n_src, Ck, X.row_cap(fmt, K, Ck), fmt.HI, fmt.LO, gen, "cuda")
        bias = X.bias_values(N, fmt, gen, "cuda") if use_bias else None
        base = X.bias_values(n_out * N, fmt, gen, "cuda").view(n_out, N) if acc else None
        got = _conv(fmt, K, Ck, N, tiles, hi.to(fmt.dtype), lo.to(fmt.dtype), tbl, kmap, perm, n_out, bias, base)
        y, _ = _ref_forward(hi.double(), lo.double(), wh, wl, tbl, kmap, n_out)
        want = y * fmt.SCALE
        for extra in (bias[None] if bias is not None else None, base):
            if extra is not None:
                want = want + extra.double()
        _assert_exact(got, want, what)
        if n_out == direct:
            assert X.conv_splits(K, n_out, Ck, N, _sms()) == 1, what
            xr = torch.randn(n_src, Ck, generator=gen, device="cuda")
            rh = xr.to(fmt.dtype)
            rl = (xr - rh.float()).to(fmt.dtype)
            a = _conv(fmt, K, Ck, N, tiles, rh, rl, tbl, kmap, perm, n_out, bias, base)
            b = _conv(fmt, K, Ck, N, tiles, rh, rl, tbl, kmap, None, n_out, bias, base)
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what + ": random operands differ from the identity order"
