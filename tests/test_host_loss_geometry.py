"""Host checks of the exact loss tests (tests/test_gpu_loss_exact.py, operands and rules in tests/exact_loss.py): the generators stay on
the grid that makes the PointInfoNCE logits and the squared distances exact, and the case matrix reaches every split geometry of the two
kernels on an H100 SXM (132 SMs) and an H100 PCIe (114 SMs)."""
import pytest
import torch

from tests import exact_loss as X

REQUIRED = {"partial last tile", "single split of several tiles", "several splits", "short last split",
            "diagonal in half 0 of a split's last tile", "diagonal in half 1 of a split's last tile"}


def _shapes():
    return [("tc", D, n) for D in X.TC_D for n in X.TC_N] + [("simt", D, n) for D in X.SIMT_D for n in X.SIMT_N]


@pytest.mark.parametrize("sms", X.SM_COUNTS)
def test_split_rule_restated(sms):
    """Hand-checked values of the restated rule: n = 3000 has a short last split and 128 SMs + 1 rows a single split."""
    assert X.nce_geometry(3000, 132) == (24, 5, 5) and X.nce_split_tiles(3000, 132)[-1] == (20, 24)
    assert X.nce_geometry(4096, 132) == (32, 4, 8) and X.nce_geometry(4096, 114) == (32, 3, 11)
    assert X.nce_geometry(1, sms) == (1, 1, 1)
    n = X.tc_size("128 SMs + 1", sms)
    assert X.nce_geometry(n, sms) == (sms + 1, 1, sms + 1)
    for n in range(1, 40 * X.YN, 37):
        ntiles, splits, tps = X.nce_geometry(n, sms)
        tiles = X.nce_split_tiles(n, sms)
        assert tiles[0][0] == 0 and tiles[-1][1] == ntiles and all(a[1] == b[0] for a, b in zip(tiles, tiles[1:]))
        assert all(0 < t1 - t0 <= tps for t0, t1 in tiles) and len(tiles) == splits
        assert splits * ntiles <= sms or splits == 1              # at most one wave of (row block, split) CTAs


@pytest.mark.parametrize("sms", X.SM_COUNTS)
def test_tensor_core_case_matrix_reaches_every_geometry(sms):
    seen = {}
    for n in X.TC_N:
        for g in X.nce_reaches(X.tc_size(n, sms), sms):
            seen.setdefault(g, []).append(n)
    assert set(seen) >= REQUIRED, (sms, sorted(seen))
    assert {n % X.YN for n in map(lambda n: X.tc_size(n, sms), X.TC_N)} >= {0, 1, 63, 64, 65, 127}


@pytest.mark.parametrize("sms", X.SM_COUNTS)
def test_permutation_moves_rows_across_halves_tiles_and_splits(sms):
    """Pattern (c): the key of a row's largest logit lies in the other column half of the same tile, in another tile of the same split
    and in another split, for some row of the case matrix."""
    seen = set()
    for n in X.TC_N:
        n = X.tc_size(n, sms)
        for D in X.TC_D:
            ci = [c[0] for c in X.NCE_CASES].index("permuted")
            pi = X.permutation(n, X.nce_seed(D, n, ci))
            i = torch.arange(n)
            col = torch.empty(n, dtype=torch.long)
            col[pi] = i                                        # row i's key sits in column pi^-1(i)
            _, _, tps = X.nce_geometry(n, sms)
            seen |= {"other half"} if bool(((col // X.YN == i // X.YN) & (col // X.HALF != i // X.HALF)).any()) else set()
            seen |= {"other tile"} if bool(((col // X.YN != i // X.YN) & (col // (X.YN * tps) == i // (X.YN * tps))).any()) else set()
            seen |= {"other split"} if bool((col // (X.YN * tps) != i // (X.YN * tps)).any()) else set()
    assert seen == {"other half", "other tile", "other split"}


@pytest.mark.parametrize("path,D,n", _shapes())
def test_every_nce_case_is_exact(path, D, n):
    """Every operand the GPU file builds: on the grid, norm <= 1 (so every logit is exact), fp16 hi plane = the value; pattern (b) keeps
    every logit <= -0.5 at T = 1/16, and pattern (d) repeats logits."""
    for sms in (X.SM_COUNTS if n == "128 SMs + 1" else X.SM_COUNTS[:1]):
        nn = X.tc_size(n, sms)
        for ci, (pattern, T) in enumerate(X.NCE_CASES):
            q, k = X.nce_operands(pattern, nn, D, X.nce_seed(D, nn, ci))
            assert q.shape == k.shape == (nn, D) and q.dtype == k.dtype == torch.float32
            assert X.on_grid(q) and X.on_grid(k), (pattern, nn, D)
            assert torch.equal(q.half().float(), q) and torch.equal(k.half().float(), k)
            if nn <= 4097:
                S = (q.double() * X.GRID) @ (k.double() * X.GRID).T          # integers: S / 2^12 is the exact dot product
                if pattern == "negative":
                    assert float(S.max()) / X.GRID ** 2 / X.EXACT_T <= -0.5
                if pattern == "tied" and nn > 9:
                    assert len(torch.unique(S)) <= 9
            assert bool((q != 0).any())


@pytest.mark.parametrize("sms", X.SM_COUNTS)
def test_pdist_case_matrix_reaches_every_split_geometry(sms):
    seen = set()
    for P in X.PD_P:
        for S in X.PD_S:
            rowblocks, splits, sps = X.pdist_geometry(P, S, sms)
            assert (splits - 1) * sps < S <= splits * sps and sps % X.PD_TILE == 0
            seen |= {"one split"} if splits == 1 else {"several splits"}
            seen |= {"split of several tiles"} if sps > X.PD_TILE and S > X.PD_TILE else set()
            seen |= {"partial B tile"} if S % X.PD_TILE else set()
            seen |= {"partial A block"} if P % X.PD_TILE else set()
            seen |= {"several A blocks and splits"} if rowblocks > 1 and splits > 1 else set()
    assert seen == {"one split", "several splits", "split of several tiles", "partial B tile", "partial A block",
                    "several A blocks and splits"}


@pytest.mark.parametrize("S", X.PD_S)
def test_pdist_operands_are_exact_and_plant_copies(S):
    for P in (1, 65):
        for D in X.PD_D:
            _, splits, sps = X.pdist_geometry(P, S, 132)
            A, B = X.pdist_operands(P, S, D, sps, seed=S + D)
            assert X.on_grid(A) and X.on_grid(B)
            assert torch.equal(A[0], B[0])
            for c in (1, 4, X.PD_TILE, sps, sps + X.PD_TILE):
                if c < S:
                    assert torch.equal(B[c], B[0]), (S, D, c)


def test_pdist_rejects_more_than_64_channels():
    """D = 65 is an argument error, returned before anything touches the (fake) pointers."""
    from pointcontrast_b200 import _lib
    fake = 256
    assert _lib.lib.pcb_pdist_rowmin(fake, 1, fake, 1, 65, fake, fake, fake, None) == _lib.ERR_ARG
    assert b"bad argument" in _lib.lib.pcb_last_error()
    assert _lib.lib.pcb_pdist_rowmin(fake, 1, fake, 1, 0, fake, fake, fake, None) == _lib.ERR_ARG
