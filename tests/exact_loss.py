"""Split rules, case matrix and exactly representable operands of the PointInfoNCE and hardest-negative tests
(tests/test_gpu_loss_exact.py; the host checks of this module are tests/test_host_loss_geometry.py).

Exactness: every feature is a multiple of 2^-6 and every row has L2 norm <= 1 (the norm limit is the contract of the tensor-core
PointInfoNCE, nce_wgmma.cu).  Then
  * the fp16 hi plane of a feature is the feature itself and the lo plane is zero;
  * every product q_d k_d is a multiple of 2^-12, and every partial sum of a dot product is a multiple of 2^-12 no larger than
    sum_d |q_d k_d| <= |q| |k| <= 1, so it needs at most 13 significant bits: the logit q.k is exact in the wgmma tiles, in the SIMT
    sgemm and in fp64, whatever the order of summation;
  * a squared distance |a - b|^2 is a multiple of 2^-12 below 4 and is exact the same way.
The generators build rows as integers m / 64 with sum_d m_d^2 <= 64^2: a Gaussian direction scaled to a radius <= 1 and truncated toward
zero component by component, which can only shrink the norm.
"""
import torch

GRID = 64                  # features are integers / GRID
YN = 128                   # nce_wgmma.cu: rows per CTA = columns per tile; a tile is two column halves of 64, each four chunks of 16
HALF = 64
PD_TILE = 64               # loss.cu pdist_min_kernel: A rows per CTA = B rows per step


# ----------------------------------------------------------------------------------------------- the library's split rules, restated
def nce_geometry(n, sms):
    """nce_tc_forward_backward: (column tiles, splits, tiles per split).  Split s covers tiles [s tps, min((s + 1) tps, ntiles))."""
    ntiles = -(-n // YN)
    splits = min(max(sms // ntiles, 1), ntiles)          # rowblocks == ntiles
    tps = -(-ntiles // splits)
    return ntiles, -(-ntiles // tps), tps


def nce_split_tiles(n, sms):
    ntiles, splits, tps = nce_geometry(n, sms)
    return [(s * tps, min(ntiles, (s + 1) * tps)) for s in range(splits)]


def nce_reaches(n, sms):
    """The geometries one size reaches on a device with `sms` SMs."""
    ntiles, splits, tps = nce_geometry(n, sms)
    tiles = nce_split_tiles(n, sms)
    out = set()
    if n % YN:
        out.add("partial last tile")
    if splits == 1 and ntiles > 1:
        out.add("single split of several tiles")
    if splits > 1:
        out.add("several splits")
    if splits > 1 and tiles[-1][1] - tiles[-1][0] < tps:
        out.add("short last split")
    for t0, t1 in tiles:
        for h in (0, 1):                                  # a diagonal element in column half h of a split's last tile
            if (t1 - 1) * YN + h * HALF < n:
                out.add(f"diagonal in half {h} of a split's last tile")
    return out


def pdist_geometry(P, S, sms):
    """pcb_pdist_rowmin: (row blocks, S-splits, B rows per split)."""
    rowblocks = -(-P // PD_TILE)
    splits = min(-(-2 * sms // rowblocks), -(-S // PD_TILE))
    splits = max(splits, 1)
    sps = -(-(-(-S // splits)) // PD_TILE) * PD_TILE
    return rowblocks, -(-S // sps), sps


# ----------------------------------------------------------------------------------------------- case matrix
TC_D = (32, 64)
TC_N = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 3000, 4095, 4096, 4097, "128 SMs + 1")
SIMT_D = (1, 16, 33, 96, 128)
SIMT_N = (1, 63, 64, 65, 300)
TEMPS = (0.07, 0.0625, 0.4)
EXACT_T = 0.0625           # 1 / T = 16: the logit scaling is exact as well
PD_P = (1, 63, 64, 65, 4097)
PD_S = (1, 63, 64, 65, 1024, 5000)
PD_D = (1, 3, 16, 32, 64)
SM_COUNTS = (114, 132)     # H100 PCIe, H100 SXM


def tc_size(n, sms):
    return YN * sms + 1 if n == "128 SMs + 1" else n


def nce_seed(D, n, ci):
    return 1000003 * D + 31 * n + ci


# (pattern, T) run for every shape: (a) random at every temperature, (b) every logit <= -0.5 at T = 1/16, (c) k a permutation of q at
# the production temperature, (d) many exactly tied logits
NCE_CASES = tuple(("random", T) for T in TEMPS) + (("negative", EXACT_T), ("permuted", 0.07), ("tied", 0.07))


# ----------------------------------------------------------------------------------------------- generators (CPU, deterministic)
def grid_rows(n, D, gen, rmin=0.5, rmax=1.0):
    """[n, D] fp32 rows m / 64, m integer, |row| <= a radius drawn in [rmin, rmax] (<= 1)."""
    x = torch.randn(n, D, generator=gen, dtype=torch.float64)
    x = x / x.norm(dim=1, keepdim=True).clamp_min(1e-30)
    r = rmin + (rmax - rmin) * torch.rand(n, 1, generator=gen, dtype=torch.float64)
    return (torch.trunc(x * r * GRID) / GRID).float()


NEG_LEAD = 56 / GRID       # pattern (b): q_0 = +7/8, k_0 = -7/8, the other channels of norm <= NEG_REST
NEG_REST = 0.48            # q.k <= -(7/8)^2 + 0.48^2 < -0.53; at 1/T = 16 every logit is below -8.5


def nce_operands(pattern, n, D, seed):
    """(q, k) fp32 [n, D] on the grid for one pattern."""
    gen = torch.Generator().manual_seed(seed)
    if pattern == "random":
        return grid_rows(n, D, gen), grid_rows(n, D, gen)
    if pattern == "negative":
        lead = torch.full((n, 1), NEG_LEAD)
        rq = grid_rows(n, D - 1, gen, 0.0, NEG_REST)
        rk = grid_rows(n, D - 1, gen, 0.0, NEG_REST)
        return torch.cat([lead, rq], 1), torch.cat([-lead, rk], 1)
    if pattern == "permuted":
        q = grid_rows(n, D, gen, 1.0, 1.0)
        return q, q[permutation(n, seed)]
    if pattern == "tied":
        pq, pk = grid_rows(3, D, gen), grid_rows(3, D, gen)
        return pq[torch.randint(0, 3, (n,), generator=gen)], pk[torch.randint(0, 3, (n,), generator=gen)]
    raise ValueError(pattern)


def permutation(n, seed):
    """Pattern (c): k_j = q_pi(j); a random permutation sends rows across column halves, tiles and splits."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed + 1))


def pdist_operands(P, S, D, sps, seed):
    """(A, B) fp32 on the grid.  B holds exact copies of a few anchor rows in the same 64-row tile (+1, +4: another thread, the same
    thread), in a later tile (+64) and in the next S-split (+sps, +sps + 64); A rows are an anchor (distance 0), an anchor with one
    channel moved one grid step toward zero (distance 2^-6, the same for every copy), or random."""
    gen = torch.Generator().manual_seed(seed)
    B = grid_rows(S, D, gen, 0.3, 0.9)
    anchors = [a for a in (0, 10, 19, 27) if a < S]
    for a in anchors:
        for c in (a + 1, a + 4, a + PD_TILE, a + sps, a + sps + PD_TILE):
            if c < S:
                B[c] = B[a]
    A = grid_rows(P, D, gen, 0.3, 0.9)
    for i in range(min(P, 4096)):
        if i % 8 == 7:
            continue
        row = B[anchors[i % len(anchors)]].clone()
        if i % 2:
            nz = torch.nonzero(row).flatten()
            if len(nz):
                d = int(nz[i % len(nz)])
                row[d] -= torch.sign(row[d]) / GRID
        A[i] = row
    return A, B


def on_grid(x):
    """x is integers / 64 with every row's squared norm <= 1, checked in integers."""
    m = x.double() * GRID
    return bool((m == m.round()).all()) and bool(((m.round().long() ** 2).sum(1) <= GRID * GRID).all())
