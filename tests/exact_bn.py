"""Chunk rules, case matrix and exactly representable operands of the BatchNorm tests (tests/test_gpu_bn_exact.py; the host checks of
this module are tests/test_host_bn_geometry.py).

Exactness: every term a kernel sums is a multiple of one quantum q, and the terms of every output sum, in absolute value, to less than
2^24 q.  Then every partial sum is an fp32 number whatever the order of summation: per row lane, per chunk, across chunks (fp64) and
across the two views.
  * Forward statistics (`colstat_kernel<0/2>`) sum a = x - p and a^2 per chunk, p = x[the chunk's first row] (the pivot), then add
    m p back.  Operands are multiples of Q = 2^-3 with |x - p| <= 2 SPREAD = 8 and chunks of at most 1024 rows, so sum|a| <= 2^13 < 2^24 Q,
    sum a^2 <= 2^16 < 2^24 Q^2 and m |p| + sum|a| < 2^24 Q for |p| <= 2000: the chunk's shifted sums and its sum of x are exact.  An
    offset such as 1000 added to the whole matrix stays on the grid: that is the |mean| >> std case the pivot exists for.
    What is left to round is t1 t1 / m and the subtraction forming the chunk's M2 (fp32), the fp64 finalize, the fp64 -> fp32 stores
    and 1 / sqrt(var + (double)eps); test_gpu_bn_exact.py bounds each.  The "zero-sum" pattern makes every chunk's shifted sum t1
    zero (its rows are the pivot and pairs p +- d), so t1 t1 / m and the subtraction are exact as well.
  * Backward sums (`colstat_kernel<1>`): g = dY (masked) on a 2^-2 grid, |g| <= 2, xhat = (x - mean) invstd on a 2^-4 grid, |xhat| <= 4
    (invstd in {1/2, 1}), so every g xhat is a multiple of BQ = 2^-6 and at most 8; dY keeps enough rows zero that a column's terms
    (and the accumulation base) stay below 2^24 BQ over all rows.  dgamma, dbeta and the per-view sums are then exact.
  * Apply (`bn_apply_kernel`): x and the mean on the 2^-3 grid, invstd a power of two, gamma a small multiple of 2^-2, beta and the
    residual on the 2^-3 grid: every y is exact in fp32, fused multiply-add or not.
"""
import functools
import zlib

import torch

LIMIT = 2 ** 24
Q = 2.0 ** -3                  # grid of x, mean, beta and the residual
SPREAD = 4.0                   # |x - offset| <= SPREAD
G_Q, G_MAX = 2.0 ** -2, 2.0    # dY grid and magnitude
BQ = G_Q * Q * 0.5             # quantum of g * xhat (xhat on Q * min(invstd))
INVSTD = (0.5, 1.0)            # backward invstd values: |xhat| <= 2 SPREAD
XHAT_MAX = 2 * SPREAD * max(INVSTD)
APPLY_INVSTD = (0.5, 1.0, 2.0)
GAMMA = (0.5, 0.75, 1.0, 1.25, -1.0)
BASE_MAX = 4.0                 # |accumulate base| of dgamma / dbeta, on the G_Q grid
EPS, MOMENTUM = 1e-5, 0.1

# ----------------------------------------------------------------------------------------------- the library's chunk rules, restated
FIN_PER_LANE = 12              # bn.cu: partials per lane held in registers by the finalize kernels
PREFETCH = 32 * FIN_PER_LANE   # chunks of one view the register prefetch covers; later ones take the plain loops


def chunk_rows(n):
    """bn.cu chunk_rows: a power of two in [16, 1024] near n / 512."""
    t, R = n // 512, 16
    while R < 1024 and R * 3 // 2 < t:
        R <<= 1
    return R


def chunks_of(rows, R):
    return -(-rows // R)


def lanes(C):
    """(channel vectors, row lanes, threads) of one column-statistics CTA."""
    cv = C // 4
    rp = max(1, 256 // cv)
    return cv, rp, cv * rp


def chunk_geometry(n, n0, C):
    """bn.cu chunk_geometry: (R, chunks, chunks0, threads, shared-memory bytes)."""
    R = chunk_rows(n)
    chunks0 = chunks_of(min(n0, n), R)
    _, rp, threads = lanes(C)
    return R, chunks0 + (chunks_of(n - n0, R) if n0 < n else 0), chunks0, threads, rp * 2 * C * 4


def finalize_pass(k):
    """Which finalize loop reads chunk k of a view: 0 = the register prefetch, i >= 1 = iteration i of the plain loop of its lane."""
    return 0 if k < PREFETCH else 1 + (k - PREFETCH) // 32


def segments(n, n0):
    return [(0, n0), (n0, n)] if n0 < n else [(0, n)]


def row_chunks(n, n0):
    """Per row: (global chunk index, first row of its chunk, rows in its chunk, index within the chunk), as int64 tensors."""
    R, _, chunks0, _, _ = chunk_geometry(n, n0, 4)
    cid, first, size, j = (torch.empty(n, dtype=torch.long) for _ in range(4))
    for s, (a, e) in enumerate(segments(n, n0)):
        r = torch.arange(a, e)
        loc = (r - a) // R
        cid[a:e] = loc + (chunks0 if s else 0)
        first[a:e] = a + loc * R
        size[a:e] = torch.clamp(e - first[a:e], max=R)
        j[a:e] = r - first[a:e]
    return cid, first, size, j


# ----------------------------------------------------------------------------------------------- shapes
MODELS = ("Res16UNet14", "Res16UNet18", "Res16UNet34", "Res16UNet34C")


@functools.lru_cache(None)
def model_bn_widths(name):
    """The width of every BatchNorm of the model (built on the meta device: no data)."""
    from pointcontrast_b200 import me
    from pointcontrast_b200.model import load_model
    from tests.refload import default_config
    with torch.device("meta"):
        net = load_model(name)(3, 32, default_config(), D=3)
    return tuple(m.bn.num_features for m in net.modules() if isinstance(m, me.MinkowskiBatchNorm))


@functools.lru_cache(None)
def bn_widths():
    return tuple(sorted({c for name in MODELS for c in model_bn_widths(name)}))


# Statistics cases: (name, n0, n1, C, offset, pattern); n1 == 0 is one view.  Chunk counts per view in the names are at that n's R.
STATS_CASES = (
    ("one row", 1, 0, 32, 0.0, "random"),
    ("383 chunks, R 16", 6128, 0, 32, 0.0, "zero-sum"),
    ("384 chunks", 6144, 0, 12, 1000.0, "random"),
    ("385 chunks, one-row last chunk", 6145, 0, 20, -1000.0, "zero-sum"),
    ("782 chunks, R 1024", 800_001, 0, 16, 1000.0, "random"),
    ("384 | 385 chunks, R 16", 6144, 6145, 4, 0.0, "random"),
    ("385 | 384 chunks, R 16, C 1024", 6145, 6144, 1024, 1000.0, "zero-sum"),
    ("431 | 421 chunks, R 1024, one-row last chunks", 430 * 1024 + 1, 420 * 1024 + 1, 8, 1000.0, "random"),
    ("431 | 421 chunks, zero-sum", 430 * 1024 + 1, 420 * 1024 + 1, 4, -1000.0, "zero-sum"),
    ("383 | one-row view, C 1024", 6123, 1, 1024, 1000.0, "random"),
    ("one-row view | 313", 1, 5000, 64, 0.0, "zero-sum"),
    ("40 | 351 chunks, R 256", 40 * 256, 89_760, 96, 1000.0, "random"),
    ("40 | 351 chunks, R 256, zero-sum", 40 * 256, 89_760, 32, 0.0, "zero-sum"),
)


@functools.lru_cache(None)
def width_cases():
    """Every BatchNorm width of the models, at two views of 1700 | 1300 rows (and the |mean| >> std offset on every other width)."""
    return tuple((f"width {C}", 1700, 1300, C, 1000.0 * (i % 2), "random") for i, C in enumerate(bn_widths()))


def stats_cases():
    return STATS_CASES + width_cases()


def reaches(n0, n1, C):
    """The geometry properties one statistics case reaches."""
    n = n0 + n1
    R, chunks, chunks0, threads, _ = chunk_geometry(n, n0 if n1 else n, C)
    out = {f"R {R}" if R in (16, 1024) else "R between"}
    _, rp, _ = lanes(C)
    out |= {"rp 1"} if rp == 1 else set()
    out |= {"rp 256"} if rp == 256 else set()
    out |= {"threads not a multiple of 32"} if threads % 32 else set()
    out |= {"two views"} if n1 else {"one view"}
    out |= {"n0 % R == 0"} if n1 and n0 % R == 0 else set()
    out |= {"n0 % R != 0"} if n1 and n0 % R else set()
    for s, rows in enumerate((n0, n1) if n1 else (n0,)):
        ch = chunks_of(rows, R)
        tag = f"view {s}: " if n1 else ""
        out.add(tag + ("< 384 chunks" if ch < PREFETCH else "384 chunks" if ch == PREFETCH else "385 chunks" if ch == PREFETCH + 1
                       else "> 416 chunks" if ch > PREFETCH + 32 else "386..416 chunks"))
        out |= {tag + "one-row view"} if rows == 1 else set()
        out |= {tag + "one-row last chunk"} if rows % R == 1 and rows > 1 else set()
    return out


# Backward cases: (name, n0, n1, C)
BACKWARD_CASES = (
    ("one view", 3001, 0, 32),
    ("two views, C 12", 2000, 1777, 12),
    ("one-row view", 1, 900, 64),
    ("431 | 421 chunks, R 1024", 430 * 1024 + 1, 420 * 1024 + 1, 8),
    ("385 | 384 chunks, R 16", 6145, 6144, 64),
    ("one view, C 1024", 3000, 0, 1024),
)
# Apply cases: (name, n0, n1, C)
APPLY_CASES = (("one view", 999, 0, 32), ("two views, C 4", 130, 77, 4), ("two views, C 96", 1000, 1001, 96), ("two views, C 20", 1, 65, 20))


# ----------------------------------------------------------------------------------------------- generators (CPU, deterministic)
def seed_of(name):
    return zlib.crc32(name.encode())


def _grid(shape, gen, k):
    return torch.randint(-k, k + 1, shape, generator=gen).double() * Q


def stats_operand(n0, n1, C, offset, pattern, seed):
    """fp32 [n, C] on the Q grid, |x - offset| <= SPREAD.  "zero-sum": every chunk is its first row p and pairs p + d, p - d (a last
    unpaired row is p), so its shifted sum is zero."""
    n = n0 + n1
    gen = torch.Generator().manual_seed(seed)
    kmax = int(SPREAD / Q)
    if pattern == "random":
        return (offset + _grid((n, C), gen, kmax)).float()
    assert pattern == "zero-sum"
    _, first, size, j = row_chunks(n, n0 if n1 else n)
    pivot = offset + _grid((n, C), gen, kmax // 2)
    d = _grid((n, C), gen, kmax // 2)
    partner = j + torch.where(j % 2 == 1, 1, -1)          # rows 2i + 1, 2i + 2 of a chunk form a pair
    start = torch.where(j % 2 == 1, torch.arange(n), torch.arange(n) - 1)
    lone = (j == 0) | (partner >= size)
    sign = torch.where(j % 2 == 1, 1.0, -1.0).double()
    x = pivot[first] + sign[:, None] * d[start.clamp(min=0)]
    x[lone] = pivot[first[lone]]
    return x.float()


def stats_terms(x, n0):
    """Per chunk and channel, in units of the exactness limit: max of sum|a| / (2^24 Q), sum a^2 / (2^24 Q^2) and
    (m |p| + sum|a|) / (2^24 Q); and whether x is on the grid.  < 1 everywhere means the chunk sums are exact."""
    n, C = x.shape
    cid, first, size, _ = row_chunks(n, n0)
    xd = x.double()
    a = xd - xd[first]
    nch = int(cid.max()) + 1
    s1 = torch.zeros(nch, C, dtype=torch.float64).index_add_(0, cid, a.abs())
    s2 = torch.zeros(nch, C, dtype=torch.float64).index_add_(0, cid, a * a)
    starts = torch.unique(first)
    p = xd[starts].abs() * size[starts, None].double()
    worst = torch.stack([s1 / (LIMIT * Q), s2 / (LIMIT * Q * Q), (p + s1) / (LIMIT * Q)]).max()
    return float(worst), bool((xd / Q == (xd / Q).round()).all())


def chunk_shifted_sums(x, n0):
    """The exact shifted sums t1 of every chunk (fp64 [chunks, C])."""
    n, C = x.shape
    cid, first, _, _ = row_chunks(n, n0)
    xd = x.double()
    return torch.zeros(int(cid.max()) + 1, C, dtype=torch.float64).index_add_(0, cid, xd - xd[first])


def backward_density(n):
    """Fraction of nonzero dY rows such that a column's |terms| (at most G_MAX XHAT_MAX each) and the base stay below 2^24 BQ."""
    room = LIMIT * BQ - BASE_MAX
    return min(1.0, 0.9 * room / (G_MAX * XHAT_MAX * n))


def backward_operands(n0, n1, C, seed):
    """(x, dY, mean [2, C], invstd [2, C], gamma, dgamma base, dbeta base, gout base): x within SPREAD of its view's mean."""
    n = n0 + n1
    gen = torch.Generator().manual_seed(seed)
    kmax = int(SPREAD / Q)
    mean = 1000.0 * (torch.arange(2)[:, None] - 0.5) + _grid((2, C), gen, 64)
    view = (torch.arange(n) >= n0).long() if n1 else torch.zeros(n, dtype=torch.long)
    x = mean[view] + _grid((n, C), gen, kmax)
    invstd = torch.tensor(INVSTD, dtype=torch.float64)[torch.randint(0, len(INVSTD), (2, C), generator=gen)]
    dy = torch.randint(-int(G_MAX / G_Q), int(G_MAX / G_Q) + 1, (n, C), generator=gen).double() * G_Q
    dy *= (torch.rand(n, 1, generator=gen) < backward_density(n)).double()
    gamma = torch.tensor(GAMMA, dtype=torch.float64)[torch.randint(0, len(GAMMA), (C,), generator=gen)]
    base = lambda k: torch.randint(-k, k + 1, (C,), generator=gen).double() * G_Q
    gbase = torch.randint(-16, 17, (n, C), generator=gen).double() * G_Q
    return (x.float(), dy.float(), mean.float(), invstd.float(), gamma.float(), base(int(BASE_MAX / G_Q)).float(),
            base(int(BASE_MAX / G_Q)).float(), gbase.float())


def backward_terms(x, dy, mean, invstd, n0, base):
    """max over columns of (sum |g xhat| + |base|) / (2^24 BQ), with g = dY unmasked (the mask only removes terms)."""
    n = x.shape[0]
    view = (torch.arange(n) >= n0).long()
    xhat = (x.double() - mean.double()[view]) * invstd.double()[view]
    t = (dy.double() * xhat).abs().sum(0) + base.double().abs()
    return float(t.max() / (LIMIT * BQ)), bool(((xhat / (Q * min(INVSTD))).frac() == 0).all())


def apply_operands(n0, n1, C, seed):
    """(x, mean [2, C], invstd [2, C], gamma, beta, residual) whose apply output is exact in fp32."""
    n = n0 + n1
    gen = torch.Generator().manual_seed(seed)
    mean = _grid((2, C), gen, 32) + torch.tensor([[-3.0], [5.0]], dtype=torch.float64)
    x = _grid((n, C), gen, 48)
    invstd = torch.tensor(APPLY_INVSTD, dtype=torch.float64)[torch.randint(0, len(APPLY_INVSTD), (2, C), generator=gen)]
    gamma = torch.tensor(GAMMA, dtype=torch.float64)[torch.randint(0, len(GAMMA), (C,), generator=gen)]
    beta, res = _grid((C,), gen, 16), _grid((n, C), gen, 16)
    return tuple(t.float() for t in (x, mean, invstd, gamma, beta, res))


def plane_palette(n, C, seed):
    """fp32 [n, C]: the edges of the 16-bit plane formats (fp16 range and clamp, fp16 subnormals and below, bf16 and fp16 ties, an fp32
    subnormal, magnitudes near fp32's limit) among random fp32 values of every magnitude."""
    edges = [0.0, 1.0, -1.0, 2.0 ** -24, -2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -30, -2.0 ** -30, 1e-40, 2.0 ** -14,
             2.0 ** -14 - 2.0 ** -24, 65000.0, 65008.0, 65504.0, 65519.0, 65520.0, 70000.0, -70000.0, 1e30, -3e38, 1 + 2.0 ** -8,
             1 + 3 * 2.0 ** -8, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 3.14159265, -0.1, 1234.5678]
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, C, generator=gen, dtype=torch.float64) * torch.exp2(torch.randint(-40, 40, (n, C), generator=gen).double())
    flat = x.view(-1)
    m = min(len(edges), flat.numel())
    flat[:m] = torch.tensor(edges[:m], dtype=torch.float64)
    return x.float()


def mask_codes(n, C, fmt, seed):
    """uint16 codes of a 16-bit hi plane (`fmt` "bf16" or "fp16"): +0, -0, the smallest and largest subnormals, the smallest normal,
    one, the largest finite, infinity and NaN, each with both signs, among random codes."""
    one, top = (0x3F80, 0x7F7F) if fmt == "bf16" else (0x3C00, 0x7BFF)
    normal, inf, nan = (0x0080, 0x7F80, 0x7FC0) if fmt == "bf16" else (0x0400, 0x7C00, 0x7E00)
    edges = [0x0000, 0x0001, normal - 1, normal, one, top, inf, nan]
    edges = edges + [e | 0x8000 for e in edges]
    gen = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, 1 << 16, (n, C), generator=gen, dtype=torch.int32)
    pick = torch.randint(0, len(edges), (n, C), generator=gen)
    use = torch.rand(n, C, generator=gen) < 0.5
    codes = torch.where(use, torch.tensor(edges, dtype=torch.int32)[pick], codes)
    return codes.to(torch.int16)


def mask_passes(codes):
    """include/pcb200.h: relu > 0 <=> the hi plane's sign bit is clear and it is not zero."""
    c = codes.to(torch.int32) & 0xFFFF
    return ((c & 0x8000) == 0) & (c != 0)
