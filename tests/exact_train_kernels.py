"""Case lists, operand generators and host restatements of the training-step kernel tests (tests/test_gpu_train_kernels_exact.py;
the host checks of this module are tests/test_host_train_kernels.py): the semantic-segmentation cross-entropy, the L2 normalisation of
the output features, the flat SGD step and the pooling gather-sum.

Exactly representable operands
  * Cross-entropy: "dominated" rows.  Every logit is an integer of magnitude <= 10^4; each row has one maximum M and every other entry
    is -inf or at most M - 200.  Then x - M is exact, expf gives exactly 1 at the maximum and 0 elsewhere (e^-200 is far below half the
    smallest subnormal), the row sum is exactly 1, logf(1) = 0, lse = M and the row loss M - x_t is an integer: the loss is the fp64
    mean of integers rounded once, and every gradient entry is 0 or +-fp32(grad_scale / count).
  * L2 normalisation: rows whose sum of squares is a power of 4 -- 4^a entries of +-2^j (a + j <= 11) in random columns, zeros
    elsewhere.  Every partial sum of squares is a multiple of 4^j below 2^24 times it, sqrtf and the reciprocal are exact, so
    y = +-2^-a and inv_norm = 2^-(a + j) exactly.  dy is a multiple of 2^-8 below 2^-2: y dy, their sums, y (y . dy), the difference
    and the power-of-two scaling all fit in 24 bits (at most 2^2 with a grid of 2^-16).
  * SGD: p, g multiples of 2^-10 below 2 and 1, lr = 2^-4, weight_decay = 2^-10, grad_scale and 1 - dampening powers of two: every
    product but momentum * buf is exact, and so is momentum * buf when momentum = 0.5.  See sgd_restate.
  * Gather-sum: small integers; every sum is exact in any order.
"""
import numpy as np
import torch

# ----------------------------------------------------------------------------------------------- cross-entropy
CE_C = (1, 2, 13, 20, 31, 32, 33, 64, 255, 1024)
CE_SMALL_N = (1, 7, 8, 9)
CE_BIG_N = 1_000_003                 # a semseg batch: n = 3 mod 8 (a partial last CTA of 8 rows)
CE_BIG_C = (13, 20, 33)              # the batch size at the finetune class counts and one width past a lane pass
CE_WIDE_N = 4099                     # the wide rows (C >= 64) at n = 3 mod 8, n C <= 2^22
GRAD_SCALES = (1.0, 0.5, 1.0 / 3.0)
CE_MIXES = ("valid", "ignore 255", "ignore inside", "out of range", "all ignored")
OUT_OF_RANGE = (-1, -5)              # with C itself
MARGIN = 200                         # dominated rows: every non-maximal entry is at most M - MARGIN (or -inf)
XMAX = 10_000


def ce_n_list(C):
    big = CE_BIG_N if C in CE_BIG_C else (CE_WIDE_N if C >= 64 else None)
    return CE_SMALL_N + ((big,) if big else ())


def ce_ignore(mix, C):
    """The ignore_index of a mix: 255, or a class inside [0, C) for "ignore inside" (255 itself is inside when C > 255)."""
    return (C // 2) if mix == "ignore inside" else 255


def ce_targets(mix, n, C, gen):
    """int64 [n] targets of a mix (CPU, deterministic).  Every mix but "valid" holds some rows of its kind; "out of range" holds C, -1
    and -5 and some 255-ignored rows."""
    t = torch.randint(0, C, (n,), generator=gen, dtype=torch.int64)
    ign = ce_ignore(mix, C)
    r = torch.rand(n, generator=gen)
    if mix == "all ignored":
        return torch.full((n,), ign, dtype=torch.int64)
    if mix in ("ignore 255", "ignore inside"):
        t[r < 0.3] = ign
        if n > 1:
            t[0] = ign
    elif mix == "out of range":
        bad = torch.tensor((C,) + OUT_OF_RANGE, dtype=torch.int64)
        sel = r < 0.4
        t[sel] = bad[torch.randint(0, 3, (int(sel.sum()),), generator=gen)]
        t[(r >= 0.4) & (r < 0.5)] = 255           # the ignore_index: inside [0, C) when C > 255
        t[: min(n, 3)] = bad[: min(n, 3)]
    return t


def ce_valid(t, C, ignore):
    return (t != ignore) & (t >= 0) & (t < C)


def ce_dominated(t, C, gen):
    """Exactly representable logits [n, C] (see the module docstring) for targets t: the maximum in a random column, and (rows % 3)
    the target at the maximum, the target elsewhere, or -inf in the non-target columns that are not the maximum."""
    n = t.shape[0]
    M = torch.randint(-XMAX // 2 + 2 * MARGIN, XMAX, (n, 1), generator=gen).double()
    x = M - MARGIN - torch.randint(0, XMAX // 2, (n, C), generator=gen).double()          # >= -XMAX
    jmax = torch.randint(0, C, (n,), generator=gen)
    valid = (t >= 0) & (t < C)
    rows = torch.arange(n)
    kind = rows % 3
    jmax = torch.where(valid & (kind == 0), t, jmax)
    if C > 1:                                     # the target elsewhere than the maximum
        other = (jmax + 1 + torch.randint(0, C - 1, (n,), generator=gen)) % C
        jmax = torch.where(valid & (kind == 1) & (jmax == t), other, jmax)
    x[rows, jmax] = M[:, 0]
    neg = (kind == 2)[:, None] & (torch.rand(n, C, generator=gen) < 0.5)
    cols = torch.arange(C)[None]
    neg &= cols != jmax[:, None]
    neg &= ~(valid[:, None] & (cols == t.clamp(0, C - 1)[:, None]))
    x[neg] = -np.inf
    return x.float(), jmax


def ce_dominated_expected(x, t, jmax, C, ignore, grad_scale):
    """(loss fp32, dlogits fp32) of dominated logits, from integer arithmetic and one fp32 division."""
    v = ce_valid(t, C, ignore)
    n = t.shape[0]
    rows = torch.arange(n)
    tl = t.clamp(0, C - 1)
    rowloss = torch.where(v, x[rows, jmax].double() - x[rows, tl].double(), 0.0)
    cnt = int(v.sum())
    loss = np.float32(float(rowloss.sum()) / cnt) if cnt else np.float32(np.nan)
    q = np.float32(grad_scale) / np.float32(cnt) if cnt else np.float32(0)
    g = torch.zeros(n, C, dtype=torch.float32)
    g[rows[v], jmax[v]] = float(q)
    g[rows[v], tl[v]] -= float(q)
    return loss, g


def ce_edge_logits(t, C, gen):
    """Random logits [n, C] with the edges of the fp64 tests, by row % 5: N(0, 3^2), -inf in some non-target columns, uniform in
    [-10^4, 10^4] (most exponentials underflow), a confident row (target 20 above every other logit), a flat row."""
    n = t.shape[0]
    x = torch.randn(n, C, generator=gen, dtype=torch.float64) * 3
    kind = torch.arange(n) % 5
    valid = (t >= 0) & (t < C)
    tl = t.clamp(0, C - 1)
    rows = torch.arange(n)
    cols = torch.arange(C)[None]
    is_t = valid[:, None] & (cols == tl[:, None])
    neg = (kind == 1)[:, None] & (torch.rand(n, C, generator=gen) < 0.5) & ~is_t
    neg[:, 0] &= valid                            # an ignored row keeps column 0 finite
    x[neg] = -np.inf
    big = kind == 2
    x[big] = (torch.rand(int(big.sum()), C, generator=gen, dtype=torch.float64) * 2 - 1) * XMAX
    conf = (kind == 3) & valid
    x[rows[conf], tl[conf]] = x[conf].max(1).values + 20
    flat = kind == 4
    x[flat] = torch.randn(int(flat.sum()), 1, generator=gen, dtype=torch.float64) * 3
    return x.float()


def ce_n_class(n):
    """The row-CTA geometry of n (8 rows per CTA of the CE and L2-norm kernels): one partial CTA, whole CTAs, or a partial last CTA."""
    if n < 8:
        return "one partial CTA"
    return "whole CTAs" if n % 8 == 0 else "partial last CTA"


# ----------------------------------------------------------------------------------------------- L2 normalisation
L2_C = (1, 3, 31, 32, 33, 64, 96, 128, 256)
L2_N = (1, 7, 8, 9, 2 ** 20 + 3)
L2_BIG_C_MAX = 64                    # n = 2^20 + 3 at C <= 64 (n C <= 2^26)


def l2_n_list(C):
    return tuple(n for n in L2_N if n < 2 ** 20 or C <= L2_BIG_C_MAX)


def l2_exact_rows(n, C, gen):
    """(x, dy) fp32 [n, C] on the device: row i holds 4^a entries of +-2^j, a in range for C, j in [-4, 11 - a]; dy = k / 256, |k| <= 64."""
    amax = 0
    while 4 ** (amax + 1) <= C:
        amax += 1
    a = torch.randint(0, amax + 1, (n,), generator=gen, device="cuda")
    j = torch.randint(-4, 8, (n,), generator=gen, device="cuda").clamp(max=11 - a)
    r = torch.rand(n, C, generator=gen, device="cuda")
    rank = r.argsort(1).argsort(1)                # a random permutation of the columns per row
    nz = rank < (4 ** a)[:, None]
    sign = torch.where(torch.rand(n, C, generator=gen, device="cuda") < 0.5, -1.0, 1.0)
    x = torch.where(nz, sign * torch.pow(2.0, j.double())[:, None].float(), torch.zeros((), device="cuda"))
    dy = torch.randint(-64, 65, (n, C), generator=gen, device="cuda").float() / 256
    return x, dy


# ----------------------------------------------------------------------------------------------- SGD
SGD_N = (1, 2, 3, 4, 5, 7, 8, 2 ** 22 + 1, 2 ** 22 + 3)
SGD_EXACT = [dict(lr=2.0 ** -4, momentum=m, weight_decay=2.0 ** -10, dampening=dmp, grad_scale=gs)
             for m in (0.5, 0.75) for dmp in (0.0, 0.5) for gs in (1.0, 0.5)]
SGD_REAL = [dict(lr=0.1, momentum=0.9, weight_decay=1e-4, dampening=0.1, grad_scale=1.0),       # semseg finetuning
            dict(lr=0.1, momentum=0.8, weight_decay=1e-4, dampening=0.0, grad_scale=0.5)]      # pretraining, two ranks
STEPS = 3


def sgd_grid(n, bound, gen):
    """fp32 [n] multiples of 2^-10 in (-bound, bound) on the device."""
    k = int(bound * 1024) - 1
    return torch.randint(-k, k + 1, (n,), generator=gen, device="cuda").float() / 1024


def sgd_restate(p, g, b, first, lr, momentum, weight_decay, grad_scale, dampening):
    """The kernel's step on fp32 device tensors, one fp32 rounding per statement:
         d = g grad_scale + wd p;   b = first ? d : momentum b + keep d;   p = p - lr b,   keep = fp32(1 - dampening).
    With lr, wd, grad_scale and keep powers of two every product is exact, so d and p round once whether or not the compiler contracts
    a product into an add.  momentum b may be inexact (momentum = 0.75): the statement is restated both ways, rounded once (a fused
    multiply-add) and twice.  -> [(p, b)] on the first step, else [(p, b) unfused, (p, b) fused]; these differ only where momentum b
    is inexact."""
    f32 = lambda v: torch.tensor(v, dtype=torch.float32).item()
    lr, m, wd, gs = f32(lr), f32(momentum), f32(weight_decay), f32(grad_scale)
    keep = float(np.float32(1.0) - np.float32(dampening))
    for s in (lr, wd, gs, keep):
        assert s == 0 or float(np.log2(abs(s))).is_integer(), s
    d = g * gs + p * wd                                            # torch rounds each operation: exact products, one rounded sum
    if first:
        bs = [d]
    else:
        mb, kd = b.double() * m, d.double() * keep                 # exact in fp64
        s = mb + kd
        assert bool(((s - mb) - kd == 0).all() & ((s - kd) - mb == 0).all()), "fp64 sum inexact: the fused restatement needs it exact"
        bs = [b * m + d * keep, s.float()]
    return [(p - bb * lr, bb) for bb in bs]


# ----------------------------------------------------------------------------------------------- gather-sum
GS_C = (4, 8, 24, 28)
GS_K = (1, 8, 27)
GS_XPAD = 8                          # ldx = C + 8, the operand in columns [4, 4 + C)
GS_YPAD = 12                         # ldy = C + 12, the output in columns [4, 4 + C)


def gs_features(n, C, gen):
    """Integer-valued fp32 [n, C] in [-64, 64] on the device."""
    return torch.randint(-64, 65, (n, C), generator=gen, device="cuda").float()


def gs_restate(X, tbl, kmap, K, n_out):
    """(Y fp64 [n_out, C], cnt fp64 [n_out]) = (sum over k of X[tbl[kmap[k]][j]], number of present neighbours), on the device."""
    Z = torch.cat([X.double(), X.new_zeros(1, X.shape[1]).double()])
    Y = torch.zeros(n_out, X.shape[1], dtype=torch.float64, device=X.device)
    cnt = torch.zeros(n_out, dtype=torch.float64, device=X.device)
    for k in range(K):
        t = tbl[kmap[k] if kmap is not None else k, :n_out].long()
        Y += Z[torch.where(t >= 0, t, X.shape[0])]
        cnt += (t >= 0).double()
    return Y, cnt
