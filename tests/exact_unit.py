"""Case matrix and exactly representable operands of the fused-unit tests (tests/test_gpu_unit_exact.py; the host checks of this module
are tests/test_host_unit_geometry.py).

A unit signature (`Sig`) is what `pcb_unit_forward` / `pcb_unit_backward` decide from their struct: the kind (k27, down, up, k1 or the
3-channel stem) with (K, Cin, Cout), ReLU, residual, fp32 output, the residual- and data-gradient modes, fp16 forward, eval mode, one
view or two, and which operands are column slices of wider (concatenation) buffers.  `model_units` restates how `fused.Runner` wires
every unit of a model and which modes its reverse sweep gives them; `signatures` holds each of them with fp16 forward on and off, two
views (the stacked pair) and, forward only, eval mode.

Forward operands: exact_conv's rule.  x planes hold at most `row_cap` nonzeros per row in the forward format (fp16 under fp16 forward,
else bf16) against weights of that format; the stem reads fp32 rows hi + lo against integer weights.  z is then exact.

Backward operands (`pcb_unit_backward` reads z, mean, invstd and the ReLU hi plane as inputs, so the test chooses them):
  * mean on the 2^-3 grid, invstd a power of two in INVSTD and gamma = c / invstd with c in SCALES (a signed power of two), so
    gamma * invstd == c exactly; z = mean + d 2^-3 with |d| <= D_MAX, so xhat is a multiple of 2^-3 invstd.
  * Paired rows: rows 2i and 2i + 1 of each view share z and the ReLU codes, and g[2i + 1] = -g[2i]; an odd last row of a view has
    g = 0.  g = v / c, v in DZ_VALUES (STEM_DZ for the stem), so every term of a view's sum of g and of g xhat is a multiple of
    q = 2^-8 / |c| times the xhat quantum and at most 1026 q; a column holds at most BN_COL_CAP nonzero g, so each sum is exact in
    any order and is exactly 0.  The kernel's dz = c (g - 0 - xhat 0) is then exactly c g (masked): v itself.
  * DZ_VALUES are h + l with h in +-{1, 2} and l = +-2^-8, whose bf16 split is exactly (h, l): exact_conv's bf16 activation
    format with BOTH planes nonzero, so a unit that drops or duplicates dz_lo is off by 2^-8 somewhere.  STEM_DZ are integers: the
    fp32 weight gradient of the stem follows exact_conv's fp32 rule (EXACT_Q).
  * Weight gradient (exact_conv's rule): the contiguous operand -- dz when wg_gather_x, else x -- holds at most `wgrad_col_cap()`
    (stem: `exact_wgrad_col_cap()`) nonzeros per column; the gathered one is dense; dW's accumulate base comes from BIAS.
  * Data gradient (exact_conv's forward rule): dz rows hold at most `row_cap(BF16, K, Cout)` nonzeros, the weights are bf16-format,
    gin's accumulate base comes from BIAS.
  * gres = masked g (+ a base on the 2^-2 grid) and dgamma / dbeta = base + 0 are exact.
Pairing zeroes the BatchNorm sums, so each signature also runs one unpaired call on exact_bn's backward operands, in which dgamma,
dbeta and gres are exact by exact_bn's rule.
"""
import functools
from typing import NamedTuple

import torch

from tests import exact_bn as XB
from tests import exact_conv as XC

MODELS = XC.MODELS
INVSTD = (0.5, 1.0)
SCALES = (0.5, 1.0, -0.5, -1.0)           # c = gamma * invstd
D_MAX = 2
Q = 2.0 ** -3
DZ_VALUES = ((1.0, 2.0 ** -8), (2.0, 2.0 ** -8), (2.0, -2.0 ** -8))      # (h, l): v = +-(h + l)
STEM_DZ = ((1.0, 0.0), (2.0, 0.0))
BN_LIMIT = 2 ** 24
BN_TERM = 1026                              # the largest |g xhat| in units of q: (2 + 2^-8) 2^8 D_MAX
BN_COL_CAP = (BN_LIMIT - 2 ** 14) // BN_TERM          # 2^14 q: room for the dgamma / dbeta accumulate base


class Sig(NamedTuple):
    kind: str
    K: int
    Cin: int
    Cout: int
    relu: bool
    res: bool
    out_p: bool
    gres_mode: int
    gin_mode: int
    fp16: bool
    eval: bool
    two_views: bool
    x_str: bool          # x_lds (x_ld for the stem) != Cin
    out_str: bool        # out_lds != Cout
    g_str: bool          # g_ld != Cout
    gin_str: bool        # gin_ld != Cin
    gres_str: bool       # gres_ld != Cout

    @property
    def tc(self):
        return self.Cin % 32 == 0 and self.Cout % 32 == 0

    def name(self):
        f = [f"{self.kind}-{self.Cin}x{self.Cout}"]
        f += ["relu"] * self.relu + ["res"] * self.res + ["outp"] * self.out_p
        f += [f"gres{self.gres_mode}"] * (self.gres_mode > 0) + [f"gin{self.gin_mode}"] * (self.gin_mode > 0)
        f += ["fp16" if self.fp16 else "bf16"] + ["eval"] * self.eval + ["2v" if self.two_views else "1v"]
        f += [s for s, on in (("xs", self.x_str), ("os", self.out_str), ("gs", self.g_str), ("is", self.gin_str), ("rs", self.gres_str)) if on]
        return "-".join(f)


def forward_part(s):
    """The fields a forward call reads (eval units never see a backward pass)."""
    return s._replace(gres_mode=0, gin_mode=0, g_str=False, gin_str=False, gres_str=False)


# ----------------------------------------------------------------------------------------------- the executor's wiring, restated
class _B:
    """A buffer of fused.Runner: width, row stride, fp32 plane, and the gradient slot it shares with its parent (None: no gradient)."""

    def __init__(self, C, ld=None, p=True, slot=None, grad=True):
        self.C, self.ld, self.p = C, ld if ld is not None else C, p
        self.slot = slot if slot is not None else [False if grad else None]

    def cols(self, c0, C):
        return _B(C, self.ld, self.p, self.slot)


@functools.lru_cache(None)
def model_units(name):
    """Static signatures (fp16 off, training, two views) of every unit of the model as fused.Runner.forward issues them and its
    backward sweep gives them gradient modes, in forward order.  Built on the meta device: no data."""
    from pointcontrast_b200.model import load_model
    from tests.refload import default_config
    with torch.device("meta"):
        m = load_model(name)(3, 32, default_config(), D=3)
    return net_units(m)


def net_units(m):
    """`model_units` of a built network (any output width: a final layer the tensor cores do not take asks for the fp32 plane of
    its input)."""
    units = []

    def kind(conv):
        K, Cin, Cout = conv.kernel.shape
        if Cin % 32 or Cout % 32:
            return "stem"
        return "up" if conv.is_transpose else {27: "k27", 8: "down", 1: "k1"}[K]

    def unit(conv, a_in, relu, residual=None, out=None, need_f32=False):
        K, Cin, Cout = conv.kernel.shape
        if out is None:
            out = _B(Cout, p=need_f32)
        units.append((kind(conv), int(K), int(Cin), int(Cout), relu, a_in, out, residual))
        return out

    def block(blk, x, out=None, need_f32=False):
        h = unit(blk.conv1, x, True)
        res = x if blk.downsample is None else unit(blk.downsample[0], x, False, need_f32=True)
        return unit(blk.conv2, h, True, residual=res, out=out, need_f32=need_f32)

    def stage(seq, x, out=None, need_f32=False):
        blocks = list(seq)
        for i, blk in enumerate(blocks):
            last = i == len(blocks) - 1
            x = block(blk, x, out if last else None, need_f32 if last else blocks[i + 1].downsample is None)
        return x

    P, I = m.PLANES, m.INIT_DIM
    a0 = _B(m.conv0p1s1.in_channels, grad=False)
    cat8, cat7 = _B(P[7] + I, p=False), _B(P[6] + P[0], p=False)
    cat6, cat5 = _B(P[5] + P[1], p=False), _B(P[4] + P[2], p=False)
    out_p1 = unit(m.conv0p1s1, a0, True, out=cat8.cols(P[7], I))
    x = unit(m.conv1p1s2, out_p1, True, need_f32=m.block1[0].downsample is None)
    b1 = stage(m.block1, x, out=cat7.cols(P[6], P[0]))
    x = unit(m.conv2p2s2, b1, True, need_f32=m.block2[0].downsample is None)
    b2 = stage(m.block2, x, out=cat6.cols(P[5], P[1]))
    x = unit(m.conv3p4s2, b2, True, need_f32=m.block3[0].downsample is None)
    b3 = stage(m.block3, x, out=cat5.cols(P[4], P[2]))
    x = unit(m.conv4p8s2, b3, True, need_f32=m.block4[0].downsample is None)
    x = stage(m.block4, x)
    unit(m.convtr4p16s2, x, True, out=cat5.cols(0, P[4]))
    x = stage(m.block5, cat5)
    unit(m.convtr5p8s2, x, True, out=cat6.cols(0, P[5]))
    x = stage(m.block6, cat6)
    unit(m.convtr6p4s2, x, True, out=cat7.cols(0, P[6]))
    x = stage(m.block7, cat7)
    unit(m.convtr7p2s2, x, True, out=cat8.cols(0, P[7]))
    x = stage(m.block8, cat8, need_f32=not (m.final.in_channels % 32 == 0 and m.final.out_channels % 32 == 0))
    x.slot[0] = True                                     # the final layer's data gradient
    sigs = []
    for kd, K, Cin, Cout, relu, a_in, out, res in reversed(units):
        gres = gin = 0
        if res is not None and res.slot[0] is not None:
            gres = 2 if res.slot[0] else 1
            res.slot[0] = True
        if a_in.slot[0] is not None:
            gin = 2 if a_in.slot[0] else 1
            a_in.slot[0] = True
        sigs.append(Sig(kd, K, Cin, Cout, relu, res is not None, out.p, gres, gin, False, False, True, a_in.ld != Cin, out.ld != Cout,
                        out.ld != Cout, gin > 0 and a_in.ld != Cin, gres > 0 and res.ld != Cout))
    return tuple(reversed(sigs))


@functools.lru_cache(None)
def signatures():
    """The case matrix: every static signature of the models with fp16 forward off and on (two views), and its forward part in eval
    mode (one view, fp16 forward: the executor's default)."""
    static = {s for name in MODELS for s in model_units(name)}
    out = set()
    for s in static:
        out |= {s._replace(fp16=f) for f in (False, True)}
        out.add(forward_part(s)._replace(fp16=True, eval=True, two_views=False))
    return tuple(sorted(out))


def training_cases():
    return tuple(s for s in signatures() if not s.eval)


def eval_cases():
    return tuple(s for s in signatures() if s.eval)


def view_split(n):
    """n0 for two views of n rows: about half, never a multiple of the BatchNorm chunk (the boundary cuts inside a chunk), >= 1."""
    R = XB.chunk_rows(n)
    n0 = max(1, n // 2)
    while n0 % R == 0 and n0 < n - 1:
        n0 += 1
    return n0


# ----------------------------------------------------------------------------------------------- backward operands
def _signs(shape, gen, device):
    return torch.randint(0, 2, shape, generator=gen, device=device).float() * 2 - 1


def pair_partner(n, n0):
    """Per row: the first row of its pair (rows 2i, 2i + 1 of each view), and whether it is the second row of a pair or a view's odd
    last row (alone)."""
    first = torch.arange(n)
    second = torch.zeros(n, dtype=torch.bool)
    alone = torch.zeros(n, dtype=torch.bool)
    for a, e in XB.segments(n, n0):
        j = torch.arange(e - a)
        first[a:e] = a + j - j % 2
        second[a:e] = j % 2 == 1
        if (e - a) % 2:
            alone[e - 1] = True
    return first, second, alone


def paired_backward(n, n0, C, row_cap, col_cap, stem, mask_fmt, seed, device="cpu"):
    """Operands of one exact backward call.  -> dict: z, mean [2, C], invstd [2, C], gamma [C], g, h / l (the bf16 split of v = c g:
    what dz must hold where the mask passes), codes and bcodes (the paired int16 hi-plane codes: out_hi and, under fp16 forward, a
    different out_bhi), gres, dgamma and dbeta bases."""
    gen = torch.Generator(device=device).manual_seed(seed)
    view = (torch.arange(n, device=device) >= n0).long()
    first, second, alone = (t.to(device) for t in pair_partner(n, n0))
    mean = torch.randint(-64, 65, (2, C), generator=gen, device=device).float() * Q
    invstd = torch.tensor(INVSTD, device=device)[torch.randint(0, len(INVSTD), (2, C), generator=gen, device=device)]
    c = torch.tensor(SCALES, device=device)[torch.randint(0, len(SCALES), (C,), generator=gen, device=device)]
    gamma = c / invstd[0]
    invstd[1] = invstd[0]                   # gamma * invstd must be c in both views
    d = torch.randint(-D_MAX, D_MAX + 1, (n, C), generator=gen, device=device).float()
    z = (mean[view] + d[first] * Q)
    # nonzero pattern per pair: at most row_cap columns per row, then at most col_cap nonzeros per column over all rows
    m = min(row_cap, C)
    nz = torch.zeros(n, C, dtype=torch.bool, device=device)
    nz.scatter_(1, torch.randint(0, C, (n, m), generator=gen, device=device), True)
    nz &= torch.rand(n, 1, generator=gen, device=device) < 0.8
    nz = nz[first] & ~alone[:, None]
    nz &= torch.cumsum(nz.long(), 0) <= col_cap - 1
    nz = nz[first] & ~alone[:, None]          # the cut may fall between the two rows of a pair: keep pairs whole
    vals = STEM_DZ if stem else DZ_VALUES
    pick = torch.randint(0, len(vals), (n, C), generator=gen, device=device)[first]
    sign = _signs((n, C), gen, device)[first] * torch.where(second, -1.0, 1.0)[:, None]
    h = torch.tensor([v[0] for v in vals], device=device)[pick] * sign * nz
    l = torch.tensor([v[1] for v in vals], device=device)[pick] * sign * nz
    g = (h + l) / c
    codes = XB.mask_codes(n, C, mask_fmt, seed + 1).to(device)[first]
    bcodes = XB.mask_codes(n, C, "bf16", seed + 2).to(device)[first]
    gbase = torch.randint(-16, 17, (n, C), generator=gen, device=device).float() * 0.25
    base = lambda: torch.randint(-16, 17, (C,), generator=gen, device=device).float() * 0.25
    return dict(z=z, mean=mean, invstd=invstd, gamma=gamma, g=g, h=h, l=l, codes=codes, bcodes=bcodes, gres_base=gbase,
                dgamma_base=base(), dbeta_base=base())


def bn_sum_terms(p, n0):
    """Largest over columns of (sum |g xhat| / q) over all rows, where q = 2^-8 / |c| 2^-3 invstd; < BN_LIMIT means exact sums."""
    n = p["z"].shape[0]
    view = (torch.arange(n, device=p["z"].device) >= n0).long()
    xhat = (p["z"].double() - p["mean"].double()[view]) * p["invstd"].double()[view]
    c = (p["gamma"] * p["invstd"][0]).double()
    q = 2.0 ** -8 / c.abs() * Q * p["invstd"][0].double()
    return float(((p["g"].double() * xhat).abs().sum(0) / q).max())


def col_nonzeros(t):
    return int((t != 0).sum(0).max()) if t.numel() else 0


def row_nonzeros(t):
    return int((t != 0).sum(1).max()) if t.numel() else 0


def backward_caps(sig, K):
    """(row cap, column cap) of the nonzero g entries for a signature."""
    if not sig.tc:
        col = XC.exact_wgrad_col_cap()
    elif sig.kind != "up":
        col = XC.wgrad_col_cap()
    else:
        col = BN_COL_CAP
    return XC.row_cap(XC.BF16, K, sig.Cout), min(col, BN_COL_CAP)


def unpaired_backward(n0, n1, C, seed):
    """exact_bn's backward operands (x is z): dgamma, dbeta and gres are exact, dz is not."""
    return XB.backward_operands(n0, n1, C, seed)
