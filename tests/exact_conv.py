"""Shapes, tile rules and exactly representable operands of the bit-exact convolution tests (tests/test_gpu_conv_exact.py; the
host checks of this module are tests/test_host_conv_geometry.py).

Exactness: every product a kernel forms is a multiple of one quantum q, and for every output element the sum of the absolute values
of all its terms (plus |bias| and |accumulate base|) is below 2^20 q.  Then every partial sum is an fp32 number whatever the order of
summation -- the tensor cores' align-and-truncate accumulation, offset splits and row splits included -- and the kernel's output must
equal an fp64 reference bit for bit.  The bounds below hold for ANY neighbour table: they only use how many nonzeros a row (forward)
or a column (weight gradient) of the operands may hold, which the generators enforce.
"""
import functools

import torch

LIMIT = 2 ** 20

# ----------------------------------------------------------------------------------------------- the library's tile rules, restated
BM, BK, WM = 128, 32, 128          # conv_wgmma.cu: output rows per CTA, channels per pipeline step; weight-gradient M block


def pick_tile(C):
    """conv.cu pick_tile: the column tile of a convolution with C output columns."""
    return next((b for b in (128, 96, 64, 32) if C % b == 0), 0)


def col_blocks(N):
    return N // pick_tile(N)


def conv_splits(K, n_out, Cin, Cout, sms):
    """conv.cu conv_splits: offset splits of pcb_conv_forward_split (1 = direct mode)."""
    base = -(-n_out // BM) * col_blocks(Cout)
    if base >= sms:
        return 1
    s = min(-(-int(0.5 * sms) // base), K * (Cin // BK), 64)
    return 1 if s < 2 else s


def m_blocks(Ca):
    """wgrad_wgmma_kernel: (number of 128-row M blocks, rows of the last one)."""
    n = -(-Ca // WM)
    return n, Ca - WM * (n - 1)


def wgrad_splits(K, n, Ca, Cb, sms):
    """conv.cu wgrad_split_splits: row splits of pcb_conv_wgrad_split."""
    base = -(-K // 2) * m_blocks(Ca)[0] * col_blocks(Cb)
    return min(max(min((2 * sms) // base, -(-n // 64)), 1), 96)


def wgrad_rows_per_split(n, splits):
    return -(-(-(-n // splits)) // 16) * 16


def wgrad_empty_splits(n, splits):
    return splits - -(-n // wgrad_rows_per_split(n, splits))


def ws_align(nbytes):
    return (nbytes + 255) // 256 * 256


# ----------------------------------------------------------------------------------------------- shapes
MODELS = ("Res16UNet14", "Res16UNet18", "Res16UNet34", "Res16UNet34C")


@functools.lru_cache(None)
def model_convs(name):
    """(kind, K, Cin, Cout) of every convolution of the model, kind in k27 / down / up / k1 (built on the meta device: no data)."""
    from pointcontrast_b200 import me
    from pointcontrast_b200.model import load_model
    from tests.refload import default_config
    with torch.device("meta"):
        net = load_model(name)(3, 32, default_config(), D=3)
    return tuple(("up" if m.is_transpose else {27: "k27", 8: "down", 1: "k1"}[m.kernel.shape[0]],) + tuple(m.kernel.shape)
                 for m in net.modules() if isinstance(m, me._ConvolutionBase))


def _tc(c):
    return c[2] % 32 == 0 and c[3] % 32 == 0


# widths the models do not reach: a 32-wide column tile with several blocks (160, 224, 416), weight-gradient M blocks whose last block
# follows full ones with 32 (160, 416) or 96 (224) rows, a 768-channel contraction (24 channel chunks), and output widths whose
# column tile has several blocks in the forward role (320: 64 x 5, 192: 96 x 2), which alone runs fp16 operands
EXTRA_CONVS = (("k27", 27, 768, 160), ("k1", 1, 416, 224), ("down", 8, 224, 416), ("up", 8, 160, 224), ("k27", 27, 192, 320),
               ("up", 8, 288, 192))


@functools.lru_cache(None)
def conv_shapes():
    return tuple(sorted({c for name in MODELS for c in model_convs(name) if _tc(c)} | set(EXTRA_CONVS)))


@functools.lru_cache(None)
def forward_cases():
    """(kind, K, Cin, Cout, role, fmt): every tensor-core convolution in the forward role (bf16 and fp16 operands) and the
    data-gradient role (bf16: the data-gradient tiles are always bf16)."""
    out = []
    for kind, K, Cin, Cout in conv_shapes():
        out += [(kind, K, Cin, Cout, "fwd", "bf16"), (kind, K, Cin, Cout, "fwd", "fp16"), (kind, K, Cin, Cout, "dgrad", "bf16")]
    return tuple(out)


def contraction(case):
    """(contraction channels, output columns) of a forward case."""
    _, _, Cin, Cout, role, _ = case
    return (Cin, Cout) if role == "fwd" else (Cout, Cin)


@functools.lru_cache(None)
def wgrad_cases():
    """(K, Ca, Cb, transpose_out): the weight gradient of every tensor-core convolution as the fused executor issues it (transposed
    convolutions gather the output gradient and write the transposed kernel)."""
    return tuple(sorted({(K, Cout, Cin, 1) if kind == "up" else (K, Cin, Cout, 0) for kind, K, Cin, Cout in conv_shapes()}))


SPLIT_ROWS = (1, 127, 128, 129)             # forward: the offset-split mode (one or two row tiles)
WGRAD_ROWS = (1, 15, 16, 17, 257)           # weight gradient: partial and whole 16-row steps
BIG_WGRAD = (1, 128, 128, 0, 6200)          # K, Ca, Cb, transpose_out, n: more row splits than rows to fill them


def direct_rows(N, sms):
    """A row count that runs pcb_conv_forward_split in direct mode (at least one CTA per SM), not a multiple of 128."""
    return BM * -(-sms // col_blocks(N)) - 37


def forward_variants(ci):
    """(rows or "direct", strided, bias, accumulate) run for forward case number ci: bias and accumulation in both modes."""
    return ((1, False, False, False), (127, True, True, False), (128, True, False, True), (129, True, True, True),
            ("direct", True, ci % 2 == 0, ci % 2 == 1))


# ----------------------------------------------------------------------------------------------- operand formats
class Fmt:
    """Operand values of a split-operand format.  Activation planes: hi in +-HI, lo in +-LO.  Weights: W = (a + b WB) SCALE with
    a in +-WA, b in {0, +-1}, whose hi/lo split (bf16, or fp16 of W 2^10) is exactly hi = a, lo = b WB in kernel units; the kernel
    scales its accumulators by SCALE.  Q: the quantum of every product, in output units."""

    def __init__(self, name, dtype, HI, LO, WA, WB, SCALE, flags):
        self.name, self.dtype, self.HI, self.LO, self.WA, self.WB, self.SCALE, self.flags = name, dtype, HI, LO, WA, WB, SCALE, flags
        self.Q = min(LO * min(WA), min(HI) * WB) * SCALE

    def per_entry(self):
        """Largest sum of |terms| one hi entry and one lo entry of a gathered row add to an output (kernel units)."""
        return max(self.HI) * (max(self.WA) + self.WB) + self.LO * max(self.WA)


# bf16: hi.lo products 2^-9, lo.hi 2^-8.  fp16: the weights are tiled as fp16(W 2^10), whose residual sits 2^12 below the hi part
BF16 = Fmt("bf16", torch.bfloat16, (1.0, 2.0), 2.0 ** -8, (1.0, 2.0), 2.0 ** -9, 1.0, 0)
FP16 = Fmt("fp16", torch.float16, (1.0,), 2.0 ** -8, (1.0, 2.0), 2.0 ** -12, 2.0 ** -10, 8 | 16)
FMTS = {"bf16": BF16, "fp16": FP16}
BIAS = (0.0, 0.5, -0.5, 1.25, -1.25)        # x SCALE; also the accumulate bases


def row_cap(fmt, K, C):
    """Nonzero hi (and lo) entries per activation row such that K gathered rows stay below 2^20 Q with |bias| + |base| added."""
    room = LIMIT * fmt.Q - 2 * max(BIAS) * fmt.SCALE
    return max(1, min(C, int(room / (K * fmt.per_entry() * fmt.SCALE))))


def forward_bound(fmt, K, m):
    """Table-free bound on the sum of |terms| of one output (output units) for rows holding at most m hi and m lo nonzeros."""
    return K * m * fmt.per_entry() * fmt.SCALE + 2 * max(BIAS) * fmt.SCALE


def _signs(shape, gen, device):
    return torch.randint(0, 2, shape, generator=gen, device=device).float() * 2 - 1


def _pick(vals, shape, gen, device):
    v = torch.tensor(vals, device=device)
    return v[torch.randint(0, len(vals), shape, generator=gen, device=device)] * _signs(shape, gen, device)


def capped_planes(n, C, m, hi_vals, lo, gen, device="cpu"):
    """fp32 hi/lo planes [n, C] with at most m nonzero hi and m nonzero lo entries per row."""
    hi = torch.zeros(n, C, device=device)
    lo_ = torch.zeros(n, C, device=device)
    if n and m:
        hi.scatter_(1, torch.randint(0, C, (n, m), generator=gen, device=device), _pick(hi_vals, (n, m), gen, device))
        lo_.scatter_(1, torch.randint(0, C, (n, m), generator=gen, device=device), lo * _signs((n, m), gen, device))
    return hi, lo_


def dense_planes(n, C, density, hi_vals, lo, gen, device="cpu"):
    """fp32 hi/lo planes [n, C], each entry nonzero with probability `density`."""
    keep = lambda: (torch.rand(n, C, generator=gen, device=device) < density).float()
    return _pick(hi_vals, (n, C), gen, device) * keep(), lo * _signs((n, C), gen, device) * keep()


def weights(K, Cin, Cout, fmt, gen, device="cpu", density=0.85):
    """(W fp32 [K][Cin][Cout], intended hi, intended lo) in kernel units (W = (hi + lo) SCALE)."""
    shape = (K, Cin, Cout)
    keep = (torch.rand(shape, generator=gen, device=device) < density).float()
    a = _pick(fmt.WA, shape, gen, device) * keep
    b = torch.randint(-1, 2, shape, generator=gen, device=device).float() * fmt.WB * keep
    return (a + b) * fmt.SCALE, a, b


def split_weights(W, fmt):
    """The weight tiles' hi/lo split in kernel units: bf16 round-to-nearest-even and the rounded residual, of W (bf16) or of W 2^10
    clamped to +-65000 (fp16) -- the restatement of tests/test_gpu_ops.py::_host_tile_image."""
    v = (W * 1024.0).clamp(-65000.0, 65000.0) if fmt is FP16 else W
    hi = v.to(fmt.dtype).float()
    return hi, (v - hi).to(fmt.dtype).float()


def bias_values(n, fmt, gen, device="cpu"):
    v = torch.tensor(BIAS, device=device)
    return v[torch.randint(0, len(BIAS), (n,), generator=gen, device=device)] * fmt.SCALE


# weight gradient (bf16 planes only): A dense, B with at most WG_COL_CAP nonzero hi (and lo) entries per column
WG_Q = 2.0 ** -8                          # lo.hi products: 2^-8 x {1, 2}
WG_A_DENSITY = 0.5


def wgrad_col_cap():
    per = max(BF16.HI) * (max(BF16.HI) + BF16.LO) + BF16.LO * max(BF16.HI)
    return int((LIMIT * WG_Q - max(BIAS)) / per)


def wgrad_bound(m):
    """Table-free bound on the sum of |terms| of one weight-gradient entry when B's columns hold at most m hi and m lo nonzeros."""
    return m * (max(BF16.HI) * (max(BF16.HI) + BF16.LO) + BF16.LO * max(BF16.HI)) + max(BIAS)


# exact fp32 kernels: full fp32 operands hi + lo (multiples of 2^-8) against integer weights / integer second operands
EXACT_Q = 2.0 ** -8
EXACT_FORWARD = (("k27", 27, 3, 32), ("down", 8, 3, 32), ("k1", 1, 3, 32), ("k27", 27, 3, 64), ("k1", 1, 96, 13), ("k1", 1, 256, 20),
                 ("synth", 27, 3, 32), ("synth", 8, 3, 64))
# (K, Ca, Cb, transpose_out, flags): the stem kernel, the generic kernel forced / transposed, final-layer widths; flag 4 = accumulate
EXACT_WGRAD = ((27, 3, 32, 0, 0), (27, 3, 32, 0, 1), (27, 3, 32, 1, 0), (27, 3, 32, 0, 4), (8, 3, 32, 0, 0), (27, 3, 64, 0, 4),
               (1, 96, 13, 0, 0), (1, 256, 20, 1, 4))


def exact_forward_bound(K, Cin):
    return K * Cin * (max(BF16.HI) + BF16.LO) * max(BF16.WA) + max(BIAS)


def exact_wgrad_bound(m):
    """The same for the exact weight gradient: A = hi + lo rows, B integers with at most m nonzeros per column."""
    return m * (max(BF16.HI) + BF16.LO) * max(BF16.HI) + max(BIAS)


def exact_wgrad_col_cap():
    return int((LIMIT * EXACT_Q - max(BIAS)) / ((max(BF16.HI) + BF16.LO) * max(BF16.HI)))
