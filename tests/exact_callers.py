"""What the PointNet++ modules, the VoteNet heads and the one-view Res16UNet callers (semantic-segmentation finetuning, the sparse-conv
detection backbone) hand the convolution and fused-unit kernels, restated once (tests/test_gpu_callers_exact.py runs every case bit for
bit and checks this restatement against recorded calls; the host checks are tests/test_host_callers_geometry.py).

The callers are built on the meta device from the library's own classes, so this module imports without a GPU.  Per caller, `Calls`
holds four sets:
  * units: exact_unit.Sig of every pcb_unit_backward struct, and of every eval-mode pcb_unit_forward struct; a training forward call
    reads exact_unit.forward_part of its unit's signature.  Kind "ident" is K = 1 on pointnet2_modules' identity table.
  * split: (K, Ck, N, role, fmt, strided, accumulate) of every direct pcb_conv_forward_split / pcb_conv_forward_split_ordered call
    (role "fwd" or "dgrad": Ck contraction channels, N output columns) and pcb_conv_wgrad_split call (role "wgrad": Ck = Ca, N = Cb).
  * exact_fwd: (K, Cin, Cout) of every pcb_conv_forward call;  exact_wgrad: (K, Ca, Cb, transpose_out, flags) of every pcb_conv_wgrad.
"""
import functools
from typing import NamedTuple

import numpy as np
import torch

from tests import exact_conv as XC
from tests import exact_unit as XU

# ----------------------------------------------------------------------------------------------- the callers' widths
# backbone_module.py (Pointnet2Backbone): SA1-SA4 as (npoint, radius, nsample, mlp); mlp[0] of SA1 is input_feature_dim (1: the
# height feature, 0: xyz only)
SA = {"sa1-height": (2048, 0.2, 64, (1, 64, 64, 128)), "sa1-xyz": (2048, 0.2, 64, (0, 64, 64, 128)),
      "sa2": (1024, 0.4, 32, (128, 128, 128, 256)), "sa3": (512, 0.8, 16, (256, 128, 128, 256)),
      "sa4": (256, 1.2, 16, (256, 128, 128, 256))}
# proposal_module.py: the vote aggregation, npoint = num_proposal, normalize_xyz
NUM_PROPOSAL = 256                        # train.py's --num_target (votenet.py's constructor default is 128)
AGG = (NUM_PROPOSAL, 0.3, 16, (256, 128, 128, 128))
# backbone_module.py: fp1, fp2
FP = (256 + 256, 256, 256)
# votenet.py: VotingModule(vote_factor, 256); vote_factor 1 is the default, 2 the other setting the heads support
SEED_DIM = 256
VOTE_FACTORS = (1, 2)
# proposal_module.py ProposalModule(num_class, num_heading_bin, num_size_cluster, ...) of the two datasets' model configs
DATASETS = {"scannet": (18, 1, 18), "sunrgbd": (10, 12, 10)}
# semantic-segmentation finetuning: Res16UNet34C(3, classes) (ScanNet 20, S3DIS 13); the detection backbone's output width
FINETUNE_CLASSES = (20, 13)
BACKBONE_OUT = 256

# ----------------------------------------------------------------------------------------------- row counts
SMS = 132                                 # H100 SXM
PROPOSAL_ROWS = 2 * NUM_PROPOSAL          # the proposal head at B = 2: offset-split mode, BatchNorm statistics fused into the reduction
VOTE_ROWS = 64 * 1024                     # the voting head at B = 64 (1024 seeds): direct mode
SA1_ROWS = 8 * 2048 * 64                  # SA1 at B = 8: B npoint nsample = 2^20 rows, run once, for its middle unit (64 -> 64)
UNIT_ROWS = {"split": PROPOSAL_ROWS, "direct": VOTE_ROWS}


class Calls(NamedTuple):
    units: frozenset
    split: frozenset
    exact_fwd: frozenset
    exact_wgrad: frozenset

    def __or__(self, o):
        return Calls(*(a | b for a, b in zip(self, o)))


_NONE = Calls(frozenset(), frozenset(), frozenset(), frozenset())


def _calls(units=(), split=(), exact_fwd=(), exact_wgrad=()):
    return Calls(frozenset(units), frozenset(split), frozenset(exact_fwd), frozenset(exact_wgrad))


def ident(Cin, Cout, out_p=False, gin_mode=1, out_str=False, g_str=False):
    """A training unit on the identity table as the PointNet++ modules and the heads issue it: ReLU, fp16 forward, one view."""
    return XU.Sig("ident", 1, Cin, Cout, True, False, out_p, 0, gin_mode, True, False, False, False, out_str, g_str, False, False)


def _unit_calls(sigs, train):
    """Training: the signatures in full (as the backward calls record them; the forward calls record exact_unit.forward_part of
    them); eval: the forward calls in eval mode."""
    if train:
        return set(sigs)
    return {XU.forward_part(s)._replace(eval=True) for s in sigs}


def _split_fwd(Ck, N):
    return (1, Ck, N, "fwd", "fp16", False, False)


def _split_bwd(Ck, N):
    """The weight gradient (accumulated) and the data gradient of a K = 1 convolution Ck -> N on the identity table."""
    return {(1, Ck, N, "wgrad", "bf16", False, True), (1, N, Ck, "dgrad", "bf16", False, False)}


# ----------------------------------------------------------------------------------------------- the callers, built on the meta device
@functools.lru_cache(None)
def sa_module(name):
    from pointcontrast_b200 import pointnet2_modules as P
    npoint, radius, nsample, mlp = AGG if name == "agg" else SA[name]
    with torch.device("meta"):
        return P.PointnetSAModuleVotes(npoint=npoint, radius=radius, nsample=nsample, mlp=list(mlp), use_xyz=True, normalize_xyz=True)


@functools.lru_cache(None)
def fp_module():
    from pointcontrast_b200 import pointnet2_modules as P
    with torch.device("meta"):
        return P.PointnetFPModule(mlp=list(FP))


@functools.lru_cache(None)
def voting_module(V):
    from pointcontrast_b200 import det_heads as D
    with torch.device("meta"):
        return D.VotingModule(V, SEED_DIM)


@functools.lru_cache(None)
def proposal_module(dataset):
    from pointcontrast_b200 import det_heads as D
    NC, NH, NS = DATASETS[dataset]
    with torch.device("meta"):
        return D.ProposalModule(NC, NH, NS, np.ones((NS, 3), dtype=np.float32), NUM_PROPOSAL, "vote_fps", seed_feat_dim=SEED_DIM)


@functools.lru_cache(None)
def res16unet(out):
    """Res16UNet34C(3, out): the finetune networks (classes) and the detection backbone's net (detection.SparseConvBackbone)."""
    from pointcontrast_b200 import detection
    from pointcontrast_b200.model import load_model
    from tests.refload import default_config
    with torch.device("meta"):
        if out == BACKBONE_OUT:
            return detection.SparseConvBackbone(3, BACKBONE_OUT).net
        return load_model("Res16UNet34C")(3, out, default_config(), D=3)


# ----------------------------------------------------------------------------------------------- what each caller issues
def sa_calls(name, train=True):
    """PointnetSAModuleVotes: layer 0 on the exact fp32 kernels (feature columns per point, the relative-xyz columns' weight and data
    gradients per row), the middle units, the last layer's split convolution and its gradients."""
    from pointcontrast_b200 import pointnet2_modules as P
    layers = P._layers(sa_module(name).mlp_module)
    C0, C = layers[0][0].out_channels, layers[0][0].in_channels - 3
    cin, CL = layers[-1][0].in_channels, layers[-1][0].out_channels
    units = [ident(conv.in_channels, conv.out_channels) for conv, _ in layers[1:-1]]
    fwd = {(1, C, C0)} if C else set()
    out = _calls(_unit_calls(units, train), {_split_fwd(cin, CL)}, fwd)
    if not train:
        return out
    return out | _calls(split=_split_bwd(cin, CL), exact_fwd={(1, C0, 3)} | ({(1, C0, C)} if C else set()),
                        exact_wgrad={(1, 3, C0, 1, 0)} | ({(1, C, C0, 1, 0)} if C else set()))


def fp_calls(train=True):
    """PointnetFPModule: every layer a unit; the last one writes the fp32 output plane."""
    from pointcontrast_b200 import pointnet2_modules as P
    layers = P._layers(fp_module().mlp)
    units = [ident(conv.in_channels, conv.out_channels, out_p=i == len(layers) - 1) for i, (conv, _) in enumerate(layers)]
    return _calls(_unit_calls(units, train))


def _head_calls(mod, gin_mode, train):
    """conv1 / conv2 as units whose input carries the 32 bias columns (Cin = C + 32) and whose output planes do too (out_lds = C + 32);
    their output gradients are the first C columns of a [rows, C + 32] buffer; conv3 into z padded to a multiple of 32 columns."""
    C = mod.conv1.in_channels
    u1 = ident(C + 32, mod.conv1.out_channels, gin_mode=gin_mode, out_str=True, g_str=True)
    u2 = ident(C + 32, mod.conv2.out_channels, out_str=True, g_str=True)
    cpad = -(-mod.conv3.out_channels // 32) * 32
    out = _calls(_unit_calls([u1, u2], train), {_split_fwd(mod.conv2.out_channels + 32, cpad)})
    return out | _calls(split=_split_bwd(mod.conv2.out_channels + 32, cpad)) if train else out


def voting_calls(V, train=True):
    """VotingModule: conv1's data gradient accumulates onto the residual gradient of the seed features (gin_mode 2)."""
    return _head_calls(voting_module(V), 2, train)


def proposal_calls(dataset, train=True):
    """ProposalModule: the vote aggregation (a set-abstraction module), then the head."""
    return sa_calls("agg", train) | _head_calls(proposal_module(dataset), 1, train)


def res16unet_calls(out, train=True):
    """Res16UNet34C(3, out) on one view through the fused executor (semseg.SegmentationTrainer, detection.SparseConvBackbone): every
    unit with n0 == n_out and fp16 forward, and the final 1x1 layer through `me` -- the exact fp32 kernels for a class count the
    tensor cores do not take, else the split kernel."""
    net = res16unet(out)
    sigs = [s._replace(fp16=True, two_views=False) for s in XU.net_units(net)]
    Cin = net.final.in_channels
    if out % 32:
        fin = _calls(exact_fwd={(1, Cin, out)}) | (_calls(exact_fwd={(1, out, Cin)}, exact_wgrad={(1, Cin, out, 0, 4)}) if train else _NONE)
    else:
        fin = _calls(split={_split_fwd(Cin, out)}) | (_calls(split=_split_bwd(Cin, out)) if train else _NONE)
    return _calls(_unit_calls(sigs, train)) | fin


CALLERS = tuple([f"sa:{k}" for k in SA] + ["fp"] + [f"vote:{V}" for V in VOTE_FACTORS] + [f"proposal:{d}" for d in DATASETS]
                + [f"res16unet:{c}" for c in FINETUNE_CLASSES + (BACKBONE_OUT,)])


def caller_calls(caller, train=True):
    kind, _, arg = caller.partition(":")
    if kind == "sa":
        return sa_calls(arg, train)
    if kind == "fp":
        return fp_calls(train)
    if kind == "vote":
        return voting_calls(int(arg), train)
    if kind == "proposal":
        return proposal_calls(arg, train)
    return res16unet_calls(int(arg), train)


@functools.lru_cache(None)
def all_calls():
    out = _NONE
    for c in CALLERS:
        out = out | caller_calls(c, True) | caller_calls(c, False)
    return out


# ----------------------------------------------------------------------------------------------- the case lists the GPU tests run
@functools.lru_cache(None)
def unit_signatures():
    """Every unit signature the callers issue that the Res16UNet case matrix (exact_unit.signatures) does not hold: training
    signatures in full (the forward test reads their forward fields) and eval signatures."""
    matrix = set(XU.signatures())
    return tuple(sorted(s for s in all_calls().units if s not in matrix))


def training_signatures():
    return tuple(s for s in unit_signatures() if not s.eval)


@functools.lru_cache(None)
def split_cases():
    return tuple(sorted(all_calls().split))


@functools.lru_cache(None)
def exact_forward_cases():
    return tuple(sorted(all_calls().exact_fwd))


@functools.lru_cache(None)
def exact_wgrad_cases():
    return tuple(sorted(all_calls().exact_wgrad))


def head_padding(Ck, N):
    """(C, X) of a head conv3 case Ck = C + 32 -> N = X rounded up to 32, else None: its input's bias column is C (hi = 1, lo = 0,
    the other 31 pad columns 0) and output columns [X, N) hold zero weights."""
    for mod in [voting_module(V) for V in VOTE_FACTORS] + [proposal_module(d) for d in DATASETS]:
        C, X = mod.conv2.out_channels, mod.conv3.out_channels
        if (Ck, N) == (C + 32, -(-X // 32) * 32):
            return C, X
    return None


def conv_mode(K, n, Ck, N, sms=SMS):
    return "direct" if XC.conv_splits(K, n, Ck, N, sms) == 1 else "split"


SPLIT_ROWS = (1, 129, PROPOSAL_ROWS, VOTE_ROWS)       # split cases: a partial first tile, then the two heads' row counts
EXACT_ROWS = (1, 129, 4097)
BIG_EXACT_WGRAD = (1, 3, 64, 1, 0)        # SA1's relative-xyz weight gradient, also run over SA1_ROWS
BIG_UNIT = ident(64, 64)                  # SA1's middle unit, run over SA1_ROWS

