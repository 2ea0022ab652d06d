"""VoteNet's training criterion on the GPU, behind the interface of the original's `models/loss_helper.py`.

    get_loss(end_points, config)    vote, objectness, box and semantic-class losses and their gradients (csrc/det_loss.cu)
    install()                       registers this module as `models.loss_helper`

After `install()`, VoteNet's unmodified `lib/train.py` and `lib/test.py` compute their loss here: two launches forward, one backward,
every scalar of `end_points` a 0-dim view of one device buffer.  The semantics, quirks included, are stated in include/pcb200.h and
DESIGN.md section 5.
"""
import ctypes
import sys

import numpy as np
import torch

from .det_eval import register
from ._lib import PcbDetLossArgs, PcbError, PcbStrided, check, lib, ptr, require_cuda, stream, workspace

FAR_THRESHOLD = 0.6
NEAR_THRESHOLD = 0.3
GT_VOTE_FACTOR = 3                                      # number of GT votes per point
OBJECTNESS_CLS_WEIGHTS = [0.2, 0.8]

# the entries of the kernel's output vector, in order; the first eight are the terms the gradient is taken of
TERMS = ("vote_loss", "objectness_loss", "center_loss", "heading_cls_loss", "heading_reg_loss", "size_cls_loss", "size_reg_loss",
         "sem_cls_loss")
OUTPUTS = TERMS + ("box_loss", "loss", "pos_ratio", "neg_ratio", "obj_acc")
# differentiable inputs, in the order of pcb_det_loss_backward's gradients
GRAD_INPUTS = ("vote_xyz", "seed_xyz", "center", "objectness_scores", "heading_scores", "heading_residuals_normalized", "size_scores",
               "size_residuals_normalized", "sem_cls_scores")
_STRIDED = ("center", "objectness_scores", "heading_scores", "heading_residuals_normalized", "size_scores", "size_residuals_normalized",
            "sem_cls_scores")


def _strided(t):
    st = list(t.stride()) + [0] * (4 - t.dim())
    return PcbStrided(t.data_ptr(), *st)


class _Inputs:
    """The fp32 / int64 device tensors of one call and the `pcb_det_loss_args` that points at them (kept alive together)."""

    def __init__(self, end_points, config):
        f32 = lambda k: end_points[k].to(torch.float32)
        i64 = lambda k: end_points[k].to(torch.int64).contiguous()
        self.t = t = {k: f32(k) for k in GRAD_INPUTS}
        for k in ("vote_xyz", "seed_xyz"):
            t[k] = t[k].contiguous()
        t["aggregated_vote_xyz"] = f32("aggregated_vote_xyz").detach().contiguous()
        seed_inds = end_points["seed_inds"]
        t["seed_inds"] = (seed_inds if seed_inds.dtype == torch.int32 else seed_inds.to(torch.int64)).contiguous()
        for k in ("vote_label", "center_label", "heading_residual_label", "size_residual_label", "box_label_mask"):
            t[k] = f32(k).detach().contiguous()
        for k in ("vote_label_mask", "heading_class_label", "size_class_label", "sem_cls_label"):
            t[k] = i64(k)
        require_cuda(t["seed_xyz"])
        NH, NS, C = int(config.num_heading_bin), int(config.num_size_cluster), int(config.num_class)
        self.mean_size = np.ascontiguousarray(np.asarray(config.mean_size_arr).astype(np.float32))
        if self.mean_size.shape != (NS, 3):
            raise PcbError(f"det_loss: mean_size_arr has shape {self.mean_size.shape}, expected ({NS}, 3)")
        B, S = t["seed_xyz"].shape[:2]
        K, K2 = t["aggregated_vote_xyz"].shape[1], t["center_label"].shape[1]
        V = t["vote_xyz"].shape[1] // max(S, 1)
        want = {"seed_xyz": (B, S, 3), "seed_inds": (B, S), "vote_xyz": (B, S * V, 3), "aggregated_vote_xyz": (B, K, 3), "center": (B, K, 3),
                "objectness_scores": (B, K, 2), "heading_scores": (B, K, NH), "heading_residuals_normalized": (B, K, NH),
                "size_scores": (B, K, NS), "size_residuals_normalized": (B, K, NS, 3), "sem_cls_scores": (B, K, C),
                "heading_class_label": (B, K2), "heading_residual_label": (B, K2), "size_class_label": (B, K2),
                "size_residual_label": (B, K2, 3), "sem_cls_label": (B, K2), "box_label_mask": (B, K2)}
        for k, shape in want.items():
            if tuple(t[k].shape) != shape:
                raise PcbError(f"det_loss: {k} has shape {tuple(t[k].shape)}, expected {shape}")
        N = t["vote_label"].shape[1]
        if tuple(t["vote_label"].shape) != (B, N, 3 * GT_VOTE_FACTOR) or tuple(t["vote_label_mask"].shape) != (B, N):
            raise PcbError("det_loss: vote_label must be [B, N, 9] and vote_label_mask [B, N]")
        if t["center_label"].dim() != 3 or t["center_label"].shape[0] != B or t["center_label"].shape[2] < 3:
            raise PcbError("det_loss: center_label must be [B, K2, >= 3]")
        self.dims = (B, S, V, N, K, K2)
        scale = np.float32(1.0) / np.float32(np.pi / NH)     # torch's fp32 tensor / Python float on the GPU: times the fp32 reciprocal
        a = PcbDetLossArgs(B, S, V, N, K, K2, NH, NS, C, int(t["seed_inds"].dtype == torch.int64), float(scale),
                           self.mean_size.ctypes.data)
        for k in ("seed_xyz", "seed_inds", "vote_xyz", "vote_label", "vote_label_mask", "aggregated_vote_xyz", "center_label",
                  "heading_class_label", "heading_residual_label", "size_class_label", "size_residual_label", "sem_cls_label",
                  "box_label_mask"):
            setattr(a, k, ptr(t[k]))
        for k in _STRIDED:
            setattr(a, k, _strided(t[k]))
        a.center_label_ld = t["center_label"].shape[2]
        self.args = a


class _DetLoss(torch.autograd.Function):
    """(out fp32 [13], objectness_label, objectness_mask, object_assignment) of the differentiable inputs in GRAD_INPUTS order."""

    @staticmethod
    def forward(ctx, inp, *tensors):
        B, S, V, N, K, K2 = inp.dims
        dev = tensors[0].device
        out = torch.empty(len(OUTPUTS), dtype=torch.float32, device=dev)
        label = torch.empty(B, K, dtype=torch.int64, device=dev)
        mask = torch.empty(B, K, dtype=torch.float32, device=dev)
        assignment = torch.empty(B, K, dtype=torch.int64, device=dev)
        sb = lib.pcb_det_loss_state_bytes(B, S, K, K2)
        state = torch.empty(sb, dtype=torch.uint8, device=dev)
        wsb = lib.pcb_det_loss_ws_bytes(B, S, K, K2)
        ws = workspace(wsb, dev)
        check(lib.pcb_det_loss_forward(ctypes.byref(inp.args), ptr(out), ptr(label), ptr(mask), ptr(assignment), ptr(state), sb, ptr(ws),
                                       wsb, stream()))
        ctx.inp = inp
        ctx.save_for_backward(label, mask, assignment, state)
        ctx.mark_non_differentiable(label, mask, assignment)
        return out, label, mask, assignment

    @staticmethod
    def backward(ctx, grad_out, *_):
        label, mask, assignment, state = ctx.saved_tensors
        inp = ctx.inp
        grads = [torch.empty(inp.t[k].shape, dtype=torch.float32, device=state.device) if ctx.needs_input_grad[1 + i] else None
                 for i, k in enumerate(GRAD_INPUTS)]
        g = grad_out.to(torch.float32).contiguous()
        check(lib.pcb_det_loss_backward(ctypes.byref(inp.args), ptr(g), ptr(label), ptr(mask), ptr(assignment), ptr(state), state.numel(),
                                        *[ptr(x) for x in grads], stream()))
        return (None, *grads)


def get_loss(end_points, config):
    """`loss_helper.get_loss`: returns (loss, end_points) with the original's keys, dtypes and shapes.  The eight terms, box_loss, loss,
    pos_ratio, neg_ratio and obj_acc are 0-dim views of one fp32 buffer; backpropagating any of them reaches center, the proposal
    scores and residuals, vote_xyz and seed_xyz (never aggregated_vote_xyz or the labels)."""
    inp = _Inputs(end_points, config)
    out, label, mask, assignment = _DetLoss.apply(inp, *[inp.t[k] for k in GRAD_INPUTS])
    v = dict(zip(OUTPUTS, out.unbind(0)))
    end_points["vote_loss"] = v["vote_loss"]
    end_points["objectness_loss"] = v["objectness_loss"]
    end_points["objectness_label"] = label
    end_points["objectness_mask"] = mask
    end_points["object_assignment"] = assignment
    for k in ("pos_ratio", "neg_ratio") + TERMS[2:] + ("box_loss", "loss", "obj_acc"):
        end_points[k] = v[k]
    return v["loss"], end_points


def install(name="models.loss_helper"):
    """Register this module as `name` (and as the attribute of its parent package), so that `from models.loss_helper import get_loss`
    -- VoteNet's lib/train.py and lib/test.py -- resolves here.  Returns the module."""
    return register(sys.modules[__name__], name)
