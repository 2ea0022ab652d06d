"""PointInfoNCE and hardest-contrastive losses on libpcb200 kernels.

Restates `pretrain/pointcontrast/lib/ddp_trainer.py:400-426` (+ `lib/criterion.py:15-19`) and `:186-238`.
The reference draws its random subsets from process-global RNGs; here the draws are explicit arguments
(`select_positives` / the `sel*` tensors) so that the oracle and this module can be fed the same indices.
Nothing in this file synchronises the host with the device.
"""
import torch

from . import _lib
from ._lib import check, lib, ptr, stream, workspace


class _PointNCEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, inv_T):
        _lib.require_cuda(q)
        q, k = q.contiguous(), k.contiguous()
        n, D = q.shape
        loss = torch.empty((), dtype=torch.float32, device=q.device)
        dq, dk = torch.empty_like(q), torch.empty_like(k)
        with torch.cuda.device(q.device):
            wsb = lib.pcb_nce_ws_bytes(n)
            ws = workspace(wsb, q.device)
            check(lib.pcb_nce_forward_backward(ptr(q), ptr(k), n, D, inv_T, ptr(loss), ptr(dq), ptr(dk), ptr(ws), wsb, stream()))
        ctx.save_for_backward(dq, dk)
        return loss

    @staticmethod
    def backward(ctx, g):
        dq, dk = ctx.saved_tensors
        return dq * g, dk * g, None


class _L2NormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _lib.require_cuda(x)
        x = x.contiguous()
        n, C = x.shape
        y = torch.empty_like(x)
        inv = torch.empty(n, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.pcb_l2norm_forward(ptr(x), n, C, ptr(y), ptr(inv), stream()))
        ctx.save_for_backward(y, inv)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, inv = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        with torch.cuda.device(dy.device):
            check(lib.pcb_l2norm_backward(ptr(dy), ptr(y), ptr(inv), y.shape[0], y.shape[1], ptr(dx), stream()))
        return dx


def l2_normalize(F):
    """F / ||F||_2 per row, no epsilon (`model/res16unet.py:262-266`) -- one kernel forward, one backward."""
    return _L2NormFunction.apply(F)


class _CrossEntropyFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index):
        _lib.require_cuda(logits)
        logits = logits.contiguous().float()
        target = target.contiguous().long()
        n, C = logits.shape
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        dlogits = torch.empty_like(logits)
        with torch.cuda.device(logits.device):
            wsb = lib.pcb_ce_ws_bytes(n)
            ws = workspace(wsb, logits.device)
            check(lib.pcb_ce_forward_backward(ptr(logits), ptr(target), n, C, int(ignore_index), 1.0, ptr(loss), ptr(dlogits), ptr(ws), wsb,
                                              stream()))
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None


def cross_entropy(logits, target, ignore_index=255):
    """`nn.CrossEntropyLoss(ignore_index=config.data.ignore_label)(soutput.F, target)` (`downstream/semseg/lib/train.py:68,120`)."""
    return _CrossEntropyFunction.apply(logits, target, ignore_index)


def select_positives(pos_pairs, npos, generator=None):
    """`ddp_trainer.py:400-415`: one uniformly random key per unique query, then at most `npos` of them.
    pos_pairs: int tensor [P, 2] on the device, grouped by column 0.  Returns (q_rows, k_rows) int64."""
    dev = pos_pairs.device
    q_unique, count = pos_pairs[:, 0].unique(return_counts=True)
    u = torch.rand(len(count), device=dev, generator=generator)
    off = torch.floor(u * count).long()
    cums = torch.cumsum(count, 0) - count
    k_sel = pos_pairs[:, 1][off + cums]
    if npos < q_unique.shape[0]:
        pick = torch.randperm(q_unique.shape[0], device=dev, generator=generator)[:npos]
        q_unique, k_sel = q_unique[pick], k_sel[pick]
    return q_unique.long(), k_sel.long()


def point_nce_loss(F0, F1, q_rows, k_rows, T):
    """loss = CrossEntropy(F0[q] F1[k]^T / T, arange)   (`ddp_trainer.py:409-426`)."""
    return _PointNCEFunction.apply(F0[q_rows], F1[k_rows], 1.0 / T)


def pdist_rowmin(A, B):
    """(min_j sqrt(|A_i - B_j|^2 + 1e-7), argmin_j) without materialising the [P, S, D] broadcast (`:182-184,215-219`)."""
    _lib.require_cuda(A)
    A, B = A.detach().contiguous().float(), B.detach().contiguous().float()
    P, D = A.shape
    S = B.shape[0]
    minval = torch.empty(P, dtype=torch.float32, device=A.device)
    argmin = torch.empty(P, dtype=torch.int32, device=A.device)
    packed = torch.empty(P, dtype=torch.int64, device=A.device)
    with torch.cuda.device(A.device):
        check(lib.pcb_pdist_rowmin(ptr(A), P, ptr(B), S, D, ptr(minval), ptr(argmin), ptr(packed), stream()))
    return minval, argmin


def hardest_contrastive_loss(F0, F1, pos_pairs, sel0, sel1, pos_sel=None, pos_thresh=0.1, neg_thresh=1.4):
    """`ddp_trainer.py:186-238`.  sel0/sel1: hard-negative candidate rows (`:199-200`); pos_sel: positive subsample
    (`:203`) or None.  The false-negative mask (`:224-234`, a CPU np.isin in the reference) stays on the device."""
    N0, N1 = F0.shape[0], F1.shape[0]
    hash_seed = max(N0, N1)
    pos_pairs = pos_pairs.long()
    sample = pos_pairs if pos_sel is None else pos_pairs[pos_sel.long()]
    i0, i1 = sample[:, 0], sample[:, 1]
    sel0, sel1 = sel0.long(), sel1.long()
    posF0, posF1 = F0[i0], F1[i1]
    subF0, subF1 = F0[sel0], F1[sel1]
    _, j01 = pdist_rowmin(posF0, subF1)
    _, j10 = pdist_rowmin(posF1, subF0)
    j01, j10 = j01.long(), j10.long()
    D01min = torch.sqrt(((posF0 - subF1[j01]) ** 2).sum(1) + 1e-7)
    D10min = torch.sqrt(((posF1 - subF0[j10]) ** 2).sum(1) + 1e-7)
    pos_keys = pos_pairs[:, 0] + pos_pairs[:, 1] * hash_seed
    mask0 = ~torch.isin(i0 + sel1[j01] * hash_seed, pos_keys)
    mask1 = ~torch.isin(sel0[j10] + i1 * hash_seed, pos_keys)
    pos_loss = torch.relu(((posF0 - posF1) ** 2).sum(1) - pos_thresh)
    neg0 = (torch.relu(neg_thresh - D01min) ** 2 * mask0).sum() / mask0.sum()
    neg1 = (torch.relu(neg_thresh - D10min) ** 2 * mask1).sum() / mask1.sum()
    return pos_loss.mean(), (neg0 + neg1) / 2
