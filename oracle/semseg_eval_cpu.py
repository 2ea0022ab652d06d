"""numpy restatement (fp64) of the semantic-segmentation evaluation (`downstream/semseg/lib/test.py:62-196`, `lib/utils.py:117-138`),
the checker of `pcb_seg_metrics` / `pcb_average_precision` and of `pointcontrast_b200.semseg.SegmentationMetrics`.

* per row: pred = first index of the maximum, a NaN counting as maximal (torch `output.max(1)[1]`, `utils.py:264-265`); prob = softmax;
  cross-entropy lse - x[t] on the rows with t in [0, C) and t != ignore_index, the batch loss their mean (NaN if there is none,
  `test.py:137-138`);
* precision@1 = 100 * hits / rows with t != 255 (`precision_at_one` hard-codes 255, `utils.py:117-128`), in fp32 as torch computes it;
* hist[t, pred] += 1 for 0 <= t < C (`fast_hist`, `utils.py:131-133`); loss and score are weighted by the batch's row count
  (`AverageMeter.update(v, num_sample)`);
* average precision per class (`test.py:55-59`): `label_binarize` makes every row whose target is not c a negative of class c, an
  ignored or out-of-range target included; sklearn's uninterpolated AP = sum over tie groups of (R_g - R_{g-1}) * P_g, with -0.0 tied
  to +0.0.  A class with NO positive in the batch gets NaN -- the reference's `np.nanmean(aps, 0)` then skips that batch, as its own
  comment expects ("there exists class with no test label at all", `test.py:146`); scikit-learn >= 1.1 returns 0.0 there instead.  A
  NaN score in a column with a positive gives NaN (sklearn raises).
"""
import warnings

import numpy as np


def argmax_first(logits):
    """`output.max(1)[1]`: the first maximal index, the first NaN if the row has one."""
    x = np.asarray(logits)
    nan = np.isnan(x)
    pred = np.argmax(np.where(nan, -np.inf, x), axis=1)
    has = nan.any(1)
    pred[has] = np.argmax(nan[has], axis=1)
    return pred


def softmax(logits):
    x = np.asarray(logits, np.float64)
    e = np.exp(x - x.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def batch_loss(logits, target, ignore_index):
    x = np.asarray(logits, np.float64)
    t = np.asarray(target, np.int64)
    C = x.shape[1]
    ok = (t != ignore_index) & (t >= 0) & (t < C)
    if not ok.any():
        return float("nan")
    m = x.max(1)
    lse = m + np.log(np.exp(x - m[:, None]).sum(1))
    return float(np.mean(lse[ok] - x[ok, t[ok]]))


def precision_at_one(pred, target):
    keep = np.asarray(target) != 255
    if not keep.any():
        return float("nan")
    hits = np.float32(np.count_nonzero(np.asarray(pred)[keep] == np.asarray(target)[keep]))
    return float(hits * np.float32(100.0 / keep.sum()))


def fast_hist(pred, target, C):
    t = np.asarray(target, np.int64)
    k = (t >= 0) & (t < C)
    return np.bincount(C * t[k] + np.asarray(pred, np.int64)[k], minlength=C * C).reshape(C, C)


def average_precision(score, target):
    """Per-class AP [C] (fp64) of score [n, C] against target [n]; NaN for a class without a positive."""
    s = np.asarray(score, np.float64)
    t = np.asarray(target, np.int64)
    n, C = s.shape
    out = np.full(C, np.nan)
    for c in range(C):
        y = t == c
        T = int(y.sum())
        col = s[:, c] + 0.0                          # -0.0 + 0.0 == +0.0
        if T == 0 or np.isnan(col).any():
            continue
        order = np.argsort(-col, kind="stable")
        sc, tp = col[order], np.cumsum(y[order])
        ends = np.flatnonzero(np.r_[sc[1:] != sc[:-1], True])        # last entry of each tie group
        tp_end = tp[ends].astype(np.float64)
        tp_before = np.r_[0.0, tp_end[:-1]]
        out[c] = np.sum((tp_end - tp_before) * tp_end / (ends + 1.0)) / T
    return out


class Accumulator:
    """`test.py:68-149,196`: the running sums over batches and the 4-tuple (loss, score, mAP, mIoU)."""

    def __init__(self, C, ignore_index):
        self.C, self.ignore_index = C, ignore_index
        self.hist = np.zeros((C, C), np.int64)
        self.stats = np.zeros(3)                       # sum loss * n, sum score * n, sum n
        self.ap_sum, self.ap_cnt = np.zeros(C), np.zeros(C, np.int64)

    def update(self, logits, target, score=None):
        """score: the AP scores (the softmax of the logits unless given)."""
        n = len(target)
        pred = argmax_first(logits)
        self.hist += fast_hist(pred, target, self.C)
        self.stats += (batch_loss(logits, target, self.ignore_index) * n, precision_at_one(pred, target) * n, n)
        ap = average_precision(softmax(logits) if score is None else score, target)
        present = fast_hist(np.asarray(target), target, self.C).diagonal() > 0       # classes with a positive in the batch
        self.ap_sum[present] += ap[present]
        self.ap_cnt[present] += 1
        return pred

    def result(self):
        return finalize(self.hist, self.stats, self.ap_sum, self.ap_cnt)


def finalize(hist, stats, ap_sum, ap_cnt):
    """(loss, score, mAP, mIoU), per-class IoU / AP / accuracy (all x100), from the accumulators (`utils.py:136-138`, `test.py:141,149,196`)."""
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        iu = np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))
        ap_class = np.where(ap_cnt > 0, ap_sum / ap_cnt, np.nan) * 100.0
        acc = hist.diagonal() / hist.sum(1) * 100
        out = (stats[0] / stats[2], stats[1] / stats[2], float(np.nanmean(ap_class)), float(np.nanmean(iu)) * 100)
    return out, dict(iou=iu * 100, ap=ap_class, acc=acc, hist=hist)
