"""The semantic-segmentation evaluation oracle (oracle/semseg_eval_cpu.py) against scikit-learn and against the reference's own
`lib/test.py::test` (tests/golden/semseg_eval.npz), and the argument checks of `pcb_seg_metrics` / `pcb_average_precision`, which
run before anything touches the device."""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import semseg_eval_cpu as O

metrics = pytest.importorskip("sklearn.metrics")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "semseg_eval.npz")


def sklearn_ap(score, target, C):
    """`test.py:55-59`: the one-hot labels of `label_binarize` (which for C > 2 is exactly this; for C <= 2 it returns one column),
    then average_precision_score per column (fp64)."""
    label = (np.asarray(target)[:, None] == np.arange(C)).astype(int)
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.array([metrics.average_precision_score(label[:, c], np.asarray(score, np.float64)[:, c]) for c in range(C)])


def ap_cases():
    g = np.random.default_rng(3)
    yield "random", g.standard_normal((300, 7)).astype(np.float32), g.integers(0, 7, 300)
    s = np.round(g.random((400, 5)) * 4).astype(np.float32) / 4             # exact fp32 ties with mixed labels
    yield "ties", s, g.integers(0, 5, 400)
    yield "all_equal", np.full((50, 3), 0.25, np.float32), g.integers(0, 3, 50)
    s = g.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), (200, 4))    # -0.0 ties +0.0
    yield "signed_zero", s, g.integers(0, 4, 200)
    yield "negative", -g.random((120, 6)).astype(np.float32) - 3.0, g.integers(0, 6, 120)
    t = np.full(90, 2)
    t[17] = 0
    t[40] = 1
    yield "one_positive", g.random((90, 3)).astype(np.float32), t
    t = g.integers(0, 4, 150)
    t[::5], t[1::7], t[2::9] = 255, -1, 7                                   # ignored and out-of-range: negatives of every class
    yield "ignored_out_of_range", g.random((150, 4)).astype(np.float32), t
    yield "n1", np.array([[0.3, 0.1]], np.float32), np.array([1])


@pytest.mark.parametrize("name,score,target", list(ap_cases()), ids=[c[0] for c in ap_cases()])
def test_oracle_ap_matches_sklearn(name, score, target):
    C = score.shape[1]
    ap = O.average_precision(score, target)
    ref = sklearn_ap(score, target, C)
    present = np.array([(target == c).any() for c in range(C)])
    assert present.any()
    assert np.all(np.abs(ap[present] - ref[present]) <= 1e-12), (ap, ref)
    assert np.isnan(ap[~present]).all()


def test_absent_class_is_nan_where_installed_sklearn_says_zero():
    """A class without a positive: the oracle (and the library) give NaN, which the reference's np.nanmean over batches skips, as its
    comment at `test.py:146` expects.  scikit-learn >= 1.1 returns 0.0 with a warning instead, which would count the batch as AP 0."""
    score = np.random.default_rng(0).random((40, 3)).astype(np.float32)
    target = np.array([0, 1] * 20)                                          # class 2 absent
    assert np.isnan(O.average_precision(score, target)[2])
    assert sklearn_ap(score, target, 3)[2] == 0.0


def test_nan_score_gives_nan():
    score = np.random.default_rng(1).random((30, 2)).astype(np.float32)
    score[4, 1] = np.nan
    ap = O.average_precision(score, np.arange(30) % 2)
    assert not np.isnan(ap[0]) and np.isnan(ap[1])


def test_argmax_and_precision():
    x = np.array([[1, 3, 3], [np.nan, 5, np.nan], [2, np.nan, 9], [-np.inf, -np.inf, -np.inf]], np.float32)
    assert O.argmax_first(x).tolist() == torch.from_numpy(x).max(1)[1].tolist() == [1, 0, 1, 0]
    assert np.isnan(O.precision_at_one(np.array([1, 2]), np.array([255, 255])))
    assert O.precision_at_one(np.array([1, 2, 0]), np.array([1, 255, 3])) == 50.0


def test_oracle_reproduces_reference_test_loop():
    """`lib/test.py::test` run unmodified on the golden logits (CPU torch softmax, scikit-learn AP): hist and mIoU exactly; loss within
    1e-6 relative (the reference's per-batch loss is torch's fp32 mean, the oracle's fp64); score and mAP within 1e-9 (the oracle
    scores the AP on the same fp32 torch softmax)."""
    z = np.load(GOLDEN)
    C = z["logits"].shape[1]
    acc = O.Accumulator(C, 255)
    off = np.r_[0, np.cumsum(z["sizes"])]
    for a, b in zip(off[:-1], off[1:]):
        x = z["logits"][a:b]
        acc.update(x, z["targets"][a:b], score=torch.softmax(torch.from_numpy(x), 1).numpy())
    (loss, score, mAP, mIoU), per = acc.result()
    loss_r, score_r, mAP_r, mIoU_r = z["result"]
    assert np.array_equal(per["hist"], z["hist"])
    assert mIoU == mIoU_r
    assert abs(loss - loss_r) <= 1e-6 * abs(loss_r)
    assert abs(score - score_r) <= 1e-9
    assert abs(mAP - mAP_r) <= 1e-9
    assert np.all(np.abs(per["ap"] - z["ap_class"]) <= 1e-9)


# ------------------------------------------------------------------------------------------------ argument checks (no GPU needed)

def _lib():
    from pointcontrast_b200 import _lib
    return _lib.lib


def test_seg_metrics_rejects_bad_arguments():
    L = _lib()
    n, C = 100, 20
    q = L.pcb_seg_metrics_ws_bytes(n)
    ws = torch.empty(q, dtype=torch.uint8)
    x, t = torch.zeros(n, C), torch.zeros(n, dtype=torch.int64)
    pred, hist, stats = torch.zeros(n, dtype=torch.int32), torch.zeros(C * C, dtype=torch.int64), torch.zeros(3, dtype=torch.float64)

    def call(n=n, C=C, x=x.data_ptr(), b=q, hist=hist.data_ptr()):
        return L.pcb_seg_metrics(x, t.data_ptr(), n, C, 255, pred.data_ptr(), None, hist, stats.data_ptr(), ws.data_ptr(), b, None)
    for rc in (call(n=0), call(C=0), call(C=1025), call(x=None), call(hist=None), call(b=q - 1)):
        assert rc == 2 and b"bad argument" in L.pcb_last_error()


def test_average_precision_rejects_bad_arguments():
    L = _lib()
    n, C = 100, 20
    q = L.pcb_average_precision_ws_bytes(n, C)
    ws = torch.empty(q, dtype=torch.uint8)
    s, t = torch.zeros(n, C), torch.zeros(n, dtype=torch.int64)
    ap_sum, ap_cnt = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.int64)

    def call(n=n, C=C, s=s.data_ptr(), b=q):
        return L.pcb_average_precision(s, t.data_ptr(), n, C, ap_sum.data_ptr(), ap_cnt.data_ptr(), ws.data_ptr(), b, None)
    for rc in (call(n=0), call(C=0), call(C=1025), call(s=None), call(b=q - 1), call(n=1 << 21, C=1024)):
        assert rc == 2 and b"bad argument" in L.pcb_last_error()
