"""fp64 numpy restatement of VoteNet's `models/loss_helper.py::get_loss` (with `lib/utils/nn_distance.py`) and its analytic gradients:
the checker of csrc/det_loss.cu.  Inputs are the end_points arrays as numpy (any float dtype, computed in fp64); the dataset config is
(mean_size [NS, 3], NH, C).  The denominators of the vote and objectness-label means are fp32, as the original's `.float()` makes them.  Ties go to the first index (torch.min / torch.argmax); the padded label slots take part in every nearest
search, as in the original.

    forward(ep, mean_size, NH, C) -> dict: the 13 outputs of pointcontrast_b200.det_loss.OUTPUTS, objectness_label / objectness_mask /
                                     object_assignment [B, K], vote_pick [B, S] (j * V + v), cidx1 [B, K], cidx2 [B, K2]
    backward(ep, res, grad)      -> dict of the gradients of GRAD_INPUTS given d/d out (13 entries, or the 8 terms)
"""
import numpy as np

TERMS = ("vote_loss", "objectness_loss", "center_loss", "heading_cls_loss", "heading_reg_loss", "size_cls_loss", "size_reg_loss",
         "sem_cls_loss")
OUTPUTS = TERMS + ("box_loss", "loss", "pos_ratio", "neg_ratio", "obj_acc")
WEIGHTS = np.array([0.2, 0.8])


def _den32(x):
    """sum(x) + 1e-6 where the original sums `.float()` of an integer tensor: fp32 even when everything else is fp64."""
    return float(np.float32(x.sum()) + np.float32(1e-6))


def _f(ep, k):
    return np.asarray(ep[k], np.float64)


def _sqd(a, b):
    """[..., N, M] squared distances ((dx dx + dy dy) + dz dz) of a [..., N, 3] to b [..., M, 3]."""
    d = a[..., :, None, :] - b[..., None, :, :]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _log_softmax(x):
    m = x.max(-1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(-1, keepdims=True))


def _softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _take(a, idx):
    """a [B, K2, ...] gathered at idx [B, K] along axis 1."""
    return a[np.arange(a.shape[0])[:, None], idx]


def _huber(x):
    a = np.abs(x)
    q = np.minimum(a, 1.0)
    return 0.5 * q * q + (a - q)


def _labels(ep, res):
    a = res["object_assignment"]
    return (_take(np.asarray(ep["heading_class_label"], np.int64), a), _take(np.asarray(ep["size_class_label"], np.int64), a),
            _take(np.asarray(ep["sem_cls_label"], np.int64), a))


def forward(ep, mean_size, NH, C):
    seed_xyz, vote_xyz = _f(ep, "seed_xyz"), _f(ep, "vote_xyz")
    B, S = seed_xyz.shape[:2]
    V = vote_xyz.shape[1] // S
    inds = np.asarray(ep["seed_inds"], np.int64)
    bb = np.arange(B)[:, None]
    gv = _f(ep, "vote_label")[bb, inds].reshape(B, S, 3, 3) + seed_xyz[:, :, None, :]
    vmask = np.asarray(ep["vote_label_mask"])[bb, inds].astype(np.float64)
    d = np.abs(vote_xyz.reshape(B, S, V, 1, 3) - gv[:, :, None, :, :])
    d = (d[..., 0] + d[..., 1]) + d[..., 2]                                # [B, S, V, 3]
    vj = d.argmin(2)                                                        # per GT vote, the nearest predicted vote
    dj = d.min(2)
    j = dj.argmin(2)
    vote_dist = dj.min(2)
    pick = j * V + np.take_along_axis(vj, j[..., None], 2)[..., 0]
    r = {"vote_pick": pick}
    vote_loss = (vote_dist * vmask).sum() / _den32(vmask)

    gt = _f(ep, "center_label")[:, :, 0:3]
    da = _sqd(_f(ep, "aggregated_vote_xyz"), gt)
    assignment = da.argmin(2)
    e = np.sqrt(da.min(2) + 1e-6)
    label = (e < 0.3).astype(np.int64)
    mask = ((e < 0.3) | (e > 0.6)).astype(np.float64)
    r.update(objectness_label=label, objectness_mask=mask, object_assignment=assignment)
    obj = _f(ep, "objectness_scores")
    ce = -np.take_along_axis(_log_softmax(obj), label[..., None], 2)[..., 0] * WEIGHTS[label]
    obj_loss = (ce * mask).sum() / (mask.sum() + 1e-6)

    dc = _sqd(_f(ep, "center"), gt)
    r["cidx1"], r["cidx2"] = dc.argmin(2), dc.argmin(1)
    lf = label.astype(np.float64)
    box_mask = _f(ep, "box_label_mask")
    lden = _den32(lf)
    center_loss = (dc.min(2) * lf).sum() / lden + (dc.min(1) * box_mask).sum() / (box_mask.sum() + 1e-6)

    hc, sc, cc = _labels(ep, r)

    def ce_of(x, y):
        return -np.take_along_axis(_log_softmax(x), y[..., None], 2)[..., 0]

    hcls = (ce_of(_f(ep, "heading_scores"), hc) * lf).sum() / lden
    hr_label = _take(_f(ep, "heading_residual_label"), assignment) / (np.pi / NH)
    hres = np.take_along_axis(_f(ep, "heading_residuals_normalized"), hc[..., None], 2)[..., 0]
    hreg = (_huber(hres - hr_label) * lf).sum() / lden
    scls = (ce_of(_f(ep, "size_scores"), sc) * lf).sum() / lden
    ms = np.asarray(mean_size, np.float32).astype(np.float64)
    sr_label = _take(_f(ep, "size_residual_label"), assignment) / ms[sc]
    sres = _f(ep, "size_residuals_normalized")[bb, np.arange(sc.shape[1])[None, :], sc]
    sreg = (_huber(sres - sr_label).mean(-1) * lf).sum() / lden
    sem = (ce_of(_f(ep, "sem_cls_scores"), cc) * lf).sum() / lden

    box = center_loss + 0.1 * hcls + hreg + 0.1 * scls + sreg
    loss = (vote_loss + 0.5 * obj_loss + box + 0.1 * sem) * 10
    BK = float(label.size)
    pred = obj.argmax(2)
    pos = np.float32(lf.sum()) / np.float32(BK)                      # the original's ratios of `.float()` sums, in fp32
    neg = np.float32(mask.sum()) / np.float32(BK) - pos
    vals = (vote_loss, obj_loss, center_loss, hcls, hreg, scls, sreg, sem, box, loss, pos, neg,
            ((pred == label) * mask).sum() / (mask.sum() + 1e-6))
    r.update(zip(OUTPUTS, (float(v) for v in vals)))
    return r


def fold(grad):
    """d/d (the eight terms) from d/d out (13 entries; 8 are taken as the terms alone)."""
    g = np.zeros(len(OUTPUTS))
    g[:len(grad)] = np.asarray(grad, np.float64)
    gl = 10 * g[9]
    gb = g[8] + gl
    return g[:8] + gl * np.array([1, 0.5, 0, 0, 0, 0, 0, 0.1]) + gb * np.array([0, 0, 1, 0.1, 1, 0.1, 1, 0])


def backward(ep, res, grad, mean_size, NH):
    G = fold(grad)
    seed_xyz, vote_xyz = _f(ep, "seed_xyz"), _f(ep, "vote_xyz")
    B, S = seed_xyz.shape[:2]
    V = vote_xyz.shape[1] // S
    bb = np.arange(B)[:, None]
    inds = np.asarray(ep["seed_inds"], np.int64)
    vmask = np.asarray(ep["vote_label_mask"])[bb, inds].astype(np.float64)
    gv = _f(ep, "vote_label")[bb, inds].reshape(B, S, 3, 3) + seed_xyz[:, :, None, :]
    pick = res["vote_pick"]
    j, v = pick // V, pick % V
    vx = vote_xyz.reshape(B, S, V, 3)
    ss = np.arange(S)[None, :]
    sgn = np.sign(vx[bb, ss, v] - gv[bb, ss, j])
    w = G[0] / _den32(vmask) * vmask
    g_vote = np.zeros((B, S, V, 3))
    g_vote[bb, ss, v] = w[..., None] * sgn
    out = {"vote_xyz": g_vote.reshape(B, S * V, 3), "seed_xyz": -(w[..., None] * sgn)}

    label, mask, a = res["objectness_label"], res["objectness_mask"], res["object_assignment"]
    lf = label.astype(np.float64)
    lden = _den32(lf)
    obj = _f(ep, "objectness_scores")
    onehot = lambda y, n: np.eye(n)[y]
    out["objectness_scores"] = (G[1] / (mask.sum() + 1e-6) * mask * WEIGHTS[label])[..., None] * (_softmax(obj) - onehot(label, 2))

    gt = _f(ep, "center_label")[:, :, 0:3]
    c = _f(ep, "center")
    K = c.shape[1]
    box_mask = _f(ep, "box_label_mask")
    gc = (G[2] / lden * lf)[..., None] * 2 * (c - _take(gt, res["cidx1"]))
    w2 = G[2] / (box_mask.sum() + 1e-6) * box_mask                      # [B, K2]
    c2 = c[bb, res["cidx2"]]                                            # the proposal each slot picked
    contrib = w2[..., None] * 2 * (c2 - gt)                             # [B, K2, 3]
    for b in range(B):
        np.add.at(gc[b], res["cidx2"][b], contrib[b])
    out["center"] = gc

    hc, sc, cc = _labels(ep, res)
    kk = np.arange(K)[None, :]
    for key, y, gi in (("heading_scores", hc, 3), ("size_scores", sc, 5), ("sem_cls_scores", cc, 7)):
        x = _f(ep, key)
        out[key] = (G[gi] / lden * lf)[..., None] * (_softmax(x) - onehot(y, x.shape[-1]))
    hr = _f(ep, "heading_residuals_normalized")
    d = hr[bb, kk, hc] - _take(_f(ep, "heading_residual_label"), a) / (np.pi / NH)
    g = np.zeros_like(hr)
    g[bb, kk, hc] = G[4] / lden * lf * np.clip(d, -1, 1)
    out["heading_residuals_normalized"] = g
    sr = _f(ep, "size_residuals_normalized")
    ms = np.asarray(mean_size, np.float32).astype(np.float64)
    d = sr[bb, kk, sc] - _take(_f(ep, "size_residual_label"), a) / ms[sc]
    g = np.zeros_like(sr)
    g[bb, kk, sc] = (G[6] / lden * lf / 3)[..., None] * np.clip(d, -1, 1)
    out["size_residuals_normalized"] = g
    return out
