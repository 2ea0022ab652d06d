"""pointcontrast_b200.det_loss and csrc/det_loss.cu against the fp64 oracle (oracle/det_loss_cpu.py), the original's fp64 numbers
(tests/golden/detection_loss.npz) and, where oracle/det_eval_ref.py staged it, the original `loss_helper.get_loss` in fp32 on the GPU.

Error bound on exactly representable operands.  Coordinates are multiples of 2^-6 below 8 in magnitude, so every fp32 difference, square,
sum of three squares and L1 distance is exact: the assignments, labels, masks and vote argmins equal the oracle's bit for bit, ties
included.  Each remaining per-element value takes at most n + 8 fp32 roundings (n = the row length of a cross-entropy: its exp-sum,
one log, subtractions; Huber and the residual normalisation fewer), i.e. a relative error below (n + 8) 2^-24 <= 26 * 6e-8 < 2e-6 of the
element's magnitude; the batch sums are fp64 and each result is rounded once to fp32 (another 6e-8).  So each loss is within
2e-6 * (sum of |element| / denominator) + 6e-8 |loss| of fp64; the test allows 4e-6 relative.  Gradients are one fp32 softmax entry or
sign / clamp times a scale (a few roundings each): within 4e-6 relative to the largest gradient of the tensor.
"""
import numpy as np
import pytest
import torch

from oracle import det_loss_cpu as O
from pointcontrast_b200 import synth
from tests.test_oracle_det_loss import CASES, GRAD_INPUTS, golden

pytestmark = pytest.mark.gpu

DATASETS = {"scannet": (1, 18, 18), "sunrgbd": (12, 10, 10)}        # NH, NS, C
LOSS_INPUTS = ("seed_xyz", "seed_inds", "vote_xyz", "aggregated_vote_xyz", "center", "objectness_scores", "heading_scores",
               "heading_residuals_normalized", "size_scores", "size_residuals_normalized", "sem_cls_scores", "center_label",
               "heading_class_label", "heading_residual_label", "size_class_label", "size_residual_label", "sem_cls_label",
               "box_label_mask", "vote_label", "vote_label_mask")


class Config:
    def __init__(self, NH, NS, C, mean_size):
        self.num_heading_bin, self.num_size_cluster, self.num_class, self.mean_size_arr = NH, NS, C, np.asarray(mean_size)


@pytest.fixture(scope="module")
def dl():
    from pointcontrast_b200 import det_loss
    return det_loss


def batch(dname, seed, B=2, N=3000, S=256, K=64, V=1, K2=64):
    NH, NS, C = DATASETS[dname]
    ms = np.random.default_rng(seed).uniform(0.3, 2.0, (NS, 3))
    return synth.synth_votenet_loss_batch(seed, B, N, S, K, V, NH, ms, C, max_obj=K2), ms, Config(NH, NS, C, ms)


def dyadic(ep):
    """Coordinates rounded to multiples of 2^-6 (|x| < 8): every distance the kernel takes is exact in fp32."""
    q = lambda a: np.clip(np.round(a * 64) / 64, -7.5, 7.5).astype(np.float32)
    out = dict(ep)
    for k in ("seed_xyz", "vote_xyz", "aggregated_vote_xyz", "center", "center_label"):
        out[k] = q(ep[k])
    out["vote_label"] = q(ep["vote_label"])
    return out


def run(dl, ep, cfg, grad_of="loss", device="cuda"):
    """(end_points after get_loss, {input: gradient}) with the loss inputs as fresh device tensors."""
    t = {k: torch.from_numpy(np.ascontiguousarray(ep[k])).to(device) for k in LOSS_INPUTS}
    for k in GRAD_INPUTS:
        t[k].requires_grad_(True)
    loss, out = dl.get_loss(dict(t), cfg)
    if grad_of is not None:
        out[grad_of].backward()
    return out, {k: (t[k].grad.cpu().numpy() if t[k].grad is not None else None) for k in GRAD_INPUTS}


def check_against(out, grads, want, gwant, rtol, gtol):
    for k in ("objectness_label", "objectness_mask", "object_assignment"):
        assert np.array_equal(out[k].cpu().numpy(), want[k]), k
    for k in O.OUTPUTS:
        a, b = float(out[k].detach()), float(want[k])
        assert abs(a - b) <= rtol * max(abs(b), 1e-3), (k, a, b)
    for k in GRAD_INPUTS:
        g, w = grads[k], gwant[k]
        scale = max(np.abs(w).max(), 1e-30)
        assert np.abs(g - w).max() <= gtol * scale, (k, np.abs(g - w).max(), scale)
        assert np.array_equal(g != 0, w != 0) or k not in ("vote_xyz", "seed_xyz"), k    # the vote argmins


@pytest.mark.parametrize("dname", sorted(DATASETS))
@pytest.mark.parametrize("V", [1, 3])
def test_exact_operands_match_oracle(dl, dname, V):
    ep, ms, cfg = batch(dname, 7 + V, V=V)
    ep = dyadic(ep)
    ep["aggregated_vote_xyz"][0, 0] = (ep["center_label"][0, 0] + ep["center_label"][0, 1]) / 2     # an exact tie (dyadic midpoint)
    ep["vote_xyz"][0, 0:V] = ep["seed_xyz"][0, 0]
    NH, NS, C = DATASETS[dname]
    r = O.forward(ep, ms, NH, C)
    out, grads = run(dl, ep, cfg)
    check_against(out, grads, r, O.backward(ep, r, np.eye(13)[9], ms, NH), 4e-6, 4e-6)


@pytest.mark.parametrize("name", CASES)
def test_golden(dl, name):
    ep, ms, (NH, NS, C), want = golden(name)
    out, grads = run(dl, ep, Config(NH, NS, C, ms))
    check_against(out, grads, want, {k: want["grad_" + k] for k in GRAD_INPUTS}, 1e-5, 1e-5)


def _strided_inputs(ep, NH, NS, C, device):
    """The proposal outputs sliced from one [B, X, K] tensor as `decode_scores` slices them, and that tensor."""
    B, K = ep["center"].shape[:2]
    parts = [ep["objectness_scores"], ep["center"], ep["heading_scores"], ep["heading_residuals_normalized"], ep["size_scores"],
             ep["size_residuals_normalized"].reshape(B, K, NS * 3), ep["sem_cls_scores"]]
    net = torch.from_numpy(np.ascontiguousarray(np.concatenate(parts, 2).transpose(0, 2, 1))).to(device).requires_grad_(True)
    nt = net.transpose(2, 1)
    o = 5 + 2 * NH + NS
    views = {"objectness_scores": nt[:, :, 0:2], "center": nt[:, :, 2:5], "heading_scores": nt[:, :, 5:5 + NH],
             "heading_residuals_normalized": nt[:, :, 5 + NH:5 + 2 * NH], "size_scores": nt[:, :, 5 + 2 * NH:o],
             "size_residuals_normalized": nt[:, :, o:o + 3 * NS].view(B, K, NS, 3), "sem_cls_scores": nt[:, :, o + 3 * NS:]}
    return net, views


@pytest.mark.parametrize("dname", sorted(DATASETS))
def test_strided_inputs(dl, dname):
    NH, NS, C = DATASETS[dname]
    ep, ms, cfg = batch(dname, 3)
    ref, gref = run(dl, ep, cfg)
    net, views = _strided_inputs(ep, NH, NS, C, "cuda")
    assert not views["heading_scores"].is_contiguous()
    t = {k: torch.from_numpy(np.ascontiguousarray(ep[k])).cuda() for k in LOSS_INPUTS if k not in views}
    t.update(views)
    t["vote_xyz"].requires_grad_(True)
    loss, out = dl.get_loss(t, cfg)
    loss.backward()
    for k in O.OUTPUTS + ("objectness_label", "objectness_mask", "object_assignment"):
        assert torch.equal(out[k], ref[k]), k
    g = net.grad.transpose(2, 1).cpu().numpy()
    B, K = ep["center"].shape[:2]
    want = np.concatenate([gref["objectness_scores"], gref["center"], gref["heading_scores"], gref["heading_residuals_normalized"],
                           gref["size_scores"], gref["size_residuals_normalized"].reshape(B, K, NS * 3), gref["sem_cls_scores"]], 2)
    assert np.array_equal(g, want)
    assert np.array_equal(t["vote_xyz"].grad.cpu().numpy(), gref["vote_xyz"])


def test_sub_loss_backwards_are_separable(dl):
    ep, ms, cfg = batch("sunrgbd", 5, V=3)
    NH, NS, C = DATASETS["sunrgbd"]
    r = O.forward(ep, ms, NH, C)
    for i, term in enumerate(O.TERMS):
        out, grads = run(dl, ep, cfg, grad_of=term)
        want = O.backward(ep, r, np.eye(8)[i], ms, NH)
        for k in GRAD_INPUTS:
            scale = np.abs(want[k]).max()
            if scale == 0:
                assert grads[k] is None or not grads[k].any(), (term, k)
            else:
                assert np.abs(grads[k] - want[k]).max() <= 1e-5 * scale, (term, k)


def test_runs_are_bit_identical(dl):
    ep, ms, cfg = batch("scannet", 11, B=8, N=4000, S=1024, K=256)
    a, ga = run(dl, ep, cfg)
    b, gb = run(dl, ep, cfg)
    for k in O.OUTPUTS:
        assert a[k].detach().cpu().numpy().tobytes() == b[k].detach().cpu().numpy().tobytes(), k
    for k in GRAD_INPUTS:
        assert ga[k].tobytes() == gb[k].tobytes(), k


def test_no_host_sync(dl):
    ep, ms, cfg = batch("sunrgbd", 12)
    t = {k: torch.from_numpy(np.ascontiguousarray(ep[k])).cuda() for k in LOSS_INPUTS}
    for k in GRAD_INPUTS:
        t[k].requires_grad_(True)
    dl.get_loss(dict(t), cfg)                          # warm-up: workspace allocation
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, out = dl.get_loss(dict(t), cfg)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss).item()


def test_out_of_range_labels_give_nan(dl):
    ep, ms, cfg = batch("sunrgbd", 13)
    NH, NS, C = DATASETS["sunrgbd"]
    r = O.forward(ep, ms, NH, C)
    j = r["object_assignment"][0, 0]
    bad = dict(ep, heading_class_label=ep["heading_class_label"].copy(), seed_inds=ep["seed_inds"].copy())
    bad["heading_class_label"][0, j] = NH
    bad["seed_inds"][1, 3] = ep["vote_label"].shape[1]
    out, grads = run(dl, bad, cfg)
    torch.cuda.synchronize()
    for k in ("heading_cls_loss", "heading_reg_loss", "vote_loss", "box_loss", "loss"):
        assert np.isnan(float(out[k])), k
    for k in ("objectness_loss", "center_loss", "size_cls_loss", "size_reg_loss", "sem_cls_loss"):
        assert np.isfinite(float(out[k])), k
    sem = dict(ep, sem_cls_label=ep["sem_cls_label"] - 100)
    out, _ = run(dl, sem, cfg)
    assert np.isnan(float(out["sem_cls_loss"])) and np.isfinite(float(out["vote_loss"]))


def _original():
    from oracle import det_eval_ref
    if det_eval_ref.load() is None:
        pytest.skip("the original VoteNet code is not staged under oracle/_ref/")
    import importlib
    return importlib.import_module("models.loss_helper")


def _margins(ep):
    """fp64 gap between the nearest label slot of every proposal and the nearest one at another distance (the assignment's margin;
    the padded slots share one position, and their tie goes to the first in both implementations), and the threshold margin."""
    d = O._sqd(np.asarray(ep["aggregated_vote_xyz"], np.float64), np.asarray(ep["center_label"], np.float64))
    s = np.sort(d, 2)
    gaps = s[..., 1:] - s[..., :1]
    e = np.sqrt(s[..., 0] + 1e-6)
    return np.where(gaps > 0, gaps, np.inf).min(2), np.minimum(np.abs(e - 0.3), np.abs(e - 0.6))


@pytest.mark.parametrize("dname", sorted(DATASETS))
def test_full_size_against_original(dl, dname):
    """B 8, 1024 seeds, 256 proposals, 64 slots.  Assignments and labels must be equal wherever the fp64 margin exceeds 1e-4 (far
    above the fp32 rounding of a squared distance below 100); values within 1e-4 relative, gradients within 1e-4 of the largest."""
    ref = _original()
    ep, ms, cfg = batch(dname, 21, B=8, N=20000, S=1024, K=256)
    gap, thr = _margins(ep)
    ours, g_ours = run(dl, ep, cfg)
    t = {k: torch.from_numpy(np.ascontiguousarray(ep[k])).cuda() for k in LOSS_INPUTS}
    for k in GRAD_INPUTS:
        t[k].requires_grad_(True)
    t["seed_inds"] = t["seed_inds"].long()
    loss, theirs = ref.get_loss(dict(t), cfg)
    loss.backward()
    sure = (gap > 1e-4) & (thr > 1e-4)
    assert sure.mean() > 0.95
    for k in ("objectness_label", "objectness_mask", "object_assignment"):
        a, b = ours[k].cpu().numpy(), theirs[k].cpu().numpy()
        assert np.array_equal(a[sure], b[sure]), k
    for k in O.OUTPUTS:
        a, b = float(ours[k]), float(theirs[k])
        assert abs(a - b) <= 1e-4 * max(abs(b), 1e-2), (k, a, b)
    for k in GRAD_INPUTS:
        a, b = g_ours[k], t[k].grad.cpu().numpy()
        assert np.abs(a - b).max() <= 1e-4 * max(np.abs(b).max(), 1e-30), k


class DatasetConfig(Config):
    """What the original's lib/test.py and ap_helper read besides the loss: ScanNet's heading rule (class2angle 0) and class2size."""

    def __init__(self, NH, NS, C, mean_size):
        super().__init__(NH, NS, C, mean_size)
        self.class2type = {c: f"c{c}" for c in range(C)}

    def class2angle(self, pred_cls, residual, to_label_format=True):
        return 0

    def class2size(self, pred_cls, residual):
        return self.mean_size_arr[pred_cls, :] + residual


def _run_lib_test(dl, install, batches, cfg):
    """The original's unmodified lib/test.py::test over `batches`, fed by a stand-in net (the batch's predictions), with the original
    criterion or, after det_loss.install(), ours; the PLY dump of batch 0 is replaced by a no-op.  Returns the logged 'eval mean' lines."""
    import importlib
    import logging
    import sys
    import types
    pkg = sys.modules["models"]
    saved = sys.modules["models.loss_helper"]
    pred_keys = ("seed_xyz", "seed_inds", "vote_xyz", "aggregated_vote_xyz", "center", "objectness_scores", "heading_scores",
                 "heading_residuals_normalized", "size_scores", "size_residuals_normalized", "sem_cls_scores")
    try:
        if install:
            dl.install()
        sys.modules.pop("lib.test", None)
        T = importlib.import_module("lib.test")
        calls = iter(range(len(batches)))

        class Net:
            def eval(self):
                return self

            def __call__(self, inputs):
                i = next(calls)
                ep = {k: torch.from_numpy(np.ascontiguousarray(batches[i][k])).cuda() for k in pred_keys}
                ep["heading_residuals"] = ep["heading_residuals_normalized"] * (np.pi / cfg.num_heading_bin)
                ep["size_residuals"] = ep["size_residuals_normalized"] * torch.from_numpy(cfg.mean_size_arr.astype(np.float32)).cuda()
                return ep

        T.dump_results = lambda *a, **k: None
        loader = [{k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in b.items() if k not in pred_keys} for b in batches]
        config = types.SimpleNamespace(test=types.SimpleNamespace(use_cls_nms=True, use_3d_nms=True, faster_eval=True, nms_iou=0.25,
                                                                  use_old_type_nms=False, per_class_proposal=True, conf_thresh=0.05,
                                                                  ap_iou_thresholds=[0.25]))
        lines = []
        handler = logging.Handler(logging.INFO)
        handler.emit = lambda r: lines.append(r.getMessage())
        root = logging.getLogger()
        old_level = root.level
        root.addHandler(handler)
        root.setLevel(logging.INFO)
        try:
            T.test(Net(), loader, cfg, config)
        finally:
            root.removeHandler(handler)
            root.setLevel(old_level)
        assert (T.criterion is dl.get_loss) == install
    finally:
        sys.modules["models.loss_helper"] = saved
        pkg.loss_helper = saved
        sys.modules.pop("lib.test", None)
    return [l for l in lines if l.startswith("eval mean")]


def test_original_test_loop_with_and_without_install(dl):
    """lib/test.py::test logs the same mean losses, ratios and accuracy (as it prints them, %f) with the original criterion and after
    det_loss.install(), over two ScanNet-shaped batches."""
    _original()
    NH, NS, C = DATASETS["scannet"]
    ms = np.random.default_rng(4).uniform(0.3, 2.0, (NS, 3))
    batches = [synth.synth_votenet_loss_batch(s, 4, 4000, 512, 128, 1, NH, ms, C) for s in (31, 32)]
    cfg = DatasetConfig(NH, NS, C, ms)
    ref = _run_lib_test(dl, False, batches, cfg)
    ours = _run_lib_test(dl, True, batches, cfg)
    assert len(ref) == len(ours) == 13
    for a, b in zip(ref, ours):
        ka, _, va = a.rpartition(": ")
        kb, _, vb = b.rpartition(": ")
        assert ka == kb and abs(float(va) - float(vb)) <= 2e-6 * max(1.0, abs(float(va))), (a, b)


def test_votenet_training_step_gradients(dl):
    """One training step of the original VoteNet (sparse-conv backbone on this library, after me.install() / pointnet2.install()):
    every parameter gradient under our criterion equals the one under the original's within 1e-3 of its norm."""
    _original()
    from oracle import det_loss_ref
    if not det_loss_ref.available():
        pytest.skip("the original VoteNet heads are not staged under oracle/_ref/")
    import importlib
    from pointcontrast_b200 import detection
    from tests.helpers import det_init
    from tests.test_host_detection import original_backbone_module
    original_backbone_module()
    ref = _original()
    votenet = importlib.import_module("models.votenet")
    NH, NS, C = DATASETS["sunrgbd"]
    ms = np.random.default_rng(6).uniform(0.3, 2.0, (NS, 3))
    cfg = Config(NH, NS, C, ms)
    ep = synth.synth_votenet_loss_batch(41, 4, 20000, 1024, 256, 1, NH, ms, C)
    torch.manual_seed(0)
    net = votenet.VoteNet(C, NH, NS, ms, input_feature_dim=0, num_proposal=256, vote_factor=1, sampling="vote_fps",
                          backbone="sparseconv")
    det_init(net.backbone_net.net, 2)
    net = net.cuda().train()
    batch = detection.voxelize_batch({"point_clouds": torch.from_numpy(ep["point_clouds"]).cuda()}, 0.025)          # the voxel size of tests/test_gpu_detection.py
    labels = ("center_label", "heading_class_label", "heading_residual_label", "size_class_label", "size_residual_label",
              "sem_cls_label", "box_label_mask", "vote_label", "vote_label_mask")

    def step(criterion):
        net.zero_grad()
        end_points = net({k: batch[k] for k in ("point_clouds", "voxel_coords", "voxel_inds", "voxel_feats")})
        for k in labels:
            end_points[k] = torch.from_numpy(ep[k]).cuda()
        loss, end_points = criterion(end_points, cfg)
        loss.backward()
        return float(loss.detach()), {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

    la, ga = step(ref.get_loss)
    lb, gb = step(dl.get_loss)
    assert abs(la - lb) <= 1e-4 * abs(la)
    assert ga.keys() == gb.keys() and len(ga) > 50
    for k in ga:
        assert (ga[k] - gb[k]).norm() <= 1e-3 * max(ga[k].norm(), 1e-12), k
