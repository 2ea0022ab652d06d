"""Semantic-segmentation evaluation on the GPU (`downstream/semseg/lib/test.py:62-196`, `lib/train.py:22-232`): `pcb_average_precision`
and `pcb_seg_metrics` against the fp64 oracle (oracle/semseg_eval_cpu.py) and torch, `SegmentationMetrics` on the reference's golden
run, `semseg.test` on synthetic rooms, and `SegmentationTrainer.train` with checkpoints, validation and resume."""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import semseg_eval_cpu as O
from tests import refload

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "semseg_eval.npz")


def _L():
    from pointcontrast_b200 import _lib
    return _lib


def gpu_ap(score, target):
    """one pcb_average_precision call on fresh accumulators: (ap_sum, ap_cnt) on the host"""
    _lib = _L()
    s = torch.as_tensor(score, dtype=torch.float32).cuda().contiguous()
    t = torch.as_tensor(target, dtype=torch.int64).cuda().contiguous()
    n, C = s.shape
    q = _lib.lib.pcb_average_precision_ws_bytes(n, C)
    ws = torch.empty(q, dtype=torch.uint8, device="cuda")
    ap_sum, ap_cnt = torch.zeros(C, dtype=torch.float64, device="cuda"), torch.zeros(C, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.pcb_average_precision(s.data_ptr(), t.data_ptr(), n, C, ap_sum.data_ptr(), ap_cnt.data_ptr(), ws.data_ptr(), q,
                                              _lib.stream()))
    return ap_sum.cpu().numpy(), ap_cnt.cpu().numpy()


def _check_ap(score, target):
    score = np.asarray(score, np.float32)
    C = score.shape[1]
    ref = O.average_precision(score, target)
    present = np.array([(np.asarray(target) == c).any() for c in range(C)])
    ap_sum, ap_cnt = gpu_ap(score, target)
    assert np.array_equal(ap_cnt, present.astype(np.int64))
    got = ap_sum[present]
    assert np.array_equal(np.isnan(got), np.isnan(ref[present]))
    ok = ~np.isnan(got)
    assert np.all(np.abs(got[ok] - ref[present][ok]) <= 1e-12), np.abs(got[ok] - ref[present][ok]).max()
    assert np.all(ap_sum[~present] == 0)


def _cases():
    g = np.random.default_rng(7)
    yield "ties", np.round(g.random((400, 5)) * 4).astype(np.float32) / 4, g.integers(0, 5, 400)
    yield "all_equal", np.full((50, 3), 0.25, np.float32), g.integers(0, 3, 50)
    yield "signed_zero", g.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), (200, 4)), g.integers(0, 4, 200)
    yield "negative", -g.random((120, 6)).astype(np.float32) - 3.0, g.integers(0, 6, 120)
    t = np.full(90, 2); t[17] = 0; t[40] = 1
    yield "one_positive", g.random((90, 3)).astype(np.float32), t
    t = g.integers(0, 4, 150); t[::5], t[1::7], t[2::9] = 255, -1, 7
    yield "ignored_out_of_range", g.random((150, 4)).astype(np.float32), t
    yield "absent_class", g.random((64, 5)).astype(np.float32), g.integers(0, 3, 64)
    s = g.random((300, 4)).astype(np.float32); s[10, 2] = np.nan
    yield "nan_score", s, g.integers(0, 4, 300)
    yield "n1", np.array([[0.3, 0.1]], np.float32), np.array([1])
    for n in (255, 256, 257, 65_537):
        yield f"n{n}", g.random((n, 13)).astype(np.float32), g.integers(0, 13, n)
    for C in (1, 13, 20, 1024):
        n = 3000
        s = np.round(g.standard_normal((n, C)) * 64).astype(np.float32) / 64           # many ties
        yield f"C{C}", s, g.integers(0, C, n)


@pytest.mark.parametrize("name,score,target", list(_cases()), ids=[c[0] for c in _cases()])
def test_average_precision_matches_oracle(name, score, target):
    _check_ap(score, target)


def test_average_precision_scannet_size():
    g = np.random.default_rng(8)
    n, C = 120_000, 20
    t = g.integers(0, C, n); t[g.random(n) < 0.1] = 255
    x = torch.from_numpy(g.standard_normal((n, C)).astype(np.float32))
    x[torch.arange(n), torch.from_numpy(np.minimum(t, C - 1))] += 1.5
    _check_ap(torch.softmax(x, 1).numpy(), t)


def test_seg_metrics_against_torch():
    from pointcontrast_b200 import losses
    from pointcontrast_b200.semseg import SegmentationMetrics
    g = np.random.default_rng(9)
    n, C = 5000, 20
    x = np.round(g.standard_normal((n, C)) * 4).astype(np.float32) / 4          # ties within rows
    x[3, [2, 7]] = np.nan
    x[4, 5] = np.nan
    x[5, :] = 1.0
    t = g.integers(0, C, n); t[g.random(n) < 0.1] = 255; t[:3] = -1
    xt, tt = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    m = SegmentationMetrics(C, 255, "cuda")
    pred, prob = m.update(xt, tt)
    assert torch.equal(pred.long(), torch.max(xt, 1)[1])
    assert pred[3] == 2 and pred[4] == 5 and pred[5] == 0
    ok = ~np.isnan(x).any(1)
    p64 = O.softmax(x[ok])
    assert np.all(np.abs(prob.cpu().numpy()[ok] - p64) <= 1e-6 * p64)
    assert np.array_equal(m.hist.cpu().numpy().reshape(C, C), O.fast_hist(pred.cpu().numpy(), t, C))
    # the batch loss: the bits of pcb_ce_forward_backward on rows without NaN
    xf, tf = xt[torch.from_numpy(ok).cuda()].contiguous(), tt[torch.from_numpy(ok).cuda()].contiguous()
    m2 = SegmentationMetrics(C, 255, "cuda")
    m2.update(xf, tf, average_precision=False)
    ce = losses.cross_entropy(xf, tf, 255)
    stats = m2.stats.cpu().numpy()
    assert np.float32(stats[0] / stats[2]) == ce.cpu().numpy() and stats[0] / stats[2] == float(ce)
    assert stats[1] / stats[2] == O.precision_at_one(torch.max(xf, 1)[1].cpu().numpy(), tf.cpu().numpy())


def test_segmentation_metrics_on_reference_golden():
    """The reference's `lib/test.py::test` on the golden logits: hist and mIoU exactly; loss and score within 1e-6 relative; per-class AP
    equal to scikit-learn's on the library's own probabilities within 1e-12; mAP within 1e-3 (percentage units) of the reference's
    torch-softmax value -- near-ties may reorder under last-bit differences of the two softmaxes."""
    sk = pytest.importorskip("sklearn.metrics")
    from pointcontrast_b200.semseg import SegmentationMetrics
    z = np.load(GOLDEN)
    C = z["logits"].shape[1]
    m = SegmentationMetrics(C, 255, "cuda")
    off = np.r_[0, np.cumsum(z["sizes"])]
    sk_aps = []
    for a, b in zip(off[:-1], off[1:]):
        t = z["targets"][a:b]
        _, prob = m.update(torch.from_numpy(z["logits"][a:b]).cuda(), torch.from_numpy(t).cuda())
        p = prob.cpu().numpy().astype(np.float64)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sk_aps.append([sk.average_precision_score((t == c).astype(int), p[:, c]) for c in range(C)])
    r = m.result()
    loss_r, score_r, mAP_r, mIoU_r = z["result"]
    assert np.array_equal(r.hist, z["hist"]) and r.mIoU == mIoU_r
    assert abs(r.loss - loss_r) <= 1e-6 * abs(loss_r) and abs(r.score - score_r) <= 1e-6 * abs(score_r)
    assert np.all(np.abs(r.ap / 100 - np.mean(sk_aps, 0)) <= 1e-12)
    print(f"mAP {r.mAP!r} vs reference {mAP_r!r}: gap {abs(r.mAP - mAP_r):.3e}")
    assert abs(r.mAP - mAP_r) <= 1e-3


# ------------------------------------------------------------------------------------------------ semseg.test and the training loop

def _rooms(root, n=5, n_raw=20_000):
    from pointcontrast_b200 import synth
    (root / "splits").mkdir(exist_ok=True)
    names = []
    for k in range(n):
        xyz, rgb, lab = synth.synth_labelled_room(200 + k, n_raw, scale=0.8 + 0.1 * k)
        synth.write_ply(root / f"scene{k:04d}_00.ply", xyz, rgb, lab)
        names.append(f"scene{k:04d}_00.ply")
    for f in ("scannetv2_train.txt", "scannetv2_val.txt"):
        (root / "splits" / f).write_text("\n".join(names) + "\n")


def _config(root, **train):
    t = dict(stat_freq=1, save_freq=2, val_freq=2, resume=None, overwrite_weights=True)
    t.update(train)
    return refload.Cfg(
        data=dict(scannet_path=str(root), ignore_label=255, return_transformation=False),
        augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
        optimizer=dict(optimizer="SGD", lr=0.01, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=1, scheduler="PolyLR",
                       max_iter=4, poly_power=0.9),
        net=dict(model="Res16UNet34C", wrapper_type=None), misc=dict(seed=123), train=t,
        test=dict(test_stat_freq=1, save_prediction=False, test_original_pointcloud=False, evaluate_original_pointcloud=False))


def _val_loader(root, cfg):
    from pointcontrast_b200 import semseg_data as S
    return S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "val", shuffle=False, augment_data=False, batch_size=2,
                                    limit_numpoints=0, split_dir=str(root / "splits"), repeat=False)


def _net(seed=1):
    from pointcontrast_b200.model import load_model
    from tests.helpers import det_init
    mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
    net = load_model("Res16UNet34C")(3, 20, mcfg, D=3).cuda()
    det_init(net, seed)
    return net


def test_semseg_test_matches_oracle_batch_by_batch(tmp_path):
    from pointcontrast_b200 import me as ME, semseg
    _rooms(tmp_path)
    cfg = _config(tmp_path)
    loader = _val_loader(tmp_path, cfg)
    assert len(loader) == 3
    batches = list(loader)
    assert [int(c[:, 0].max()) + 1 for c, _, _ in batches] == [2, 2, 1]
    net = _net()
    got = semseg.test(net, loader, cfg)
    acc = O.Accumulator(20, 255)
    net.eval()
    with torch.no_grad():
        for coords, feats, target in batches:
            out = net(ME.SparseTensor(feats, coords).to("cuda")).F
            m = semseg.SegmentationMetrics(20, 255, "cuda")
            _, prob = m.update(out, target)
            acc.update(out.cpu().numpy(), target.cpu().numpy(), score=prob.cpu().numpy())
    want = acc.result()[0]
    assert abs(got[0] - want[0]) <= 1e-6 * abs(want[0])
    assert got[1] == want[1] and got[3] == want[3]
    assert abs(got[2] - want[2]) <= 1e-9
    bad = _config(tmp_path)
    bad["test"]["save_prediction"] = True
    with pytest.raises(NotImplementedError):
        semseg.test(net, loader, bad)


def _train_loader(root, cfg):
    from pointcontrast_b200 import semseg_data as S
    gen = torch.Generator(device="cuda"); gen.manual_seed(0)
    return S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "train", shuffle=True, augment_data=True, batch_size=2,
                                    limit_numpoints=0, split_dir=str(root / "splits"), draws=S.Draws("cuda", gen))


def test_train_checkpoints_validation_and_resume(tmp_path, monkeypatch):
    from pointcontrast_b200 import semseg
    _rooms(tmp_path)
    run = tmp_path / "run"; run.mkdir()
    monkeypatch.chdir(run)
    cfg = _config(tmp_path)
    val = _val_loader(tmp_path, cfg)
    tr = semseg.SegmentationTrainer(_net(), cfg)
    best, best_iter = tr.train(_train_loader(tmp_path, cfg), val)
    w = run / "weights"
    main = w / "checkpoint_NoneRes16UNet34C.pth"
    assert main.exists() and os.readlink(w / "weights.pth") in ("checkpoint_NoneRes16UNet34C.pth", "checkpoint_NoneRes16UNet34Cbest_val.pth")
    final = torch.load(main, map_location="cpu", weights_only=False)
    assert set(final) == {"iteration", "epoch", "arch", "state_dict", "optimizer", "best_val", "best_val_iter"}
    assert final["iteration"] == 4 and final["arch"] == "Res16UNet34C"
    # the final checkpoint precedes the final validation (`train.py:226-231`): it holds the best up to iteration 4 exclusive
    assert best_iter in (0, 2, 4) and best == tr.best_val and final["best_val"] <= best
    if best_iter:
        bv = torch.load(w / "checkpoint_NoneRes16UNet34Cbest_val.pth", map_location="cpu", weights_only=False)
        assert bv["best_val"] == best and bv["best_val_iter"] == best_iter == bv["iteration"]

    # the same run keeping every checkpoint (`_iter_{n}` names); record the uninterrupted run's state at iteration 2 as it is saved
    run2 = tmp_path / "run2"; run2.mkdir()
    monkeypatch.chdir(run2)
    cfg2 = _config(tmp_path, overwrite_weights=False)
    tr2 = semseg.SegmentationTrainer(_net(), cfg2)
    seen = {}
    save = semseg.checkpoint

    def spy(model, optimizer, epoch, iteration, *a, **k):
        if iteration == 2 and "lr" not in seen:
            seen.update(lr=tr2.scheduler.get_last_lr()[0], last_epoch=tr2.scheduler.last_epoch, mom=optimizer.flat_buf.clone(), epoch=epoch)
        save(model, optimizer, epoch, iteration, *a, **k)
    monkeypatch.setattr(semseg, "checkpoint", spy)
    tr2.train(_train_loader(tmp_path, cfg2), val)
    monkeypatch.setattr(semseg, "checkpoint", save)
    it2 = run2 / "weights" / "checkpoint_NoneRes16UNet34C_iter_2.pth"
    st2 = torch.load(it2, map_location="cpu", weights_only=False)
    assert st2["iteration"] == 2 and seen["last_epoch"] == 2
    assert abs(seen["lr"] - 0.01 * (1 - 2 / 5) ** 0.9) < 1e-12

    # resume a fresh trainer (other weights) from the iteration-2 checkpoint
    res = tmp_path / "resume"; res.mkdir()
    os.symlink(it2, res / "weights.pth")
    tr3 = semseg.SegmentationTrainer(_net(seed=5), _config(tmp_path, resume=str(res)))
    tr3.resume(str(res))
    assert tr3.curr_iter == 3 and tr3.epoch == seen["epoch"] == st2["epoch"]
    assert tr3.scheduler.last_epoch == 2 and tr3.scheduler.get_last_lr()[0] == seen["lr"] == tr3.optimizer.param_groups[0]["lr"]
    assert torch.equal(tr3.optimizer.flat_buf, seen["mom"]) and not tr3.optimizer._first
    assert tr3.best_val == st2["best_val"] and tr3.best_val_iter == st2["best_val_iter"]
    for k, v in st2["state_dict"].items():
        assert torch.equal(tr3.model.state_dict()[k].cpu(), v), k
    # and the loop itself resumes: two more steps to max_iter
    run3 = tmp_path / "run3"; run3.mkdir()
    monkeypatch.chdir(run3)
    tr4 = semseg.SegmentationTrainer(_net(seed=5), _config(tmp_path, resume=str(res)))
    tr4.train(_train_loader(tmp_path, tr4.config), val)
    assert torch.load(run3 / "weights" / "checkpoint_NoneRes16UNet34C.pth", map_location="cpu", weights_only=False)["iteration"] == 4
    assert tr4.curr_iter == 5
