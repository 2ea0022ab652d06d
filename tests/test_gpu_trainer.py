"""Trainer entry (pointcontrast_b200/trainer.py, mirror of pretrain/pointcontrast/lib/ddp_trainer.py) on the GPU:
loss curve against the CPU oracle under identical data / positive draws / SGD, and checkpoint save + resume."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import loss_cpu
from oracle import me_cpu as OR
from tests import refload
from tests.helpers import det_init, model_backend

pytestmark = pytest.mark.gpu


def test_loss_curve_matches_cpu_oracle():
    """6 SGD steps (lr 0.1, momentum 0.8, wd 1e-4, PointInfoNCE T=0.4) on two small scene pairs: the GPU path (fused
    executor + FlatSGD) and the fp32 CPU oracle (torch.optim.SGD) see the same batches and the same positive draws."""
    from pointcontrast_b200 import losses, me, optim, synth
    from pointcontrast_b200.model import load_model
    batches = [synth.collate_pairs([synth.synth_pair(20 + 2 * s, scale=0.12), synth.synth_pair(21 + 2 * s, scale=0.12)]) for s in range(2)]
    cfg = refload.default_config()
    net = load_model("Res16UNet34C")(3, 32, cfg, D=3)
    det_init(net, 7)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    net = net.cuda().train()
    opt = optim.FlatSGD(net.parameters(), lr=0.1, momentum=0.8, weight_decay=1e-4)
    with model_backend(OR) as mod:
        onet = mod.Res16UNet34C(3, 32, cfg, D=3)
        onet.load_state_dict(state)
        onet.train()
        oopt = torch.optim.SGD(onet.parameters(), lr=0.1, momentum=0.8, weight_decay=1e-4)
        rng = np.random.default_rng(3)
        curve, ocurve = [], []
        for step in range(6):
            b = batches[step % 2]
            pairs = b["correspondences"]
            nq = len(np.unique(pairs[:, 0]))
            q, k = loss_cpu.select_positives(pairs, rng.random(nq).astype(np.float32), 4096,
                                             rng.choice(nq, 4096, replace=False) if nq > 4096 else None)
            opt.zero_grad()
            F = [net(me.SparseTensor(torch.from_numpy(b[f"sinput{v}_F"]), coords=torch.from_numpy(b[f"sinput{v}_C"])).to("cuda")).F for v in "01"]
            loss = losses.point_nce_loss(F[0], F[1], q.cuda(), k.cuda(), 0.4)
            loss.backward(); opt.step()
            oopt.zero_grad()
            Fo = [onet(OR.SparseTensor(torch.from_numpy(b[f"sinput{v}_F"]), coords=torch.from_numpy(b[f"sinput{v}_C"]))).F for v in "01"]
            lo = loss_cpu.point_nce_loss(Fo[0], Fo[1], q, k, 0.4)
            lo.backward(); oopt.step()
            curve.append(float(loss.detach())); ocurve.append(float(lo.detach()))
    rel = [abs(a - b) / abs(b) for a, b in zip(curve, ocurve)]
    if os.environ.get("PCB_REPORT_DIR"):
        json.dump({"gpu": curve, "cpu_oracle_fp32": ocurve, "rel": rel}, open(os.path.join(os.environ["PCB_REPORT_DIR"], "loss_curve.json"), "w"), indent=1)
    assert rel[0] < 1e-3, (curve, ocurve)              # same weights: the 1e-3 loss bar
    assert max(rel) < 1e-2, (curve, ocurve)            # after 5 updates through an ill-conditioned backward
    assert ocurve[-1] < ocurve[0] and curve[-1] < curve[0]


def test_loss_curve_100_steps_against_fp64_and_fp32_oracles():
    """100 SGD steps (the reference's optimiser settings: lr 0.1, momentum 0.8, wd 1e-4, ExponentialLR 0.99 applied every step here,
    PointInfoNCE T = 0.4) on two small scene-pair batches.  The GPU path replays exactly the steps of the committed golden curves
    (tests/golden/loss_curve_100.npz, made by tests/golden/make_loss_curve.py on the CPU oracle in fp64 and in fp32: same batches,
    same deterministic weights, same positive draws).  Training from scratch at this learning rate is chaotic: a single ReLU entry
    whose pre-activation is zero to within rounding (tests/test_gpu_model.py, pinned-decision test) changes the step-0 gradient by
    ~5e-3 and the trajectories separate step by step (the fp32 CPU oracle against fp64: 3e-8 at step 0, 1e-5 at step 2, 6e-3 at its
    worst, back to 2e-4 at the end).  Stated tolerance on |gpu - fp64| / fp64:
        steps 0..2 (before the amplification)   <= 1e-3
        every step                              <= 0.1        (the loss falls fastest on steps 5..15)
        mean of the last 10 steps               <= 2e-2
    and both curves train (last loss < 0.8 x first)."""
    from pointcontrast_b200 import losses, optim
    from pointcontrast_b200.model import load_model
    from tests.golden import make_loss_curve as G
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "loss_curve_100.npz"))
    assert int(gold["steps"]) == G.STEPS and tuple(gold["seeds"]) == G.SEEDS and float(gold["scale"]) == G.SCALE
    c64, c32 = gold["oracle_fp64"], gold["oracle_fp32"]
    batches, draws = G.setup()
    net = load_model("Res16UNet34C")(3, 32, refload.default_config(), D=3)
    det_init(net, G.INIT_SEED)
    net = net.cuda().train()
    opt = optim.FlatSGD(net.parameters(), lr=0.1, momentum=0.8, weight_decay=1e-4)
    sch = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    dev = [{k: torch.from_numpy(b[k]).cuda() for k in ("sinput0_F", "sinput0_C", "sinput1_F", "sinput1_C")} for b in batches]
    gpu = []
    for step in range(G.STEPS):
        b = dev[step % 2]
        q, k = draws[step]
        opt.zero_grad()
        F0, F1 = net.forward_pair(b["sinput0_F"], b["sinput0_C"], b["sinput1_F"], b["sinput1_C"], torch.device("cuda"))
        loss = losses.point_nce_loss(F0, F1, q.cuda(), k.cuda(), 0.4)
        loss.backward(); opt.step(); sch.step()
        gpu.append(loss.detach())
    gpu = torch.stack(gpu).cpu().numpy().astype(np.float64)
    d_gpu = np.abs(gpu - c64) / c64
    d_f32 = np.abs(c32 - c64) / c64
    if os.environ.get("PCB_REPORT_DIR"):
        json.dump({"gpu": gpu.tolist(), "oracle_fp64": c64.tolist(), "oracle_fp32": c32.tolist(), "gpu_vs_fp64": d_gpu.tolist(),
                   "fp32_vs_fp64": d_f32.tolist()}, open(os.path.join(os.environ["PCB_REPORT_DIR"], "loss_curve_100.json"), "w"), indent=1)
    assert c64[-1] < 0.8 * c64[0] and gpu[-1] < 0.8 * gpu[0]                        # the curves train
    assert (d_gpu[:3] <= 1e-3).all(), d_gpu[:3]
    assert d_gpu.max() <= 0.1, (int(np.argmax(d_gpu)), float(d_gpu.max()), float(d_f32.max()))
    assert abs(gpu[-10:].mean() - c64[-10:].mean()) / c64[-10:].mean() <= 2e-2


def test_trainers_step_and_checkpoint_roundtrip(tmp_path, monkeypatch):
    from pointcontrast_b200.config import default_config
    from pointcontrast_b200.data import SyntheticPairLoader
    from pointcontrast_b200.trainer import get_trainer
    monkeypatch.chdir(tmp_path)
    cfg = default_config(["trainer.batch_size=1", "misc.nceT=0.4", "opt.max_iter=2", "trainer.lr_update_freq=2", "trainer.stat_freq=1"])
    loader = SyntheticPairLoader(1, scale=0.12, num_batches=2, pin=True)
    torch.manual_seed(0)
    tr = get_trainer("PointNCELossTrainer")(cfg, loader)
    tr.train()                                        # 2 iterations; checkpoints at iter 1 and 2 (`ddp_trainer.py:258-263`)
    assert tr.curr_iter == 2 and os.path.islink("weights/weights.pth")
    state = torch.load("weights/weights.pth", map_location="cpu", weights_only=False)
    assert set(state) == {"curr_iter", "state_dict", "optimizer", "scheduler", "config"} and state["curr_iter"] == 2
    assert "conv0p1s1.kernel" in state["state_dict"] and "bn0.bn.running_mean" in state["state_dict"]
    assert len(state["optimizer"]["state"]) == len(list(tr.model.parameters()))
    tr2 = get_trainer("PointNCELossTrainer")(cfg, loader)     # resumes from weights/weights.pth in the cwd
    assert tr2.curr_iter == 2
    for (n, a), (_, b) in zip(tr.model.state_dict().items(), tr2.model.state_dict().items()):
        assert torch.equal(a.cpu(), b.cpu()), n
    assert torch.equal(tr.optimizer.flat_buf.cpu(), tr2.optimizer.flat_buf.cpu())
    l2 = tr2._train_iter(iter(loader), None)
    assert np.isfinite(l2)
    # the hardest-contrastive trainer (`ddp_trainer.py:171-326`) runs and returns the three scalars
    th = get_trainer("HardestContrastiveLossTrainer")(default_config(["trainer.batch_size=1"]), loader)
    out = th._train_iter(iter(loader), None)
    assert len(out) == 3 and all(np.isfinite(v) for v in out) and abs(out[0] - (out[1] + out[2])) < 1e-4


def test_pipelined_iterations_equal_one_at_a_time(tmp_path, monkeypatch):
    """`Trainer.iter_losses(it, n)` (iteration i+1 enqueued before the loss of iteration i is read back; what `train()` runs between two
    LR / checkpoint boundaries) returns the losses of n `_train_iter` calls on a twin trainer, and leaves the same parameters."""
    from pointcontrast_b200.config import default_config
    from pointcontrast_b200.data import SyntheticPairLoader
    from pointcontrast_b200.trainer import get_trainer
    monkeypatch.chdir(tmp_path)
    cfg = default_config(["trainer.batch_size=1", "misc.nceT=0.4"])
    loader = SyntheticPairLoader(1, scale=0.12, num_batches=2, pin=True)
    outs = []
    for mode in ("single", "pipelined"):
        torch.manual_seed(0)
        tr = get_trainer("PointNCELossTrainer")(cfg, loader)
        it = iter(loader)
        ls = [tr._train_iter(it, None) for _ in range(4)] if mode == "single" else list(tr.iter_losses(it, 4))
        torch.cuda.synchronize()
        outs.append((ls, tr.optimizer.flat_param.clone()))
    (l_a, p_a), (l_b, p_b) = outs
    assert len(l_a) == len(l_b) == 4 and all(isinstance(v, float) for v in l_b)
    assert max(abs(a - b) / abs(a) for a, b in zip(l_a, l_b)) < 1e-5, (l_a, l_b)      # the loss's gather backward uses atomics: not bit for bit
    assert float((p_a - p_b).norm() / p_a.norm()) < 1e-5
