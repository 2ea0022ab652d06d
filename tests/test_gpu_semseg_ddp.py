"""Data-parallel semantic-segmentation finetuning (`downstream/semseg/lib/train.py` under DistributedDataParallel) with world size 2.
Two processes share ONE GPU over gloo (NCCL refuses two ranks on one device; gloo all-reduces CUDA tensors through the host); with two
devices visible the step check also runs over NCCL, one rank per device, which is the path a torchrun launch takes.

  * one `SegmentationTrainer.train_step` at iter_size 2: parameters, momentum and flat gradients bit-identical on both ranks and equal
    to one process that sums the two ranks' accumulated gradients and applies the SGD kernel with grad_scale 1/2; per-rank BatchNorm
    statistics; the flat gradient reduced in three all-reduces, the two chunks launched during the LAST sub-batch's backward sweep;
  * `SegmentationTrainer.train` with checkpoints and validation inside the run, and its resumption;
  * `semseg.test` on a sharded pass loader returns the single-process result;
  * without a process group the trainer issues no collective, installs no hook, and steps as before.
"""
import os
import socket

import numpy as np
import pytest
import torch

from tests import refload

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _spawn(fn, *args, backend="gloo"):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(fn, _free_port(), backend) + args, nprocs=2, join=True)


def _worker(rank, fn, port, backend, *args):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=2)
    try:
        fn(rank, *args)
    finally:
        dist.destroy_process_group()


def _net(seed=1):
    from pointcontrast_b200.model import load_model
    from tests.helpers import det_init
    mcfg = refload.default_config(); mcfg["net"]["normalize_feature"] = False
    net = load_model("Res16UNet34C")(3, 20, mcfg, D=3).cuda()
    det_init(net, seed)
    return net


def _step_cfg():
    return refload.Cfg(optimizer=dict(optimizer="SGD", lr=0.01, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=2,
                                      scheduler="PolyLR", max_iter=100, poly_power=0.9), data=dict(ignore_label=255))


def _sub_batches(rank):
    """Rank `rank`'s two sub-batches: synthetic rooms with random labels (15 % ignored)."""
    from pointcontrast_b200 import synth
    rng = np.random.default_rng(rank)
    subs = []
    for k in range(2):
        sc = synth.synth_scene(10 * rank + k, scale=0.25, voxel=0.05, n_raw=40_000)
        t = rng.integers(0, 20, len(sc["coords"])); t[rng.random(len(t)) < 0.15] = 255
        subs.append((torch.from_numpy(sc["coords"]), torch.from_numpy(sc["feats"]), torch.from_numpy(t)))
    return subs


def _bn(model):
    return {k: v.cpu() for k, v in model.state_dict().items() if "running" in k}


def _accumulate(tr, subs):
    """train_step's gradient accumulation without the step: the flat gradient of the sub-batches on the current weights."""
    from pointcontrast_b200 import losses, me as ME
    tr.model.train()
    tr.optimizer.zero_grad()
    for coords, feats, target in subs:
        out = tr.model(ME.SparseTensor(feats, coords).to(tr.device)).F
        (losses.cross_entropy(out, target.to(tr.device), 255) / len(subs)).backward()
    torch.cuda.synchronize()
    return tr.optimizer.flat_grad.clone()


# ------------------------------------------------------------------------------------------------ one step

def _step_rank(rank, out_dir):
    import torch.distributed as dist
    from pointcontrast_b200 import losses, semseg
    tr = semseg.SegmentationTrainer(_net(), _step_cfg())
    assert tr.world == 2 and tr.optimizer.grad_scale == 0.5 and len(tr.grads.chunk_after) == 2
    # which sub-batch's backward (or the tail before the step) issues each all-reduce
    phase, issued = [0], []
    ce, all_reduce, finish = losses.cross_entropy, dist.all_reduce, tr.grads.finish

    def counting_ce(*a, **k):
        phase[0] += 1
        return ce(*a, **k)

    def spy_all_reduce(t, *a, **k):
        issued.append((phase[0], t.numel()))
        return all_reduce(t, *a, **k)

    def spy_finish():
        phase[0] = "tail"
        finish()

    losses.cross_entropy, dist.all_reduce, tr.grads.finish = counting_ce, spy_all_reduce, spy_finish
    try:
        tr.grads.timing = {}
        tr.train_step(_sub_batches(rank), shift_coords=False)
        torch.cuda.synchronize()
    finally:
        losses.cross_entropy, dist.all_reduce = ce, all_reduce
    o = tr.optimizer
    torch.save({"param": o.flat_param.cpu(), "buf": o.flat_buf.cpu(), "grad": o.flat_grad.cpu(), "bn": _bn(tr.model), "issued": issued,
                "events": len(tr.grads.timing["allreduce"])}, os.path.join(out_dir, f"rank{rank}.pt"))


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_two_rank_step_equals_sum_of_accumulated_gradients(tmp_path, backend):
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one device per rank")
    _spawn(_step_rank, str(tmp_path), backend=backend)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt") for r in (0, 1))
    for k in ("param", "buf", "grad"):
        assert torch.equal(r0[k], r1[k]), k
    n = r0["grad"].numel()
    for r in (r0, r1):
        assert r["events"] == 3
        assert [p for p, _ in r["issued"]] == [2, 2, "tail"], r["issued"]         # nothing during the first sub-batch's backward
        assert sum(m for _, m in r["issued"]) == n                                 # every element reduced exactly once
    assert any(not torch.equal(r0["bn"][k], r1["bn"][k]) for k in r0["bn"])      # per-rank BatchNorm statistics
    # one process: each rank's accumulated gradient on the same initial weights, summed, one SGD step with grad_scale 1/2
    from pointcontrast_b200 import semseg
    from tests.helpers import rel_err
    grads = []
    for rank in (0, 1):
        tr = semseg.SegmentationTrainer(_net(), _step_cfg())
        grads.append(_accumulate(tr, _sub_batches(rank)))
        bn = _bn(tr.model)
        for k in bn:
            assert torch.equal((r0, r1)[rank]["bn"][k], bn[k]), (rank, k)        # the forward pass is deterministic
    tr = semseg.SegmentationTrainer(_net(), _step_cfg())
    tr.optimizer.flat_grad.copy_(grads[0] + grads[1])
    tr.optimizer.grad_scale = 0.5
    tr.optimizer.step()
    torch.cuda.synchronize()
    assert rel_err(r0["grad"], grads[0] + grads[1]) < 1e-5
    assert rel_err(r0["param"], tr.optimizer.flat_param) < 1e-5 and rel_err(r0["buf"], tr.optimizer.flat_buf) < 1e-5


# ------------------------------------------------------------------------------------------------ the training loop

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
    max_iter = train.pop("max_iter", 4)
    t.update(train)
    return refload.Cfg(
        data=dict(scannet_path=str(root), ignore_label=255, return_transformation=False),
        augmentation=dict(data_aug_color_trans_ratio=0.10, data_aug_color_jitter_std=0.05),
        optimizer=dict(optimizer="SGD", lr=0.01, sgd_momentum=0.9, sgd_dampening=0.1, weight_decay=1e-4, iter_size=2, scheduler="PolyLR",
                       max_iter=max_iter, poly_power=0.9),
        net=dict(model="Res16UNet34C", wrapper_type=None), misc=dict(seed=123), train=t,
        test=dict(test_stat_freq=1, save_prediction=False, test_original_pointcloud=False, evaluate_original_pointcloud=False))


def _loaders(root, cfg, rank, val_batch=2, shuffle=False):
    from pointcontrast_b200 import semseg_data as S
    gen = torch.Generator(device="cuda"); gen.manual_seed(0)
    train = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "train", shuffle=True, augment_data=True, batch_size=1,
                                     limit_numpoints=0, split_dir=str(root / "splits"), draws=S.Draws("cuda", gen), iter_size=2)
    val = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "val", shuffle=shuffle, augment_data=False, batch_size=val_batch,
                                   limit_numpoints=0, split_dir=str(root / "splits"), repeat=False, rank=rank, world=2)
    return train, val


def _train_rank(rank, root):
    import pathlib
    import torch.distributed as dist
    from pointcontrast_b200 import semseg
    root = pathlib.Path(root)
    run = root / f"run{rank}"; run.mkdir()
    os.chdir(run)
    cfg = _config(root)
    tr = semseg.SegmentationTrainer(_net(seed=1 + rank), cfg)           # other weights on rank 1: construction broadcasts rank 0's
    start = tr.optimizer.flat_param.cpu()
    train, val = _loaders(root, cfg, rank)
    assert train.world == 2 and train.rank == rank and val.world == 2 and len(val) == (2, 1)[rank]
    best = tr.train(train, val)
    dist.barrier()                                                     # rank 0's last checkpoint is written
    # resume rank 0's checkpoints with other weights on both ranks, two more steps
    res = root / f"resume{rank}"; res.mkdir()
    os.chdir(res)
    tr2 = semseg.SegmentationTrainer(_net(seed=7 + rank), _config(root, resume=str(root / "run0" / "weights"), max_iter=6))
    tr2.resume(str(root / "run0" / "weights"))
    resumed = (tr2.curr_iter, tr2.optimizer.flat_param.cpu(), tr2.optimizer.flat_buf.cpu())
    tr2.train(*_loaders(root, tr2.config, rank))
    torch.save({"start": start, "best": best, "param": tr.optimizer.flat_param.cpu(), "resumed": resumed, "curr_iter": tr2.curr_iter,
                "param2": tr2.optimizer.flat_param.cpu(), "buf2": tr2.optimizer.flat_buf.cpu()}, root / f"train{rank}.pt")


def test_two_rank_train_checkpoints_validation_and_resume(tmp_path):
    _rooms(tmp_path)
    _spawn(_train_rank, str(tmp_path))
    r0, r1 = (torch.load(tmp_path / f"train{r}.pt", weights_only=False) for r in (0, 1))
    assert torch.equal(r0["start"], r1["start"])
    assert (tmp_path / "run0" / "weights" / "checkpoint_NoneRes16UNet34C.pth").exists()
    assert not (tmp_path / "run1" / "weights").exists() and not (tmp_path / "resume1" / "weights").exists()
    assert r0["best"] == r1["best"] and r0["best"][1] in (0, 2, 4)
    assert torch.equal(r0["param"], r1["param"])
    final = torch.load(tmp_path / "run0" / "weights" / "checkpoint_NoneRes16UNet34C.pth", map_location="cpu", weights_only=False)
    assert final["iteration"] == 4
    for r in (r0, r1):
        it, p, b = r["resumed"]
        assert it == 5 and torch.equal(p, r0["param"]) and torch.equal(b, r0["resumed"][2])
        assert r["curr_iter"] == 7
    assert torch.equal(r0["param2"], r1["param2"]) and torch.equal(r0["buf2"], r1["buf2"])
    assert torch.load(tmp_path / "resume0" / "weights" / "checkpoint_NoneRes16UNet34C.pth", map_location="cpu",
                      weights_only=False)["iteration"] == 6


# ------------------------------------------------------------------------------------------------ sharded evaluation

CASES = [(1, False), (1, True), (2, False), (2, True)]


def _capture_results(monkeypatch):
    """The SegmentationResults `test` computes, in order."""
    from pointcontrast_b200 import semseg
    got, result = [], semseg.SegmentationMetrics.result

    def spy(self):
        r = result(self)
        got.append(r)
        return r
    monkeypatch.setattr(semseg.SegmentationMetrics, "result", spy)
    return got


def _test_rank(rank, root):
    import pathlib
    from pointcontrast_b200 import semseg
    root = pathlib.Path(root)
    cfg = _config(root)
    got = _capture_results(pytest.MonkeyPatch())
    out = []
    for bs, shuffle in CASES:
        _, val = _loaders(root, cfg, rank, val_batch=bs, shuffle=shuffle)
        t = semseg.test(_net(), val, cfg)
        out.append((t, got[-1].hist, got[-1].ap))
    torch.save(out, root / f"test{rank}.pt")


def test_sharded_test_equals_single_process(tmp_path, monkeypatch):
    from pointcontrast_b200 import semseg, semseg_data as S
    _rooms(tmp_path)
    _spawn(_test_rank, str(tmp_path))
    ranks = [torch.load(tmp_path / f"test{r}.pt", weights_only=False) for r in (0, 1)]
    cfg = _config(tmp_path)
    got = _capture_results(monkeypatch)
    for i, (bs, shuffle) in enumerate(CASES):
        ld = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "val", shuffle=shuffle, augment_data=False, batch_size=bs,
                                      limit_numpoints=0, split_dir=str(tmp_path / "splits"), repeat=False)
        one = S.VoxelizationPassLoader(ld.dataset, bs, ld.collate_fn, shuffle=shuffle, normalize_color=True, seed=cfg.misc.seed)
        want = semseg.test(_net(), one, cfg)
        hist = got[-1].hist
        for r in ranks:
            t, h, ap = r[i]
            assert np.array_equal(h, hist), (bs, shuffle)
            for a, b in zip(t, want):
                assert abs(a - b) <= 1e-12 * abs(b), (bs, shuffle, t, want)
    with pytest.raises(ValueError, match="save_prediction"):
        bad = _config(tmp_path)
        bad["test"]["save_prediction"] = True
        ld = S.initialize_data_loader(S.ScannetVoxelization2cmDataset, cfg, "val", shuffle=False, augment_data=False, batch_size=1,
                                      limit_numpoints=0, split_dir=str(tmp_path / "splits"), repeat=False, rank=0, world=2)
        semseg.test(_net(), ld, bad)


# ------------------------------------------------------------------------------------------------ world 1

def test_world1_issues_no_collective_and_steps_as_before(monkeypatch):
    import torch.distributed as dist
    from pointcontrast_b200 import semseg
    assert not (dist.is_available() and dist.is_initialized())

    def refuse(*a, **k):
        raise AssertionError("a collective at world 1")
    for name in ("all_reduce", "broadcast"):
        monkeypatch.setattr(dist, name, refuse)
    subs = _sub_batches(0)
    tr = semseg.SegmentationTrainer(_net(), _step_cfg())
    assert tr.world == 1 and tr.grads.comm is None and not tr.grads.chunk_after and "_fused_after_unit" not in tr.model.__dict__
    assert tr.optimizer.grad_scale == 1.0
    tr.train_step(subs, shift_coords=False)
    torch.cuda.synchronize()
    # the step as it is without the data-parallel layer: accumulate, then the SGD kernel
    want = []
    for _ in range(2):
        ref = semseg.SegmentationTrainer(_net(), _step_cfg())
        _accumulate(ref, subs)
        ref.optimizer.step()
        torch.cuda.synchronize()
        want.append(ref.optimizer.flat_param.clone())
    if torch.equal(want[0], want[1]):                    # a deterministic backward: bit for bit
        assert torch.equal(tr.optimizer.flat_param, want[0])
    else:
        from tests.helpers import rel_err
        assert rel_err(tr.optimizer.flat_param, want[0]) < 1e-6
