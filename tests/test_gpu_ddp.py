"""Data-parallel step of the trainer (`pretrain/pointcontrast/lib/ddp_trainer.py:96-102`: DistributedDataParallel) with
world_size 2.  Two processes share ONE GPU over the gloo backend (NCCL refuses two ranks on one device; gloo all-reduces CUDA
tensors through the host), so this runs on the single-GPU test box; with two devices visible the same test also runs over NCCL,
one rank per device, which is the path `bench.py --gpus N` takes.

Checked after one `train_step` on different per-rank batches:
  * parameters (and SGD momentum buffers) are bit-identical on the two ranks;
  * they equal (1e-5; the loss's gather backward uses atomics, so not bit for bit) ONE process that computes rank 0's and
    rank 1's gradients one after the other, adds them and applies the SGD kernel with grad_scale = 1/2;
  * BatchNorm running statistics stay per rank (`broadcast_buffers=False`): they differ between the ranks and each equals
    its single-process replay;
  * the chunked, backward-overlapped all-reduce reduced every element exactly once (three chunks, covering the flat buffer).
"""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu

SCALE = 0.12


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _make_trainer(rank, world):
    from pointcontrast_b200.config import default_config
    from pointcontrast_b200.data import SyntheticPairLoader
    from pointcontrast_b200.trainer import get_trainer
    cfg = default_config([f"trainer.batch_size={world}", f"misc.num_gpus={world}", "misc.nceT=0.4"])
    loader = SyntheticPairLoader(1, scale=SCALE, num_batches=1, rank=rank, pin=False)
    torch.manual_seed(0)                      # same initial weights on every rank / in the replay
    tr = get_trainer("PointNCELossTrainer")(cfg, loader)
    return tr, loader.batches[0]


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        tr, batch = _make_trainer(rank, world)
        assert tr.world == 2 and tr.optimizer.grad_scale == 0.5
        assert len(tr._chunk_after) == 2, "the backward-overlapped chunking did not engage"
        tr.timing = {}
        tr.train_step(batch)
        torch.cuda.synchronize()
        n_chunks = len(tr.timing["allreduce"])
        tr.timing = None
        torch.save({"param": tr.optimizer.flat_param.cpu(), "buf": tr.optimizer.flat_buf.cpu(), "grad": tr.optimizer.flat_grad.cpu(),
                    "bn": {k: v.cpu() for k, v in tr.model.state_dict().items() if "running" in k}, "chunks": n_chunks},
                   os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_two_rank_step_equals_mean_of_single_rank_gradients(tmp_path, backend):
    """gloo: both ranks on device 0 (the single-GPU test box); nccl: one rank per device (needs two GPUs)."""
    import torch.multiprocessing as mp
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs one device per rank")
    port = _free_port()
    mp.spawn(_worker, args=(2, port, str(tmp_path), backend), nprocs=2, join=True)
    r0 = torch.load(tmp_path / "rank0.pt")
    r1 = torch.load(tmp_path / "rank1.pt")
    assert r0["chunks"] == 3 and r1["chunks"] == 3
    assert torch.equal(r0["param"], r1["param"]) and torch.equal(r0["buf"], r1["buf"]) and torch.equal(r0["grad"], r1["grad"])
    assert any(not torch.equal(r0["bn"][k], r1["bn"][k]) for k in r0["bn"])          # per-rank BatchNorm statistics
    # single-process replay: gradients of rank 0's batch, then of rank 1's batch, summed, one SGD step with grad_scale 1/2
    grads, bns = [], []
    for rank in (0, 1):
        tr, batch = _make_trainer(rank, 1)
        tr.generator.manual_seed(1234 + rank)                 # the positive draws of that rank
        tr.optimizer.zero_grad()
        F0, F1 = tr._forward_views(batch)
        from pointcontrast_b200 import losses
        pos = batch["correspondences"].to(tr.device)
        q, k = losses.select_positives(pos, tr.npos, tr.generator)
        losses.point_nce_loss(F0, F1, q, k, tr.T).backward()
        grads.append(tr.optimizer.flat_grad.clone())
        bns.append({k_: v.cpu() for k_, v in tr.model.state_dict().items() if "running" in k_})
    tr.optimizer.flat_grad.copy_(grads[0] + grads[1])
    tr.optimizer.flat_param.copy_(_make_trainer(0, 1)[0].optimizer.flat_param)      # initial weights (the loop above did not step)
    tr.optimizer.grad_scale = 0.5
    tr.optimizer.step()
    torch.cuda.synchronize()
    from tests.helpers import rel_err
    assert rel_err(r0["grad"], grads[0] + grads[1]) < 1e-5
    assert rel_err(r0["param"], tr.optimizer.flat_param) < 1e-6
    for rank, r in ((0, r0), (1, r1)):
        for k in r["bn"]:
            assert torch.equal(r["bn"][k], bns[rank][k]), (rank, k)        # forward pass: deterministic
