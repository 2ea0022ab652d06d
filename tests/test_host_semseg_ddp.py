"""Data-parallel semantic-segmentation finetuning, the host side (CPU; gloo where a process group is needed): the training loader's
rank shards, the sharded evaluation pass, and the two-collective reduction of `SegmentationMetrics`."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Items:
    """A dataset whose item i is i (the loaders only index it)."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i


def _ids(items):
    return list(items)


@pytest.mark.parametrize("world", [2, 3])
def test_training_shards_are_disjoint_and_cover_each_epoch(world):
    """Three shuffled epochs; between draws each rank consumes a different amount of the global torch RNG (as augmentation and scene
    sizes make it do), yet the ranks' shards of every epoch are disjoint and together the whole dataset."""
    from pointcontrast_b200.semseg_data import VoxelizationLoader
    n, bs = 12, 2
    loaders = [VoxelizationLoader(_Items(n), bs, _ids, shuffle=True, rank=r, world=world, seed=123) for r in range(world)]
    assert all(len(l) == -(-n // world) // bs for l in loaders)
    per_epoch = n // world
    draws = [[] for _ in range(world)]
    for r, l in enumerate(loaders):
        torch.manual_seed(1000 + r)
        for _ in range(3 * per_epoch):
            torch.rand(1 + 7 * r)                       # a rank-specific amount of global RNG use between draws
            draws[r].append(next(l.sampler))
    perms = set()
    for e in range(3):
        shards = [set(d[e * per_epoch:(e + 1) * per_epoch]) for d in draws]
        assert all(len(s) == per_epoch for s in shards)
        assert set().union(*shards) == set(range(n)) and sum(map(len, shards)) == n
        perms.add(tuple(d[e * per_epoch] for d in draws))
    assert len(perms) > 1                               # shuffled: not the same order every epoch


def test_training_loader_world1_keeps_the_global_rng_order():
    from pointcontrast_b200.semseg_data import VoxelizationLoader
    torch.manual_seed(5)
    sampler = VoxelizationLoader(_Items(9), 3, _ids, shuffle=True).sampler
    got = [next(sampler) for _ in range(9)]
    torch.manual_seed(5)
    assert got == torch.randperm(9).tolist()
    with pytest.raises(ValueError):
        VoxelizationLoader(_Items(9), 3, _ids, shuffle=True, rank=0, world=2)        # no shared seed


@pytest.mark.parametrize("n,bs,world", [(7, 2, 2), (7, 2, 3), (5, 1, 2), (3, 2, 3), (2, 4, 2)])
@pytest.mark.parametrize("shuffle", [False, True])
def test_pass_shards_interleave_to_the_single_process_batches(n, bs, world, shuffle):
    """Rank r's batches are batches r, r + world, ... of one process's pass, item for item: short last batches and ranks without a
    batch included."""
    from pointcontrast_b200.semseg_data import VoxelizationPassLoader
    one = VoxelizationPassLoader(_Items(n), bs, _ids, shuffle=shuffle, seed=7)
    ranks = [VoxelizationPassLoader(_Items(n), bs, _ids, shuffle=shuffle, rank=r, world=world, seed=7) for r in range(world)]
    for _ in range(2):                                   # two passes: the shuffled order moves on identically everywhere
        want = [tuple(b) for b in one]
        shards = [[tuple(b) for b in l] for l in ranks]
        assert [len(s) for s in shards] == [len(l) for l in ranks] and sum(map(len, shards)) == len(want)
        got = [shards[b % world][b // world] for b in range(len(want))]
        assert got == want
        assert sorted(sum(want, ())) == list(range(n)) and len(want[-1]) == n - bs * (len(want) - 1)
    if (n + bs - 1) // bs < world:
        assert len(ranks[-1]) == 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


C = 4


def _fill(m, rank):
    """Per-rank values in every field, the fp64 ones with fractions so a bitwise integer sum of them is not their sum."""
    g = np.random.default_rng(rank)
    m.stats.copy_(torch.from_numpy(g.random(3) * 100 + 0.3))
    m.ap_sum.copy_(torch.from_numpy(g.random(C)))
    m.hist.copy_(torch.from_numpy(g.integers(0, 1000, C * C)))
    m.ap_cnt.copy_(torch.from_numpy(g.integers(0, 5, C)))


def _metrics_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from pointcontrast_b200.semseg import SegmentationMetrics
        from pointcontrast_b200.semseg_data import VoxelizationPassLoader, VoxelizationLoader
        m = SegmentationMetrics(C, 255, "cpu")
        _fill(m, rank)
        m.all_reduce()
        wrong = SegmentationMetrics(C, 255, "cpu")
        _fill(wrong, rank)
        dist.all_reduce(wrong._buf)                      # the whole buffer summed as int64
        l = VoxelizationLoader(_Items(8), 2, _ids, shuffle=True, seed=1)
        p = VoxelizationPassLoader(_Items(8), 2, _ids)
        torch.save({"buf": m._buf.clone(), "wrong": wrong._buf.clone(), "loader": (l.rank, l.world), "pass": (p.rank, p.world)},
                   os.path.join(out, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_metrics_all_reduce_sums_each_field_in_its_own_type(tmp_path):
    from pointcontrast_b200.semseg import SegmentationMetrics
    world = 2
    mp.spawn(_metrics_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    got = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    assert torch.equal(got[0]["buf"], got[1]["buf"])
    assert got[0]["loader"] == (0, 2) and got[1]["loader"] == (1, 2)                   # the training loader's shard: the process group's
    assert got[0]["pass"] == got[1]["pass"] == (0, 1)                                  # the pass loader: sharded only when asked
    parts = []
    for r in range(world):
        m = SegmentationMetrics(C, 255, "cpu")
        _fill(m, r)
        parts.append(m)
    red = SegmentationMetrics(C, 255, "cpu")
    red._buf.copy_(got[0]["buf"])
    assert torch.equal(red.stats, parts[0].stats + parts[1].stats)
    assert torch.equal(red.ap_sum, parts[0].ap_sum + parts[1].ap_sum)
    assert torch.equal(red.hist, parts[0].hist + parts[1].hist)
    assert torch.equal(red.ap_cnt, parts[0].ap_cnt + parts[1].ap_cnt)
    bad = SegmentationMetrics(C, 255, "cpu")
    bad._buf.copy_(got[0]["wrong"])
    assert torch.equal(bad.hist, red.hist)
    assert not torch.equal(bad.stats, red.stats)
