"""ScanNet frame-pair data path (SURVEY.md 8f-2 / 8f-3): the on-disk formats of the reference's preprocessing --
`<scene>/pcd/<frame>.npz` holding `pcd` = world-frame points [N,3] (`pretrain/data_preprocess/scannet_pair/point_cloud_extractor.py:80`)
and the pair list `overlap-30-full.txt` with lines `<file0> <file1> <overlap>` (`generate_list.py:20-28`; this repository writes it
with `pair_list.compute_full_overlapping` + `pair_list.generate_list`, or `python -m pointcontrast_b200.pair_list`) -- and a mirror of
`ScanNetMatchPairDataset` / `default_collate_pair_fn` / the infinite samplers (`lib/ddp_data_loaders.py:52-265`,
`lib/data_sampler.py:13-70`) whose per-sample work (voxelisation, correspondence search) runs on the GPU (`voxel.make_pair`)
instead of `ME.utils.sparse_quantize` + one open3d KD-tree query per point on CPU workers.

    ds = ScanNetMatchPairDataset("train", config=config, device="cuda:0")
    loader = PairLoader(ds, batch_size=4, rank=rank, world=world)      # yields the batch dict `Trainer._train_iter` consumes
"""
import math
import os
import random

import numpy as np
import torch

from . import voxel


def read_pair_list(path):
    """`generate_list.py:20-28` output: one `<file0> <file1> [overlap]` per line -> [(file0, file1), ...] (`ddp_data_loaders.py:176-181`)."""
    pairs = []
    with open(path) as f:
        for line in f:
            parts = line.strip().split()
            if len(parts) >= 2:
                pairs.append((parts[0], parts[1]))
    return pairs


def load_frame(path):
    """`np.load(file)["pcd"]` (`ddp_data_loaders.py:199-202`): float [N,3]."""
    return np.load(path)["pcd"]


def rotation_about(axis, theta):
    """`M(axis, theta)` = expm(cross(I, axis/|axis| * theta)) (`ddp_data_loaders.py:114-116`), by Rodrigues' formula."""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a) * theta
    th = np.linalg.norm(a)
    if th < 1e-12:
        return np.eye(3)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]) / th
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def sample_random_trans(pcd, randg, rotation_range=360):
    """`ddp_data_loaders.py:137-142`: centre on the mean, then a random rotation (same draws from `randg`)."""
    T = np.eye(4)
    R = rotation_about(randg.rand(3) - 0.5, rotation_range * np.pi / 180.0 * (randg.rand(1)[0] - 0.5))
    T[:3, :3] = R
    T[:3, 3] = R.dot(-np.mean(pcd, axis=0))
    return T


class Jitter:
    """`lib/transforms.py:21-30`."""

    def __init__(self, mu=0, sigma=0.01):
        self.mu, self.sigma = mu, sigma

    def __call__(self, coords, feats):
        if random.random() < 0.95:
            feats = feats + np.random.normal(self.mu, self.sigma, feats.shape).astype(feats.dtype)
        return coords, feats


class ScanNetMatchPairDataset:
    """`ddp_data_loaders.py:144-265`.  `__getitem__` returns the same 8-tuple (xyz0, xyz1, coords0, coords1, feats0, feats1, matches,
    trans) as numpy arrays; the voxelisation and the radius matching in between run on `device`."""

    def __init__(self, phase, transform=None, random_rotation=True, random_scale=True, manual_seed=False, config=None, device="cuda"):
        if phase != "train":
            raise NotImplementedError
        self.phase = phase
        self.transform = transform
        self.voxel_size = config.data.voxel_size
        self.matching_search_voxel_size = config.data.voxel_size * config.trainer.positive_pair_search_voxel_size_multiplier
        self.random_scale, self.random_rotation = random_scale, random_rotation
        self.min_scale, self.max_scale = config.trainer.min_scale, config.trainer.max_scale
        self.rotation_range = config.trainer.rotation_range
        self.randg = np.random.RandomState()
        if manual_seed:
            self.reset_seed()
        self.root = config.data.dataset_root_dir
        self.files = read_pair_list(os.path.join(self.root, config.data.scannet_match_dir))
        self.device = torch.device(device)

    def reset_seed(self, seed=0):
        self.randg.seed(seed)

    def __len__(self):
        return len(self.files)

    def __getitem__(self, idx):
        xyz0 = load_frame(os.path.join(self.root, self.files[idx][0]))
        xyz1 = load_frame(os.path.join(self.root, self.files[idx][1]))
        search = self.matching_search_voxel_size
        if self.random_scale and random.random() < 0.95:
            scale = self.min_scale + (self.max_scale - self.min_scale) * random.random()
            search *= scale
            xyz0, xyz1 = scale * xyz0, scale * xyz1
        if self.random_rotation:
            T0 = sample_random_trans(xyz0, self.randg, self.rotation_range)
            T1 = sample_random_trans(xyz1, self.randg, self.rotation_range)
            trans = T1 @ np.linalg.inv(T0)
            xyz0 = xyz0 @ T0[:3, :3].T + T0[:3, 3]
            xyz1 = xyz1 @ T1[:3, :3].T + T1[:3, 3]
        else:
            trans = np.identity(4)
        # voxelisation + matching on the GPU (`:228-245`): one point per voxel, matches within `search` after moving view 0 by `trans`
        p0 = torch.from_numpy(np.ascontiguousarray(xyz0, dtype=np.float32)).to(self.device)
        p1 = torch.from_numpy(np.ascontiguousarray(xyz1, dtype=np.float32)).to(self.device)
        out = voxel.make_pair(p0, p1, trans, self.voxel_size, search / self.voxel_size)
        xyz0, xyz1 = out["xyz0"].cpu().numpy(), out["xyz1"].cpu().numpy()
        coords0, coords1 = out["coords0"].cpu().numpy(), out["coords1"].cpu().numpy()      # == floor(xyz / voxel_size) (`:258-259`)
        matches = out["corr"].cpu().numpy()
        feats0, feats1 = np.ones((len(xyz0), 3), np.float32), np.ones((len(xyz1), 3), np.float32)
        if self.transform:
            coords0, feats0 = self.transform(coords0, feats0)
            coords1, feats1 = self.transform(coords1, feats1)
        return (xyz0, xyz1, coords0, coords1, feats0, feats1, matches, trans)


def default_collate_pair_fn(list_data):
    """`ddp_data_loaders.py:52-112`: batch-index-first int32 coordinates, correspondences offset into the batched rows."""
    xyz0, xyz1, coords0, coords1, feats0, feats1, matching, trans = list(zip(*list_data))
    C0, C1, M, lens = [], [], [], []
    o0 = o1 = 0
    for b in range(len(coords0)):
        n0, n1 = coords0[b].shape[0], coords1[b].shape[0]
        C0.append(torch.cat([torch.full((n0, 1), b, dtype=torch.int32), torch.from_numpy(np.asarray(coords0[b])).int()], 1))
        C1.append(torch.cat([torch.full((n1, 1), b, dtype=torch.int32), torch.from_numpy(np.asarray(coords1[b])).int()], 1))
        m = np.asarray(matching[b]).reshape(-1, 2)
        if len(m) == 0:
            m = np.zeros((1, 2), np.int64)                       # "in case 0 matching" (`:82-84`)
        M.append(torch.from_numpy(m.astype(np.int64) + np.array([[o0, o1]])))
        lens.append([n0, n1])
        o0 += n0; o1 += n1
    return {"pcd0": torch.cat([torch.from_numpy(np.asarray(x)) for x in xyz0]).float(),
            "pcd1": torch.cat([torch.from_numpy(np.asarray(x)) for x in xyz1]).float(),
            "sinput0_C": torch.cat(C0).int(), "sinput0_F": torch.cat([torch.from_numpy(np.asarray(f)) for f in feats0]).float(),
            "sinput1_C": torch.cat(C1).int(), "sinput1_F": torch.cat([torch.from_numpy(np.asarray(f)) for f in feats1]).float(),
            "correspondences": torch.cat(M).int(), "T_gt": torch.cat([torch.from_numpy(np.asarray(t)) for t in trans]).float(),
            "len_batch": lens}


def shared_randperm(n, seed, count):
    """A permutation of range(n): from the global torch RNG when `seed` is None, else the `count`-th one of `seed`'s own sequence
    (the same on every process)."""
    if seed is None:
        return torch.randperm(n)
    g = torch.Generator()
    g.manual_seed((int(seed) * 1_000_003 + int(count)) % (1 << 63))
    return torch.randperm(n, generator=g)


class DistributedInfSampler:
    """`lib/data_sampler.py:13-70`: an endless permutation; rank r of R takes entries it*R + r.  The permutations come from the
    global torch RNG, or with `seed` from a generator of their own seeded by (seed, permutation count): ranks that draw different
    amounts from the global RNG between two permutations still share them, so their shards stay disjoint."""

    def __init__(self, n, num_replicas=1, rank=0, shuffle=True, seed=None):
        self.n, self.num_replicas, self.rank, self.shuffle, self.seed = n, num_replicas, rank, shuffle, seed
        self.it = self.permutations = 0
        self.reset_permutation()

    def reset_permutation(self):
        self._perm = (shared_randperm(self.n, self.seed, self.permutations) if self.shuffle else torch.arange(self.n)).tolist()
        self.permutations += 1

    def __iter__(self):
        return self

    def __next__(self):
        value = self._perm[(self.it * self.num_replicas + self.rank) % len(self._perm)]
        self.it += 1
        if self.it * self.num_replicas >= len(self._perm):
            self.reset_permutation()
            self.it = 0
        return value

    def __len__(self):
        return int(math.ceil(self.n / self.num_replicas))


class PairLoader:
    """`make_data_loader` (`ddp_data_loaders.py:272-309`): per-rank batch = global batch // world, infinite, `drop_last`."""

    def __init__(self, dataset, batch_size, rank=0, world=1, shuffle=True, pin=True):
        self.dataset, self.batch_size = dataset, batch_size
        self.sampler = DistributedInfSampler(len(dataset), world, rank, shuffle)
        self.pin = pin and torch.cuda.is_available()

    def __len__(self):
        return len(self.sampler) // self.batch_size

    def __iter__(self):
        while True:
            batch = default_collate_pair_fn([self.dataset[next(self.sampler)] for _ in range(self.batch_size)])
            if self.pin:
                batch = {k: (v.pin_memory() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
            yield batch
