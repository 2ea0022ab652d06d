"""Generates tests/golden/semseg_augment.npz: the reference's own semantic-segmentation augmentation
(`downstream/semseg/lib/transforms.py`, `lib/voxelizer.py`, wired as `lib/dataset.py:275-309,330-351` does) on two seeded synthetic
labelled rooms, with every random draw recorded.

    python tests/golden/make_semseg_golden.py <PointContrast root>

The two reference modules are loaded by file path (`lib/__init__.py` imports open3d).  `MinkowskiEngine` is a stand-in whose
`utils.sparse_quantize` is the oracle's (ME 0.4.3 label semantics, rows in key order), and `collections.Iterable` is aliased for
Python >= 3.10.  `random.random` and `np.random.{uniform,rand,randn,choice,shuffle}` are wrapped to record each draw.

Scene 0: ScanNet at 2 cm (`ScannetVoxelization2cmDataset`: elastic distortion, no clip); scene 1: S3DIS (`StanfordDataset`:
5 cm, clipped to 8 m cubes).  Seeds are searched so that scene 0 takes the elastic, dropout and auto-contrast branches.
"""
import collections
import collections.abc
import importlib.util
import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import semseg_data_cpu as O  # noqa: E402
from pointcontrast_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "semseg_augment.npz")


def load_reference(root):
    collections.Iterable = collections.abc.Iterable
    me = types.ModuleType("MinkowskiEngine")
    me.utils = types.SimpleNamespace(sparse_quantize=O.sparse_quantize)
    sys.modules["MinkowskiEngine"] = me
    mods = []
    for name in ("transforms", "voxelizer"):
        path = os.path.join(root, "downstream", "semseg", "lib", name + ".py")
        spec = importlib.util.spec_from_file_location("ref_semseg_" + name, path)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods.append(m)
    return mods


class Recorder:
    def __init__(self):
        self.rec = []
        self.orig = dict(random=random.random, uniform=np.random.uniform, rand=np.random.rand, randn=np.random.randn,
                         choice=np.random.choice, shuffle=np.random.shuffle)

    def install(self):
        o, rec = self.orig, self.rec

        def w_random():
            v = o["random"](); rec.append(("random", v)); return v

        def w_uniform(*a, **k):
            v = o["uniform"](*a, **k); rec.append(("uniform", v)); return v

        def w_rand(*a):
            v = o["rand"](*a); rec.append(("rand", np.array(v))); return v

        def w_randn(*a):
            v = o["randn"](*a); rec.append(("randn", np.array(v))); return v

        def w_choice(*a, **k):
            v = o["choice"](*a, **k); rec.append(("choice", np.array(v))); return v

        def w_shuffle(x):
            perm = list(range(len(x)))
            o["shuffle"](perm)                       # the same Fisher-Yates draws as shuffling the list itself
            y = list(x)
            x[:] = [y[i] for i in perm]
            rec.append(("shuffle", np.array(perm)))

        random.random, np.random.uniform, np.random.rand = w_random, w_uniform, w_rand
        np.random.randn, np.random.choice, np.random.shuffle = w_randn, w_choice, w_shuffle

    def uninstall(self):
        random.random = self.orig["random"]
        for k in ("uniform", "rand", "randn", "choice", "shuffle"):
            setattr(np.random, k, self.orig[k])


def reference_scene(T, V, coords, feats, labels, p, rec):
    """`dataset.py:275-309` with `augment_data=True` and the transform lists of `dataset.py:330-351`.  Also returns whether the
    auto-contrast branch was taken (it drew a blend factor after its gate)."""
    taken = {}

    class AutoContrast(T.ChromaticAutoContrast):
        def __call__(self, *args):
            n = len(rec.rec)
            r = super().__call__(*args)
            taken["contrast"] = len(rec.rec) - n == 2
            return r

    prevoxel = T.Compose([T.ElasticDistortion(p["elastic"])])
    inputs = T.Compose([T.RandomDropout(0.2), T.RandomHorizontalFlip("z", False), AutoContrast(),
                        T.ChromaticTranslation(p["trans_ratio"]), T.ChromaticJitter(p["jitter_std"])])
    vox = V.Voxelizer(voxel_size=p["voxel_size"], clip_bound=p["clip_bound"], use_augmentation=True, scale_augmentation_bound=p["scale_bound"],
                      rotation_augmentation_bound=p["rotation_bound"], translation_augmentation_ratio_bound=p["translation_ratio_bound"],
                      ignore_label=255)
    out = {}
    coords, feats, labels = prevoxel(coords, feats, labels)
    out["elastic"] = coords.copy()
    coords, feats, labels, trans = vox.voxelize(coords, feats, labels)
    out["transformation"] = trans
    out["vox_coords"], out["vox_feats"], out["vox_labels"] = coords.copy(), feats.copy(), labels.copy()
    coords, feats, labels = inputs(coords, feats, labels)
    lut = O.label_map(p["num_labels"], p["ignore_labels"], 255)
    out["coords"], out["feats"], out["labels"] = coords, feats, lut[np.asarray(labels)]
    return out, taken["contrast"]


def main(root):
    T, V = load_reference(root)
    z = {}
    scenes = [("scannet2cm", O.SCANNET_2CM, 11, 8_000, 1.0, (1, 2, 3, 4, 5, 6, 7, 8, 9)),
              ("stanford", O.STANFORD, 12, 5_000, 2.6, (0, 1, 2, 3, 4, 5, 6, 7, 8))]
    for s, (name, p, room_seed, n, scale, labs) in enumerate(scenes):
        xyz, rgb, lab = synth.synth_labelled_room(room_seed, n, scale=scale, labels=labs, num_labels=p["num_labels"])
        for seed in range(1000):
            random.seed(seed)
            np.random.seed(seed)
            rec = Recorder()
            rec.install()
            try:
                out, took_contrast = reference_scene(T, V, xyz.copy(), rgb.astype(np.float32), lab.astype(np.int32), p, rec)
            finally:
                rec.uninstall()
            kinds = [k for k, _ in rec.rec]
            took_dropout = "choice" in kinds
            if s == 1 or (kinds[1] == "randn" and took_dropout and took_contrast):
                break
        print(name, "seed", seed, "draws", kinds, "voxels", len(out["vox_coords"]), "->", len(out["coords"]))
        pre = f"s{s}_"
        z[pre + "name"] = np.array(name)
        z[pre + "xyz"], z[pre + "rgb"], z[pre + "label"] = xyz, rgb, lab
        z[pre + "kinds"] = np.array(kinds)
        for i, (k, v) in enumerate(rec.rec):
            v = np.asarray(v)
            if k == "randn" and v.ndim == 4:
                v = v.astype(np.float32)             # the elastic noise grid: the reference casts it to float32 at once
            if k in ("choice", "shuffle"):
                v = v.astype(np.int32)
            z[f"{pre}d{i}"] = v
        for k, v in out.items():
            z[pre + k] = np.asarray(v)
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
