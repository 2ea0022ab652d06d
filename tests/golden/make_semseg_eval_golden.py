"""Generates tests/golden/semseg_eval.npz: the reference's own evaluation loop (`downstream/semseg/lib/test.py::test`, unmodified) on
seeded logits.

    python tests/golden/make_semseg_eval_golden.py <PointContrast root>

`lib/test.py` and `lib/utils.py` are loaded by file path under the package name `lib`, with stand-ins for what is not installed:
`MinkowskiEngine.SparseTensor` (holds the features), `omegaconf`, and the `lib.pc_utils` / `lib.distributed_utils` modules `utils.py`
imports from (plyfile, pandas; one process).  The "model" returns the committed logits of the batch it is called on; the loader's
iterator has `.next()`; `config.misc.is_cuda` is False, so everything runs on the CPU with torch's softmax and scikit-learn's
`average_precision_score`.  `print_info` is wrapped to record the final histogram and per-class AP it is handed.

Data: 20 classes, four batches of uneven size with about 10 % ignored rows (255); every class has a positive in every batch, so the
rule for a class absent from a batch does not enter.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "semseg_eval.npz")
C = 20
SIZES = (701, 1240, 515, 968)


class Cfg(dict):
    def __getattr__(self, k):
        v = self[k]
        return Cfg(v) if isinstance(v, dict) else v


def load_reference(root):
    lib = types.ModuleType("lib")
    lib.__path__ = []
    sys.modules["lib"] = lib
    stubs = {"omegaconf": dict(OmegaConf=object),
             "lib.pc_utils": dict(colorize_pointcloud=None, save_point_cloud=None),
             "lib.distributed_utils": dict(get_world_size=lambda: 1, get_rank=lambda: 0)}
    for name, attrs in stubs.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    me = types.ModuleType("MinkowskiEngine")

    class SparseTensor:
        def __init__(self, feats, coords):
            self.F, self.C = feats, coords

        def to(self, device):
            return self
    me.SparseTensor = SparseTensor
    sys.modules["MinkowskiEngine"] = me
    mods = {}
    for name in ("utils", "test"):
        path = os.path.join(root, "downstream", "semseg", "lib", name + ".py")
        spec = importlib.util.spec_from_file_location("lib." + name, path)
        m = importlib.util.module_from_spec(spec)
        sys.modules["lib." + name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods["test"]


def make_batches(seed=0):
    g = np.random.default_rng(seed)
    logits, targets = [], []
    for n in SIZES:
        t = np.concatenate([np.arange(C), g.integers(0, C, n - C)])
        g.shuffle(t)
        x = g.standard_normal((n, C)).astype(np.float32) * 2.0
        x[np.arange(n), t] += g.random(n).astype(np.float32) * 3.0          # the target's logit raised: a better-than-chance model
        t[g.random(n) < 0.1] = 255
        for c in range(C):                                                 # keep a positive of every class after the ignores
            if not (t == c).any():
                t[np.flatnonzero(t == 255)[0]] = c
        logits.append(x)
        targets.append(t.astype(np.int64))
    return logits, targets


def main(root):
    T = load_reference(root)
    logits, targets = make_batches()
    seen = {}

    def print_info(*args, **kw):
        seen["hist"], seen["ap_class"] = np.array(args[8]), np.array(args[9])
    T.print_info = print_info

    class Dataset:
        NUM_LABELS = C

        def reorder_result(self, x):
            return x

        def get_classnames(self):
            return None

    class Iter:
        def __init__(self):
            self.i = 0

        def next(self):
            i, self.i = self.i, self.i + 1
            n = len(targets[i])
            model.batch = i
            return torch.zeros(n, 4, dtype=torch.int32), torch.zeros(n, 3), torch.from_numpy(targets[i])

    class Loader:
        dataset = Dataset()

        def __iter__(self):
            return Iter()

        def __len__(self):
            return len(targets)

    class Model:
        batch = 0

        def eval(self):
            pass

        def __call__(self, sinput):
            return types.SimpleNamespace(F=torch.from_numpy(logits[self.batch]))
    model = Model()
    config = Cfg(misc=dict(is_cuda=False), data=dict(ignore_label=255, return_transformation=False), net=dict(wrapper_type=None),
                 augmentation=dict(normalize_color=False), train=dict(empty_cache_freq=1),
                 test=dict(save_prediction=False, test_original_pointcloud=False, evaluate_original_pointcloud=False, test_stat_freq=100))
    loss, score, mAP, mIoU = T.test(model, Loader(), config)
    print("loss", loss, "score", score, "mAP", mAP, "mIoU", mIoU)
    z = dict(sizes=np.array(SIZES), logits=np.concatenate(logits), targets=np.concatenate(targets),
             result=np.array([loss, score, mAP, mIoU], np.float64), hist=seen["hist"].astype(np.int64), ap_class=seen["ap_class"])
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
