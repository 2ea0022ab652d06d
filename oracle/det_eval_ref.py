"""Stages the original VoteNet evaluation code next to the oracle, so that the GPU tests and profiles/bench_det_eval.py can run it
unmodified against pointcontrast_b200.det_eval:

    python oracle/det_eval_ref.py       (also run by __graft_entry__.build(), after oracle/detection_ref.py)

Copies, byte for byte, from `<root>/downstream/votenet_det_new/` into `oracle/_ref/votenet/` (git-ignored), beside the backbone that
oracle/detection_ref.py stages there: `models/{ap_helper,dump_helper,loss_helper}.py`, `lib/test.py`, `lib/utils/*.py` and the two
dataset model-util modules with what they load (`lib/datasets/scannet/{model_util_scannet.py, meta_data/scannet_means.npz}`,
`lib/datasets/sunrgbd/{model_util_sunrgbd.py, sunrgbd_utils.py}`).  Empty `__init__.py` files make `lib` and its subdirectories
regular packages.  <root> is $PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the original is absent nothing
is staged.  Nothing under pointcontrast_b200/ imports this.

load() imports the staged code the way the original runs it (its root and `lib/utils` on sys.path), with stubs for the modules it
imports but this path never calls (plyfile, trimesh, matplotlib, cv2: PLY writes and plotting).
"""
import importlib
import os
import shutil
import sys
import types

SRC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "downstream", "votenet_det_new")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "votenet")
FILES = [os.path.join("models", f) for f in ("ap_helper.py", "dump_helper.py", "loss_helper.py")] + [
    os.path.join("lib", "test.py"),
    os.path.join("lib", "datasets", "scannet", "model_util_scannet.py"),
    os.path.join("lib", "datasets", "scannet", "meta_data", "scannet_means.npz"),
    os.path.join("lib", "datasets", "sunrgbd", "model_util_sunrgbd.py"),
    os.path.join("lib", "datasets", "sunrgbd", "sunrgbd_utils.py"),
]
PACKAGES = ("models", "lib", os.path.join("lib", "utils"), os.path.join("lib", "datasets"), os.path.join("lib", "datasets", "scannet"),
            os.path.join("lib", "datasets", "sunrgbd"))
STUBS = ("plyfile", "trimesh", "matplotlib", "matplotlib.pyplot", "cv2")


def stage(verbose=False):
    if not os.path.isfile(os.path.join(SRC, "models", "ap_helper.py")):
        return False
    if os.path.isdir(os.path.join(ROOT, "lib")):
        shutil.rmtree(os.path.join(ROOT, "lib"))
    for f in FILES:
        os.makedirs(os.path.dirname(os.path.join(ROOT, f)), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, f), os.path.join(ROOT, f))
    shutil.copytree(os.path.join(SRC, "lib", "utils"), os.path.join(ROOT, "lib", "utils"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    for pkg in PACKAGES:
        open(os.path.join(ROOT, pkg, "__init__.py"), "a").close()
    if verbose:
        print("staged", SRC, "(evaluation) ->", ROOT)
    return True


def available():
    return all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES)


class _Anything:
    """Stands for any attribute of a stubbed module (`pyplot.cm.jet` in a default argument, PlyData, ...); never called here."""

    def __getattr__(self, attr):
        return self


def _stub_attr(attr):
    if attr.startswith("__"):
        raise AttributeError(attr)
    return _Anything()


def load():
    """Imports the staged evaluation code; returns the module `models.ap_helper` (the original's), or None where nothing is staged."""
    if not available():
        return None
    for name in STUBS:
        try:
            importlib.import_module(name)
        except ImportError:
            stub = types.ModuleType(name)
            stub.__getattr__ = _stub_attr
            sys.modules[name] = stub
    if "matplotlib.pyplot" in sys.modules and isinstance(sys.modules["matplotlib"], types.ModuleType):
        sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    for p in (os.path.join(ROOT, "lib", "utils"), ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module("models.ap_helper")


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
