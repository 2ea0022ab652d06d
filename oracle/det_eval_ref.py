"""The original VoteNet evaluation code, staged by oracle/stage_ref.py under `oracle/_ref/votenet/` (`models/ap_helper.py`,
`lib/test.py`, `lib/utils/`, the dataset model-util modules), so that the GPU tests and profiles/bench_det_eval.py can run it unmodified
against pointcontrast_b200.det_eval.  Nothing under pointcontrast_b200/ imports this.

load() imports the staged code the way the original runs it (its root and `lib/utils` on sys.path), with stubs for the modules it
imports but this path never calls (plyfile, trimesh, matplotlib, cv2: PLY writes and plotting).  Both stay installed after it returns:
the staged code imports from them at call time.
"""
import importlib
import os
import sys
import types

from oracle import stage_ref

STUBS = ("plyfile", "trimesh", "matplotlib", "matplotlib.pyplot", "cv2")


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
    if not stage_ref.available("votenet"):
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
    for p in (stage_ref.path("votenet", "lib", "utils"), stage_ref.path("votenet")):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module("models.ap_helper")
