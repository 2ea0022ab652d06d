"""The original sparse-conv detection backbone (`models/backbone_module.py`, `models/backbone/sparseconv/`, and the PointNet++ Python
layer it imports), staged by oracle/stage_ref.py under `oracle/_ref/votenet/models/`, so that the tests and profiles/bench_detection.py
can run it unmodified on this library (after `me.install()` and `pointnet2.install()`), with ROOT on sys.path as the original runs
with its root there.  Nothing under pointcontrast_b200/ imports this.
"""
from oracle import stage_ref

ROOT = stage_ref.path("votenet")


def available():
    return stage_ref.available("votenet")
