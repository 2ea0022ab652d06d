"""The original pair-list scripts (`compute_full_overlapping.py`, `generate_list.py`), staged by oracle/stage_ref.py under
`oracle/_ref/data_preprocess/`, so that tests/test_oracle_pair_list.py can run them unmodified.  Nothing under pointcontrast_b200/
imports this.

run(script, argv) executes a staged script as `python <script> <argv>` would, with stub `open3d` and `SensorData` modules in place of
the absent packages: the stub's `voxel_down_sample` and `KDTreeFlann.search_radius_vector_3d` are oracle/pair_list_cpu.py's.
"""
import os
import runpy
import types

import numpy as np

from oracle import stage_ref


def available():
    return stage_ref.available("data_preprocess")


class PointCloud:
    """open3d.geometry.PointCloud: `points` an fp64 [n, 3] array."""

    def __init__(self):
        self.points = np.zeros((0, 3))
        self.colors = None

    def voxel_down_sample(self, voxel_size):
        from oracle import pair_list_cpu as O
        out = PointCloud()
        out.points = O.voxel_down_sample(self.points, voxel_size)
        return out


class KDTreeFlann:
    """open3d.geometry.KDTreeFlann: search_radius_vector_3d returns [k, indices, squared distances] of the points within the radius
    (oracle decision, ascending distance)."""

    def __init__(self, pcd):
        from scipy.spatial import cKDTree
        self.points = np.asarray(pcd.points, np.float64)
        self.tree = cKDTree(self.points)

    def search_radius_vector_3d(self, point, radius):
        from oracle import pair_list_cpu as O
        cand = np.asarray(self.tree.query_ball_point(np.asarray(point, np.float64), radius * (1 + 1e-9)), np.int64)
        cand = cand[O.within(self.points[cand], point, radius)]
        d = self.points[cand] - np.asarray(point, np.float64)
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        order = np.argsort(d2, kind="stable")
        return [len(cand), list(cand[order]), list(d2[order])]


def _stubs():
    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud, KDTreeFlann=KDTreeFlann)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64))
    sd = types.ModuleType("SensorData")
    sd.SensorData = type("SensorData", (), {})
    return {"open3d": o3d, "SensorData": sd}


def run(script, argv):
    """Runs the staged `script` (`compute_full_overlapping.py` or `generate_list.py`) with command-line arguments `argv` under the
    stubs."""
    script = stage_ref.path("data_preprocess", script)
    with stage_ref.installed(_stubs(), argv=[script] + list(argv)):
        runpy.run_path(script, run_name="__main__")
