"""Stages the original pair-list scripts next to the oracle, so that tests/test_oracle_pair_list.py can run them unmodified:

    python oracle/pair_list_ref.py      (also run by __graft_entry__.build())

Copies `<root>/pretrain/data_preprocess/scannet_pair/{compute_full_overlapping.py, generate_list.py}` byte for byte into
`oracle/_ref/data_preprocess/` (git-ignored).  <root> is $PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the
original is absent nothing is staged.  Nothing under pointcontrast_b200/ imports this.

run(script, argv) executes a staged script as `python <script> <argv>` would, with stub `open3d` and `SensorData` modules in place of
the absent packages: the stub's `voxel_down_sample` and `KDTreeFlann.search_radius_vector_3d` are oracle/pair_list_cpu.py's.
"""
import os
import runpy
import shutil
import sys
import types

import numpy as np

SRC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "pretrain", "data_preprocess", "scannet_pair")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "data_preprocess")
FILES = ("compute_full_overlapping.py", "generate_list.py")


def stage(verbose=False):
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return False
    os.makedirs(ROOT, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(ROOT, f))
    if verbose:
        print("staged", SRC, "(pair list) ->", ROOT)
    return True


def available():
    return all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES)


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
        from scipy.spatial import cKDTree             # only where the stub runs: stage() needs no scipy
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
    """Runs the staged `script` (a name of FILES) with command-line arguments `argv` under the stubs."""
    saved_argv, saved_mods = sys.argv, {k: sys.modules.get(k) for k in ("open3d", "SensorData")}
    sys.argv = [os.path.join(ROOT, script)] + list(argv)
    sys.modules.update(_stubs())
    try:
        runpy.run_path(os.path.join(ROOT, script), run_name="__main__")
    finally:
        sys.argv = saved_argv
        for k, v in saved_mods.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
