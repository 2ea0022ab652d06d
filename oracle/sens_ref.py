"""The original `.sens` extraction scripts (`SensorData.py`, `reader.py`, `point_cloud_extractor.py`, `plyfile.py`), staged by
oracle/stage_ref.py under `oracle/_ref/sens/`, so that tests/test_oracle_sens.py, tests/golden/make_sens_golden.py and
profiles/bench_sens.py can run them unmodified.  Nothing under pointcontrast_b200/ imports this.

run(script, argv) executes a staged script as `python <script> <argv>` would (the staged directory first on sys.path, so that
`from SensorData import SensorData` and `from plyfile import ...` find the staged files), with two stand-ins, neither of which
touches the arithmetic:

* `imageio.imwrite(path, a)` and `cv2.imread(path, -1)` are a lossless array codec (`np.save` / `np.load` through an open file) in
  place of 16-bit PNG; neither package is installed here;
* `np.fromstring(bytes, dtype)` is `np.frombuffer(bytes, dtype).copy()` while the script runs: NumPy 2.3 removed fromstring's binary
  mode, which `SensorData.export_depth_images` calls (an API bridge, like `collections.Sequence` in `me.install()`).
"""
import contextlib
import os
import runpy
import types

import numpy as np

from oracle import stage_ref


def available():
    return stage_ref.available("sens")


def _imwrite(path, a):
    with open(path, "wb") as f:
        np.save(f, np.asarray(a))


def _imread(path, flags=1):
    with open(path, "rb") as f:
        return np.load(f)


def _stubs():
    imageio = types.ModuleType("imageio")
    imageio.imwrite = _imwrite
    cv2 = types.ModuleType("cv2")
    cv2.imread = _imread
    return {"imageio": imageio, "cv2": cv2}


@contextlib.contextmanager
def installed():
    """The stand-ins, the staged directory on sys.path and the fromstring bridge, for code that imports the staged modules."""
    had = "fromstring" in np.__dict__
    saved_fromstring = np.__dict__.get("fromstring")
    # SensorData and plyfile are removed so that the staged ones are imported: oracle/pair_list_ref.py installs a stub SensorData
    with stage_ref.installed({"SensorData": None, "plyfile": None, **_stubs()}, path=[stage_ref.path("sens")]):
        np.fromstring = lambda b, dtype=float, *a, **k: np.frombuffer(b, dtype).copy()
        try:
            yield
        finally:
            if had:
                np.fromstring = saved_fromstring
            else:
                del np.fromstring


def run(script, argv):
    """Runs the staged `script` (`reader.py` or `point_cloud_extractor.py`) with command-line arguments `argv`."""
    script = stage_ref.path("sens", script)
    with installed(), stage_ref.installed(argv=[script] + list(argv)):
        runpy.run_path(script, run_name="__main__")


def sensor_data(path):
    """The original `SensorData(path)` (every byte of every frame read into Python)."""
    with installed():
        import SensorData
        return SensorData.SensorData(path)


def extract(sens_path, scene_dir, frame_skip):
    """The reference README's per-scene commands up to the npz frames: `reader.py --export_depth_images --export_poses
    --export_intrinsics`, then `point_cloud_extractor.py --save_npz` into `<scene_dir>/pcd`."""
    run("reader.py", ["--filename", sens_path, "--output_path", scene_dir, "--frame_skip", str(frame_skip), "--export_depth_images",
                      "--export_poses", "--export_intrinsics"])
    run("point_cloud_extractor.py", ["--input_path", scene_dir, "--output_path", os.path.join(scene_dir, "pcd"), "--save_npz"])
