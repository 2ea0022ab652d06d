"""Stages the original `.sens` extraction scripts next to the oracle, so that tests/test_oracle_sens.py,
tests/golden/make_sens_golden.py and profiles/bench_sens.py can run them unmodified:

    python oracle/sens_ref.py      (also run by __graft_entry__.build())

Copies `<root>/pretrain/data_preprocess/scannet_pair/{SensorData.py, reader.py, point_cloud_extractor.py, plyfile.py}` byte for byte
into `oracle/_ref/sens/` (git-ignored).  <root> is $PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the
original is absent nothing is staged.  Nothing under pointcontrast_b200/ imports this.

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
import shutil
import sys
import types

import numpy as np

SRC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "pretrain", "data_preprocess", "scannet_pair")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "sens")
FILES = ("SensorData.py", "reader.py", "point_cloud_extractor.py", "plyfile.py")
_MODULES = ("SensorData", "plyfile", "imageio", "cv2")


def stage(verbose=False):
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return False
    os.makedirs(ROOT, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(ROOT, f))
    if verbose:
        print("staged", SRC, "(.sens extraction) ->", ROOT)
    return True


def available():
    return all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES)


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
    saved_mods = {k: sys.modules.get(k) for k in _MODULES}
    saved_path = list(sys.path)
    had = "fromstring" in np.__dict__
    saved_fromstring = np.__dict__.get("fromstring")
    for k in ("SensorData", "plyfile"):
        sys.modules.pop(k, None)                     # oracle/pair_list_ref.py installs a stub SensorData while it runs
    sys.modules.update(_stubs())
    sys.path.insert(0, ROOT)
    np.fromstring = lambda b, dtype=float, *a, **k: np.frombuffer(b, dtype).copy()
    try:
        yield
    finally:
        sys.path[:] = saved_path
        if had:
            np.fromstring = saved_fromstring
        else:
            del np.fromstring
        for k, v in saved_mods.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def run(script, argv):
    """Runs the staged `script` (a name of FILES) with command-line arguments `argv`."""
    saved_argv = sys.argv
    sys.argv = [os.path.join(ROOT, script)] + list(argv)
    try:
        with installed():
            runpy.run_path(os.path.join(ROOT, script), run_name="__main__")
    finally:
        sys.argv = saved_argv


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


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
