"""Stages the original VoteNet detection preprocessing next to the oracle, so that tests/test_oracle_det_prep.py,
tests/golden/make_det_prep_golden.py and profiles/bench_det_prep.py can run it unmodified:

    python oracle/det_prep_ref.py      (also run by __graft_entry__.build())

Copies, byte for byte, `<root>/downstream/votenet_det_new/lib/datasets/scannet/{batch_load_scannet_data.py, load_scannet_data.py,
scannet_utils.py}`, `.../sunrgbd/{sunrgbd_data.py, sunrgbd_utils.py}`, `.../lib/utils/pc_util.py` and the plyfile the original ships
(`<root>/pretrain/data_preprocess/scannet_pair/plyfile.py`; the copy under `sunrgbd_trainval/` is a link out of the tree) into
`oracle/_ref/det_prep/` (git-ignored), keeping `sunrgbd_data.py`'s relative `../utils/` import path.  <root> is $PCB_REFERENCE_ROOT, with
the same default as oracle/stage_ref.py; where the original is absent nothing is staged.  Nothing under pointcontrast_b200/ imports this.

scannet() and sunrgbd() run the staged scripts with stand-ins for `cv2`, `PIL`, `trimesh` and `matplotlib`, which they import but this
path does not compute with.  Their hard-coded relative roots are redirected through the working directory, without editing a file: a
scratch directory holds `scans` and `meta_data/` links (ScanNet) or a `sunrgbd_trainval` link (SUN RGB-D) and becomes the working
directory while the script runs.
"""
import contextlib
import importlib.util
import os
import runpy
import shutil
import sys
import tempfile
import types

SRC = os.environ.get("PCB_REFERENCE_ROOT", "/root/reference")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "det_prep")
_LIB = os.path.join("downstream", "votenet_det_new", "lib")
FILES = {
    os.path.join(_LIB, "datasets", "scannet", "batch_load_scannet_data.py"): os.path.join("scannet", "batch_load_scannet_data.py"),
    os.path.join(_LIB, "datasets", "scannet", "load_scannet_data.py"): os.path.join("scannet", "load_scannet_data.py"),
    os.path.join(_LIB, "datasets", "scannet", "scannet_utils.py"): os.path.join("scannet", "scannet_utils.py"),
    os.path.join(_LIB, "datasets", "sunrgbd", "sunrgbd_data.py"): os.path.join("sunrgbd", "sunrgbd_data.py"),
    os.path.join(_LIB, "datasets", "sunrgbd", "sunrgbd_utils.py"): os.path.join("sunrgbd", "sunrgbd_utils.py"),
    os.path.join(_LIB, "utils", "pc_util.py"): os.path.join("utils", "pc_util.py"),
    os.path.join("pretrain", "data_preprocess", "scannet_pair", "plyfile.py"): os.path.join("utils", "plyfile.py"),
}
_MODULES = ("cv2", "PIL", "PIL.Image", "trimesh", "matplotlib", "matplotlib.pyplot", "plyfile", "pc_util", "sunrgbd_utils",
            "scannet_utils", "load_scannet_data")


def stage(verbose=False):
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return False
    for src, dst in FILES.items():
        os.makedirs(os.path.dirname(os.path.join(ROOT, dst)), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, src), os.path.join(ROOT, dst))
    if verbose:
        print("staged", SRC, "(VoteNet detection preprocessing) ->", ROOT)
    return True


def available():
    return all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES.values())


@contextlib.contextmanager
def installed(cwd, paths):
    """The stand-ins in sys.modules, `paths` on sys.path and `cwd` as the working directory while inside."""
    saved = {k: sys.modules.get(k) for k in _MODULES}
    saved_path, saved_cwd = list(sys.path), os.getcwd()
    for k in _MODULES:
        sys.modules.pop(k, None)
    pil = types.ModuleType("PIL")
    pil.Image = types.ModuleType("PIL.Image")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot.cm = types.SimpleNamespace(jet=None)     # a default argument of pc_util.write_ply_color
    sys.modules.update({"cv2": types.ModuleType("cv2"), "PIL": pil, "PIL.Image": pil.Image, "trimesh": types.ModuleType("trimesh"),
                        "matplotlib": mpl, "matplotlib.pyplot": mpl.pyplot})
    sys.path[:0] = paths
    os.chdir(cwd)
    try:
        yield
    finally:
        os.chdir(saved_cwd)
        sys.path[:] = saved_path
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def scannet(scans_root, label_map_file, scan_names, out_dir):
    """`python batch_load_scannet_data.py` with `scans` -> scans_root, `meta_data/scannet_train.txt` = scan_names and
    `meta_data/scannetv2-labels.combined.tsv` -> label_map_file; its `./scannet_train_detection_data` is a link to out_dir."""
    with tempfile.TemporaryDirectory() as cwd:
        os.makedirs(os.path.join(cwd, "meta_data"))
        os.symlink(os.path.abspath(scans_root), os.path.join(cwd, "scans"))
        os.symlink(os.path.abspath(label_map_file), os.path.join(cwd, "meta_data", "scannetv2-labels.combined.tsv"))
        with open(os.path.join(cwd, "meta_data", "scannet_train.txt"), "w") as f:
            f.write("".join(n + "\n" for n in scan_names))
        os.makedirs(out_dir, exist_ok=True)
        os.symlink(os.path.abspath(out_dir), os.path.join(cwd, "scannet_train_detection_data"))
        with installed(cwd, [os.path.join(ROOT, "scannet"), os.path.join(ROOT, "utils")]):
            runpy.run_path(os.path.join(ROOT, "scannet", "batch_load_scannet_data.py"), run_name="__main__")


def sunrgbd(trainval_root, out_dir, v1=True, splits=("train", "val")):
    """What `python sunrgbd_data.py --gen_v1_data` (v1) / `--gen_v2_data` runs, with `./sunrgbd_trainval` -> trainval_root and the
    output folders under out_dir."""
    os.makedirs(out_dir, exist_ok=True)
    with tempfile.TemporaryDirectory() as cwd:
        os.symlink(os.path.abspath(trainval_root), os.path.join(cwd, "sunrgbd_trainval"))
        with installed(cwd, [os.path.join(ROOT, "sunrgbd"), os.path.join(ROOT, "utils")]):
            spec = importlib.util.spec_from_file_location("_ref_sunrgbd_data", os.path.join(ROOT, "sunrgbd", "sunrgbd_data.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            for split in splits:
                mod.extract_sunrgbd_data(os.path.join(cwd, "sunrgbd_trainval", f"{split}_data_idx.txt"), split="training",
                                         output_folder=os.path.join(out_dir, f"sunrgbd_pc_bbox_votes_50k_{'v1' if v1 else 'v2'}_{split}"),
                                         save_votes=True, num_point=50000, use_v1=v1, skip_empty_scene=False)


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
