"""The original VoteNet detection preprocessing (`lib/datasets/scannet/{batch_load_scannet_data.py, load_scannet_data.py,
scannet_utils.py}`, `lib/datasets/sunrgbd/{sunrgbd_data.py, sunrgbd_utils.py}`, `lib/utils/pc_util.py` and the plyfile the original
ships), staged by oracle/stage_ref.py under `oracle/_ref/det_prep/`, so that tests/test_oracle_det_prep.py,
tests/golden/make_det_prep_golden.py and profiles/bench_det_prep.py can run it unmodified.  Nothing under pointcontrast_b200/ imports
this.

scannet() and sunrgbd() run the staged scripts with stand-ins for `cv2`, `PIL`, `trimesh` and `matplotlib`, which they import but this
path does not compute with.  Their hard-coded relative roots are redirected through the working directory, without editing a file: a
scratch directory holds `scans` and `meta_data/` links (ScanNet) or a `sunrgbd_trainval` link (SUN RGB-D) and becomes the working
directory while the script runs.
"""
import importlib.util
import os
import runpy
import tempfile
import types

from oracle import stage_ref


def available():
    return stage_ref.available("det_prep")


def installed(cwd, paths):
    """The stand-ins in sys.modules, `paths` on sys.path and `cwd` as the working directory while inside."""
    pil = types.ModuleType("PIL")
    pil.Image = types.ModuleType("PIL.Image")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot.cm = types.SimpleNamespace(jet=None)     # a default argument of pc_util.write_ply_color
    stubs = {"plyfile": None, "pc_util": None, "sunrgbd_utils": None, "scannet_utils": None, "load_scannet_data": None,  # the staged ones
             "cv2": types.ModuleType("cv2"), "PIL": pil, "PIL.Image": pil.Image, "trimesh": types.ModuleType("trimesh"), "matplotlib": mpl,
             "matplotlib.pyplot": mpl.pyplot}
    return stage_ref.installed(stubs, path=paths, cwd=cwd)


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
        with installed(cwd, [stage_ref.path("det_prep", "scannet"), stage_ref.path("det_prep", "utils")]):
            runpy.run_path(stage_ref.path("det_prep", "scannet", "batch_load_scannet_data.py"), run_name="__main__")


def sunrgbd(trainval_root, out_dir, v1=True, splits=("train", "val")):
    """What `python sunrgbd_data.py --gen_v1_data` (v1) / `--gen_v2_data` runs, with `./sunrgbd_trainval` -> trainval_root and the
    output folders under out_dir."""
    os.makedirs(out_dir, exist_ok=True)
    with tempfile.TemporaryDirectory() as cwd:
        os.symlink(os.path.abspath(trainval_root), os.path.join(cwd, "sunrgbd_trainval"))
        with installed(cwd, [stage_ref.path("det_prep", "sunrgbd"), stage_ref.path("det_prep", "utils")]):
            spec = importlib.util.spec_from_file_location("_ref_sunrgbd_data", stage_ref.path("det_prep", "sunrgbd", "sunrgbd_data.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            for split in splits:
                mod.extract_sunrgbd_data(os.path.join(cwd, "sunrgbd_trainval", f"{split}_data_idx.txt"), split="training",
                                         output_folder=os.path.join(out_dir, f"sunrgbd_pc_bbox_votes_50k_{'v1' if v1 else 'v2'}_{split}"),
                                         save_votes=True, num_point=50000, use_v1=v1, skip_empty_scene=False)
