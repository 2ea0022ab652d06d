"""The original semantic-segmentation preprocessing (`lib/datasets/preprocessing/{stanford.py, scannet.py}`, `lib/{pc_utils.py,
utils.py}` and the plyfile the original ships), staged by oracle/stage_ref.py under `oracle/_ref/semseg_prep/`, so that
tests/test_oracle_semseg_prep.py, tests/golden/make_semseg_prep_golden.py and profiles/bench_semseg_prep.py can run it unmodified.
Nothing under pointcontrast_b200/ imports this.

stanford() and scannet() run the staged scripts with the staged `lib/` as the package `lib` and the staged plyfile as `plyfile`, and
with stand-ins for what they import but this path does not compute with: `omegaconf`, `lib.distributed_utils` and `tqdm` (a pass-through).
One stand-in does compute: `MinkowskiEngine.utils.sparse_quantize` is oracle/semseg_prep_cpu.py's restatement of ME 0.4.3, which is not
installed here -- so the quantisation in these runs is the restatement, not the original's arithmetic (DESIGN.md section 5).  The
scripts' hard-coded roots are redirected at run time without editing the files: stanford.py's functions are called with the roots as
arguments (its `generate_splits` writes `./splits/stanford/` under the working directory, which is set to `split_cwd`), and scannet.py,
which runs at import, sees a `pathlib.Path` that maps its two placeholder roots to the given ones and a serial `ProcessPoolExecutor`.
"""
import concurrent.futures
import contextlib
import importlib.util
import os
import pathlib
import runpy
import types

from oracle import stage_ref


def available():
    return stage_ref.available("semseg_prep")


def _serial_pool(max_workers=None):
    class Pool:
        def map(self, fn, items):
            return map(fn, items)
    return Pool()


@contextlib.contextmanager
def installed(redirect=None):
    """The staged modules and the stand-ins in sys.modules (and `redirect`: {placeholder root: root} for pathlib.Path) while inside."""
    from oracle import semseg_prep_cpu
    lib = types.ModuleType("lib")
    lib.__path__ = [stage_ref.path("semseg_prep", "lib")]
    me = types.ModuleType("MinkowskiEngine")
    me.utils = types.SimpleNamespace(sparse_quantize=semseg_prep_cpu.sparse_quantize)
    stubs = {
        "lib.utils": None, "lib.pc_utils": None, "plyfile": None, "pathlib": None,      # imported afresh: the staged ones, the real pathlib
        "lib": lib, "MinkowskiEngine": me,
        "omegaconf": types.SimpleNamespace(OmegaConf=None),
        "lib.distributed_utils": types.SimpleNamespace(get_world_size=lambda: 1, get_rank=lambda: 0),
        "tqdm": types.SimpleNamespace(tqdm=lambda it, *a, **k: it),
    }
    if redirect:
        class Path(pathlib.PosixPath):
            def __init__(self, *args):
                super().__init__(*[redirect.get(a, a) if isinstance(a, str) else a for a in args])
        stubs["pathlib"] = types.SimpleNamespace(Path=Path)
    saved_pool = concurrent.futures.ProcessPoolExecutor
    concurrent.futures.ProcessPoolExecutor = _serial_pool
    try:
        with stage_ref.installed(stubs, path=[stage_ref.path("semseg_prep")]):
            yield
    finally:
        concurrent.futures.ProcessPoolExecutor = saved_pool


def stanford(in_root, out_root, split_cwd):
    """The original `convert_to_ply(in_root, out_root)` then `generate_splits(out_root)` with the working directory `split_cwd` (its
    split files land in `<split_cwd>/splits/stanford/`)."""
    with installed():
        spec = importlib.util.spec_from_file_location("_ref_semseg_stanford_prep", stage_ref.path("semseg_prep", "stanford.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.Stanford3DDatasetConverter.convert_to_ply(in_root, out_root)
        os.makedirs(split_cwd, exist_ok=True)
        with stage_ref.installed(cwd=split_cwd):
            mod.generate_splits(out_root)


def scannet(raw_root, out_root):
    """The original scannet.py with its roots `/path/ScanNet_data/` -> raw_root and `/path/scans_processed/` -> out_root."""
    with installed({"/path/ScanNet_data/": str(raw_root), "/path/scans_processed/": str(out_root)}):
        runpy.run_path(stage_ref.path("semseg_prep", "scannet.py"), run_name="_ref_semseg_scannet_prep")
