"""Stages the original semantic-segmentation preprocessing next to the oracle, so that tests/test_oracle_semseg_prep.py,
tests/golden/make_semseg_prep_golden.py and profiles/bench_semseg_prep.py can run it unmodified:

    python oracle/semseg_prep_ref.py      (also run by __graft_entry__.build())

Copies, byte for byte, `<root>/downstream/semseg/lib/datasets/preprocessing/{stanford.py, scannet.py}`, `<root>/downstream/semseg/lib/
{pc_utils.py, utils.py}` and the plyfile the original ships, `<root>/pretrain/data_preprocess/scannet_pair/plyfile.py`, into
`oracle/_ref/semseg_prep/` (git-ignored).  <root> is $PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the
original is absent nothing is staged.  Nothing under pointcontrast_b200/ imports this.

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
import shutil
import sys
import types

SRC = os.environ.get("PCB_REFERENCE_ROOT", "/root/reference")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "semseg_prep")
FILES = {
    os.path.join("downstream", "semseg", "lib", "datasets", "preprocessing", "stanford.py"): "stanford.py",
    os.path.join("downstream", "semseg", "lib", "datasets", "preprocessing", "scannet.py"): "scannet.py",
    os.path.join("downstream", "semseg", "lib", "pc_utils.py"): os.path.join("lib", "pc_utils.py"),
    os.path.join("downstream", "semseg", "lib", "utils.py"): os.path.join("lib", "utils.py"),
    os.path.join("pretrain", "data_preprocess", "scannet_pair", "plyfile.py"): "plyfile.py",
}
_MODULES = ("lib", "lib.utils", "lib.pc_utils", "lib.distributed_utils", "plyfile", "omegaconf", "MinkowskiEngine", "tqdm", "pathlib")


def stage(verbose=False):
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return False
    for src, dst in FILES.items():
        os.makedirs(os.path.dirname(os.path.join(ROOT, dst)), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, src), os.path.join(ROOT, dst))
    if verbose:
        print("staged", SRC, "(semseg preprocessing) ->", ROOT)
    return True


def available():
    return all(os.path.isfile(os.path.join(ROOT, f)) for f in FILES.values())


def _serial_pool(max_workers=None):
    class Pool:
        def map(self, fn, items):
            return map(fn, items)
    return Pool()


@contextlib.contextmanager
def installed(redirect=None):
    """The staged modules and the stand-ins in sys.modules (and `redirect`: {placeholder root: root} for pathlib.Path) while inside."""
    from oracle import semseg_prep_cpu
    saved = {k: sys.modules.get(k) for k in _MODULES}
    saved_path, saved_pool = list(sys.path), concurrent.futures.ProcessPoolExecutor
    for k in _MODULES:
        sys.modules.pop(k, None)
    lib = types.ModuleType("lib")
    lib.__path__ = [os.path.join(ROOT, "lib")]
    me = types.ModuleType("MinkowskiEngine")
    me.utils = types.SimpleNamespace(sparse_quantize=semseg_prep_cpu.sparse_quantize)
    sys.modules.update({
        "lib": lib, "MinkowskiEngine": me,
        "omegaconf": types.SimpleNamespace(OmegaConf=None),
        "lib.distributed_utils": types.SimpleNamespace(get_world_size=lambda: 1, get_rank=lambda: 0),
        "tqdm": types.SimpleNamespace(tqdm=lambda it, *a, **k: it),
    })
    if redirect:
        class Path(pathlib.PosixPath):
            def __init__(self, *args):
                super().__init__(*[redirect.get(a, a) if isinstance(a, str) else a for a in args])
        sys.modules["pathlib"] = types.SimpleNamespace(Path=Path)
    concurrent.futures.ProcessPoolExecutor = _serial_pool
    sys.path.insert(0, ROOT)
    try:
        yield
    finally:
        sys.path[:] = saved_path
        concurrent.futures.ProcessPoolExecutor = saved_pool
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def stanford(in_root, out_root, split_cwd):
    """The original `convert_to_ply(in_root, out_root)` then `generate_splits(out_root)` with the working directory `split_cwd` (its
    split files land in `<split_cwd>/splits/stanford/`)."""
    cwd = os.getcwd()
    with installed():
        spec = importlib.util.spec_from_file_location("_ref_semseg_stanford_prep", os.path.join(ROOT, "stanford.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.Stanford3DDatasetConverter.convert_to_ply(in_root, out_root)
        os.makedirs(split_cwd, exist_ok=True)
        os.chdir(split_cwd)
        try:
            mod.generate_splits(out_root)
        finally:
            os.chdir(cwd)


def scannet(raw_root, out_root):
    """The original scannet.py with its roots `/path/ScanNet_data/` -> raw_root and `/path/scans_processed/` -> out_root."""
    with installed({"/path/ScanNet_data/": str(raw_root), "/path/scans_processed/": str(out_root)}):
        runpy.run_path(os.path.join(ROOT, "scannet.py"), run_name="_ref_semseg_scannet_prep")


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
