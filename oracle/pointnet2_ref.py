"""Compiles the original repository's PointNet++ extension (`downstream/votenet_det_new/models/backbone/pointnet2/_ext_src`) for sm_90a,
so that the GPU tests and profiles/bench_pointnet2.py can run the reference's own kernels next to this library's.  Its Python layer is
staged by oracle/stage_ref.py under `oracle/_ref/votenet/pointnet2/`, where the tests run it unmodified on pointcontrast_b200.pointnet2
and on oracle.pointnet2_cpu.

    python -m oracle.pointnet2_ref       (also run by __graft_entry__.build())

Builds `oracle/_ref/pointnet2_ext/_ext*.so` (git-ignored) with torch.utils.cpp_extension, TORCH_CUDA_ARCH_LIST=9.0a and
`-O3 --fmad=false`: with one rounding per operation the reference's distance predicates are reproducible on the host (DESIGN.md §6).
The original repository is found at oracle/stage_ref.py's REFERENCE.  Where it is absent nothing is built; where it is present, a
failing compile raises.  Nothing under pointcontrast_b200/ imports this.
"""
import glob
import importlib.machinery
import importlib.util
import os

from oracle import stage_ref

SRC = os.path.join(stage_ref.REFERENCE, "downstream", "votenet_det_new", "models", "backbone", "pointnet2", "_ext_src")
OUT = os.path.join(stage_ref.STAGED, "pointnet2_ext")


def _built():
    so = glob.glob(os.path.join(OUT, "_ext*.so"))
    return so[0] if so else None


def build(verbose=False):
    """Compile (or bring up to date) the reference extension; False where the original repository is absent."""
    if not os.path.isdir(SRC):
        return False
    from torch.utils import cpp_extension
    os.makedirs(OUT, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    sources = sorted(glob.glob(os.path.join(SRC, "src", "*.cpp")) + glob.glob(os.path.join(SRC, "src", "*.cu")))
    cpp_extension.load(name="_ext", sources=sources, extra_include_paths=[os.path.join(SRC, "include")], extra_cflags=["-O3"],
                       extra_cuda_cflags=["-O3", "--fmad=false"], build_directory=OUT, verbose=verbose)
    if verbose:
        print("built", _built())
    return True


def load():
    """The compiled reference `_ext` module (CUDA tensors only), or None where it was not built."""
    so = _built()
    if so is None:
        return None
    import torch  # noqa: F401  (the extension links against torch's libraries)
    loader = importlib.machinery.ExtensionFileLoader("_ext", so)
    spec = importlib.util.spec_from_file_location("_ext", so, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print("built" if build(True) else f"{SRC} not present: nothing built")
