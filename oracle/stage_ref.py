"""Stages the original PointContrast repository's Python model package next to the oracle, so that it can be executed
unmodified where the repository itself is not present (`bench.py --impl reference`, the CPU baseline leg of `bench.py`, and
`tests/test_gpu_c1.py::test_reference_model_file_runs_on_cuda_fused`).

    python oracle/stage_ref.py        (also run by __graft_entry__.build())

Copies `<root>/pretrain/pointcontrast/model/` (res16unet.py, resnet.py, modules/) byte for byte into
`oracle/_ref/pointcontrast/model/` (git-ignored), where <root> is $PCB_REFERENCE_ROOT, by default /root/reference.  Where the
original repository is absent nothing is staged.  Nothing in the product path imports it.  The reference's arithmetic layer (MinkowskiEngine 0.4.3, C++/CUDA) is not part of the original repository,
so there is nothing to compile (DESIGN.md "Oracle").
"""
import os
import shutil

SRC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "pretrain", "pointcontrast", "model")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "pointcontrast", "model")


def stage(verbose=False):
    if not os.path.isdir(SRC):
        return False
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    shutil.copytree(SRC, DST, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    if verbose:
        print("staged", SRC, "->", DST)
    return True


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present: nothing staged")
