"""Stages the original repository's sparse-conv detection backbone so that the tests and profiles/bench_detection.py can run it
unmodified on this library (after `me.install()` and `pointnet2.install()`):

    python oracle/detection_ref.py       (also run by __graft_entry__.build())

Copies, byte for byte, from `<root>/downstream/votenet_det_new/models/` into `oracle/_ref/votenet/models/` (git-ignored):
`backbone_module.py`, `backbone/sparseconv/{config.py, models/, lib/}` and the PointNet++ Python layer `backbone/pointnet2/
{pointnet2_utils.py, pointnet2_modules.py, pytorch_utils.py}` that `backbone_module.py` imports.  Empty `__init__.py` files make
`models` and `models.backbone` importable as packages (the original runs with its root on sys.path).  <root> is $PCB_REFERENCE_ROOT,
with the same default as oracle/stage_ref.py; where the original is absent nothing is staged.  Nothing under pointcontrast_b200/
imports this.
"""
import os
import shutil

MODELS = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "downstream", "votenet_det_new", "models")
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "votenet")
DST = os.path.join(ROOT, "models")
FILES = ("backbone_module.py",)
TREES = (os.path.join("backbone", "sparseconv", "config.py"), os.path.join("backbone", "sparseconv", "__init__.py"),
         os.path.join("backbone", "sparseconv", "models"), os.path.join("backbone", "sparseconv", "lib"))
PN2 = ("pointnet2_utils.py", "pointnet2_modules.py", "pytorch_utils.py")


def stage(verbose=False):
    if not os.path.isfile(os.path.join(MODELS, "backbone_module.py")):
        return False
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    os.makedirs(os.path.join(DST, "backbone", "pointnet2"))
    for f in FILES:
        shutil.copyfile(os.path.join(MODELS, f), os.path.join(DST, f))
    for t in TREES:
        src = os.path.join(MODELS, t)
        if os.path.isdir(src):
            shutil.copytree(src, os.path.join(DST, t), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        elif os.path.isfile(src):
            os.makedirs(os.path.dirname(os.path.join(DST, t)), exist_ok=True)
            shutil.copyfile(src, os.path.join(DST, t))
    for f in PN2:
        shutil.copyfile(os.path.join(MODELS, "backbone", "pointnet2", f), os.path.join(DST, "backbone", "pointnet2", f))
    for pkg in (DST, os.path.join(DST, "backbone"), os.path.join(DST, "backbone", "pointnet2")):
        open(os.path.join(pkg, "__init__.py"), "a").close()
    if verbose:
        print("staged", MODELS, "->", DST)
    return True


def available():
    return os.path.isfile(os.path.join(DST, "backbone_module.py"))


if __name__ == "__main__":
    print("staged" if stage(True) else f"{MODELS} not present: nothing staged")
