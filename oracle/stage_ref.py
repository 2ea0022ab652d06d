"""Stages the parts of the original PointContrast repository that the tests, the golden-data generators, the profiles and
`bench.py`'s reference leg run unmodified, and gives them one way to run it under stand-in modules.

    python oracle/stage_ref.py        (also run by __graft_entry__.build())

MANIFEST lists every staged file and tree: its path under the original repository's root (`$PCB_REFERENCE_ROOT`, by default
/root/reference), its destination under `oracle/_ref/` (git-ignored) and whether it is a file, a tree or an empty `__init__.py` that
makes a directory importable as a package.  Entries are grouped by the destination root they share.  stage() copies each group byte for
byte into a freshly cleared destination, and only when all of the group's sources exist; where the original repository is absent nothing
is staged and nothing already staged is touched.  `oracle/_ref/pointnet2_ext/`, the reference extension oracle/pointnet2_ref.py
compiles, is no group's destination.  path() and available() are the only code that locates and checks staged files: each `*_ref.py`
exposes its group's check as its own `available()`, and paths elsewhere are built with path().

installed() puts stand-in modules, sys.path entries, a working directory and sys.argv in place for the staged code and restores all of
them on exit.  The `*_ref.py` modules beside this one hold the stand-ins and runners specific to each part.  Nothing under
pointcontrast_b200/ imports any of this.  The reference's arithmetic layer (MinkowskiEngine 0.4.3, C++/CUDA) is not part of the original
repository, so it is not staged (DESIGN.md "Oracle").
"""
import contextlib
import os
import shutil
import sys

REFERENCE = os.environ.get("PCB_REFERENCE_ROOT", "/root/reference")
STAGED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")

FILE, TREE, PACKAGE = "file", "tree", "package"
_VOTENET = "downstream/votenet_det_new/"
_PAIR = "pretrain/data_preprocess/scannet_pair/"
_SEMSEG = "downstream/semseg/lib/"


def _mirror(kind, prefix, *names):
    """Entries staging `<prefix><name>` as `<name>`."""
    return [(kind, prefix + n, n) for n in names]


def _packages(*dirs):
    return [(PACKAGE, None, d) for d in dirs]


# group (destination root under oracle/_ref/) -> [(kind, source under REFERENCE, destination under the group)]
MANIFEST = {
    # the pretraining model package (res16unet.py, resnet.py, modules/)
    "pointcontrast/model": [(TREE, "pretrain/pointcontrast/model", "")],
    "votenet": [
        # the sparse-conv detection backbone and the PointNet++ Python layer it imports
        *_mirror(FILE, _VOTENET, "models/backbone_module.py", "models/backbone/sparseconv/__init__.py",
                 "models/backbone/sparseconv/config.py", "models/backbone/pointnet2/pointnet2_utils.py",
                 "models/backbone/pointnet2/pointnet2_modules.py", "models/backbone/pointnet2/pytorch_utils.py"),
        *_mirror(TREE, _VOTENET, "models/backbone/sparseconv/models", "models/backbone/sparseconv/lib"),
        # the evaluation code, the criterion and the dataset model-util modules with what they load
        *_mirror(FILE, _VOTENET, "models/ap_helper.py", "models/dump_helper.py", "models/loss_helper.py", "lib/test.py",
                 "lib/datasets/scannet/model_util_scannet.py", "lib/datasets/scannet/meta_data/scannet_means.npz",
                 "lib/datasets/sunrgbd/model_util_sunrgbd.py", "lib/datasets/sunrgbd/sunrgbd_utils.py"),
        *_mirror(TREE, _VOTENET, "lib/utils"),
        # the detection datasets
        *_mirror(FILE, _VOTENET, "lib/datasets/scannet/scannet_detection_dataset.py",
                 "lib/datasets/sunrgbd/sunrgbd_detection_dataset.py"),
        # the VoteNet heads
        *_mirror(FILE, _VOTENET, "models/votenet.py", "models/voting_module.py", "models/proposal_module.py"),
        # the PointNet++ Python layer a second time, on its own, for the operator tests
        *_mirror(FILE, _VOTENET + "models/backbone/", "pointnet2/pointnet2_utils.py", "pointnet2/pointnet2_modules.py",
                 "pointnet2/pytorch_utils.py"),
        *_packages("models", "models/backbone", "models/backbone/pointnet2", "lib", "lib/utils", "lib/datasets",
                   "lib/datasets/scannet", "lib/datasets/sunrgbd"),
    ],
    # the pair-list scripts
    "data_preprocess": _mirror(FILE, _PAIR, "compute_full_overlapping.py", "generate_list.py"),
    # the .sens extraction scripts
    "sens": _mirror(FILE, _PAIR, "SensorData.py", "reader.py", "point_cloud_extractor.py", "plyfile.py"),
    # the semantic-segmentation full point-cloud evaluation
    "semseg/lib": _mirror(FILE, _SEMSEG, "utils.py", "datasets/scannet.py", "datasets/stanford.py"),
    # the semantic-segmentation preprocessing, with the plyfile the original ships
    "semseg_prep": [
        (FILE, _SEMSEG + "datasets/preprocessing/stanford.py", "stanford.py"),
        (FILE, _SEMSEG + "datasets/preprocessing/scannet.py", "scannet.py"),
        *_mirror(FILE, "downstream/semseg/", "lib/pc_utils.py", "lib/utils.py"),
        (FILE, _PAIR + "plyfile.py", "plyfile.py"),
    ],
    # the VoteNet detection preprocessing, keeping sunrgbd_data.py's relative `../utils/` import path; its plyfile is the one under
    # scannet_pair/ (the copy under sunrgbd_trainval/ is a link out of the tree)
    "det_prep": [
        *_mirror(FILE, _VOTENET + "lib/datasets/", "scannet/batch_load_scannet_data.py", "scannet/load_scannet_data.py",
                 "scannet/scannet_utils.py", "sunrgbd/sunrgbd_data.py", "sunrgbd/sunrgbd_utils.py"),
        *_mirror(FILE, _VOTENET + "lib/", "utils/pc_util.py"),
        (FILE, _PAIR + "plyfile.py", "utils/plyfile.py"),
    ],
}


def path(group, *parts):
    """The staged `parts` of `group` (a MANIFEST key), whether or not they are staged."""
    if group not in MANIFEST:
        raise KeyError(f"no staged group {group!r}")
    return os.path.join(STAGED, group, *parts)


def _present(kind, p):
    if kind == PACKAGE:
        p = os.path.join(p, "__init__.py")
    return os.path.isdir(p) if kind == TREE else os.path.isfile(p)


def available(group):
    """Whether every entry of `group` is staged."""
    return all(_present(kind, path(group, dst)) for kind, _, dst in MANIFEST[group])


def stage(verbose=False):
    """Stages every group whose sources all exist under REFERENCE; returns the names of the groups staged."""
    staged = []
    for group, entries in MANIFEST.items():
        if not all(_present(kind, os.path.join(REFERENCE, src)) for kind, src, _ in entries if kind != PACKAGE):
            continue
        if os.path.isdir(path(group)):
            shutil.rmtree(path(group))
        for kind, src, dst in entries:
            if kind == TREE:
                shutil.copytree(os.path.join(REFERENCE, src), path(group, dst), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"),
                                dirs_exist_ok=True)
            elif kind == FILE:
                os.makedirs(os.path.dirname(path(group, dst)), exist_ok=True)
                shutil.copyfile(os.path.join(REFERENCE, src), path(group, dst))
            else:
                os.makedirs(path(group, dst), exist_ok=True)
                open(path(group, dst, "__init__.py"), "a").close()
        staged.append(group)
        if verbose:
            print("staged", REFERENCE, "->", path(group))
    return staged


_ABSENT = object()


@contextlib.contextmanager
def installed(modules=None, path=(), cwd=None, argv=None):
    """While inside: `modules` ({name: module, or None to remove the name}) in sys.modules, `path` ahead of sys.path, `cwd` as the
    working directory and `argv` as sys.argv.  On exit, whether or not the body raised, each of those sys.modules names, sys.path, the
    working directory and sys.argv are as they were on entry."""
    modules = dict(modules or {})
    saved = {k: sys.modules.get(k, _ABSENT) for k in modules}
    saved_path, saved_cwd, saved_argv = list(sys.path), os.getcwd(), sys.argv
    try:
        for k, m in modules.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
        sys.path[:0] = path
        if cwd is not None:
            os.chdir(cwd)
        if argv is not None:
            sys.argv = list(argv)
        yield
    finally:
        sys.argv = saved_argv
        os.chdir(saved_cwd)
        sys.path[:] = saved_path
        for k, v in saved.items():
            if v is _ABSENT:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


if __name__ == "__main__":
    groups = stage(True)
    print(f"staged {len(groups)} of {len(MANIFEST)} groups" if groups else f"{REFERENCE} not present: nothing staged")
