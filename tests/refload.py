"""Import pieces of the original PointContrast repository on top of a chosen MinkowskiEngine-compatible module: the
tree named by PCB_REFERENCE_ROOT, else the model package staged by `oracle/stage_ref.py` (the trainer module is not staged).
Used by the golden-data generators under tests/golden/, by `bench.py`'s reference legs and by
`tests/test_gpu_c1.py::test_reference_model_file_runs_on_cuda_fused`."""
import importlib
import os
import sys
import types

REF_PC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", ""), "pretrain", "pointcontrast")
if not os.environ.get("PCB_REFERENCE_ROOT") or not os.path.isdir(REF_PC):       # the model package staged by oracle/stage_ref.py
    _staged = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "pointcontrast")
    if os.path.isdir(os.path.join(_staged, "model")):
        REF_PC = _staged


def available():
    return os.path.isdir(os.path.join(REF_PC, "model"))


def _purge():
    for k in [k for k in sys.modules if k == "model" or k.startswith("model.") or k == "lib" or k.startswith("lib.")]:
        del sys.modules[k]


def load_reference_model_module(me_module_installer):
    """Returns the reference's `model` package imported against the ME surface installed by `me_module_installer()`."""
    _purge()
    me_module_installer()
    sys.path.insert(0, REF_PC)
    try:
        return importlib.import_module("model")
    finally:
        sys.path.remove(REF_PC)


def load_reference_trainer_module(me_module_installer):
    _purge()
    me_module_installer()
    for name in ("tensorboardX", "omegaconf"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.SummaryWriter = object
            m.OmegaConf = object
            sys.modules[name] = m
    sys.path.insert(0, REF_PC)
    try:
        return importlib.import_module("lib.ddp_trainer")
    finally:
        sys.path.remove(REF_PC)


class Cfg(dict):
    """attribute-style nested config, enough for `config.net.x` / `config.opt.y`."""
    def __getattr__(self, k):
        v = self[k]
        return Cfg(v) if isinstance(v, dict) else v


def default_config():
    return Cfg(net=dict(model="Res16UNet34C", model_n_out=32, conv1_kernel_size=3, normalize_feature=True),
               opt=dict(bn_momentum=0.05))
