"""Host checks of pointcontrast_b200/pointnet2_modules.py (no GPU): the new entry points are exported and reject bad arguments before
touching a device; every module VoteNet builds has the original's parameters and buffers (names, order, shapes, dtypes, seeded values);
unsupported options raise."""
import pytest
import torch

from oracle import pointnet2_cpu as O
from tests.test_oracle_pointnet2 import reference_modules

# every PointnetSAModuleVotes / PointnetFPModule VoteNet constructs (backbone_module.py, proposal_module.py), as constructor kwargs
SA = {
    "sa1": dict(npoint=2048, radius=0.2, nsample=64, mlp=[1, 64, 64, 128], use_xyz=True, normalize_xyz=True),
    "sa1_no_height": dict(npoint=2048, radius=0.2, nsample=64, mlp=[0, 64, 64, 128], use_xyz=True, normalize_xyz=True),
    "sa2": dict(npoint=1024, radius=0.4, nsample=32, mlp=[128, 128, 128, 256], use_xyz=True, normalize_xyz=True),
    "sa3": dict(npoint=512, radius=0.8, nsample=16, mlp=[256, 128, 128, 256], use_xyz=True, normalize_xyz=True),
    "sa4": dict(npoint=256, radius=1.2, nsample=16, mlp=[256, 128, 128, 256], use_xyz=True, normalize_xyz=True),
    "vote_aggregation": dict(npoint=256, radius=0.3, nsample=16, mlp=[256, 128, 128, 128], use_xyz=True, normalize_xyz=True),
}
FP = {"fp1": dict(mlp=[256 + 256, 256, 256]), "fp2": dict(mlp=[256 + 256, 256, 256])}


def test_entry_points_are_exported():
    from pointcontrast_b200 import _lib
    for name in ("pcb_sa_layer0", "pcb_sa_pool", "pcb_sa_pool_grad", "pcb_sa_xyz_rows"):
        assert name in _lib.EXPORTS and getattr(_lib.lib, name)


def test_bad_arguments_return_status_2():
    from pointcontrast_b200 import _lib
    L = _lib.lib
    big = 1 << 31
    rcs = [L.pcb_sa_layer0(None, None, None, 1, 10, 4, 8, 0.2, None, 0, None, 64, None, None, None, 64, None),     # NULL pointers
           L.pcb_sa_layer0(None, None, None, 1, big, 4, 8, 0.2, None, 0, None, 64, None, None, None, 64, None),    # N >= 2^31
           L.pcb_sa_layer0(None, None, None, 1, 10, 4, 0, 0.2, None, 0, None, 64, None, None, None, 64, None),     # S < 1
           L.pcb_sa_layer0(None, None, None, 1, 10, 4, 8, float("nan"), None, 0, None, 64, None, None, None, 64, None),
           L.pcb_sa_layer0(None, None, None, 1, 10, 4, 8, 0.2, None, 0, None, 64, None, None, None, 32, None),     # ldz < C0
           L.pcb_sa_pool(None, 64, 4, 8, 64, None, None, None, None, None, None, 64, None),
           L.pcb_sa_pool(None, 64, 0, 8, 64, None, None, None, None, None, None, 64, None),                          # M < 1
           L.pcb_sa_pool(None, 32, 4, 8, 64, None, None, None, None, None, None, 64, None),                          # ldz < C
           L.pcb_sa_pool_grad(None, 64, None, None, 64, 4, 8, 64, None, None),
           L.pcb_sa_pool_grad(None, 64, None, None, 64, big, 8, 64, None, None),                                     # M S >= 2^31
           L.pcb_sa_xyz_rows(None, None, 4, 8, 0.2, None, None),
           L.pcb_sa_xyz_rows(None, None, 4, 0, 0.2, None, None)]
    assert rcs == [_lib.ERR_ARG] * len(rcs)


def _pair(kind, kw, seed=3):
    """(the staged original module, ours), each constructed from its own copy of kw after the same manual_seed."""
    from pointcontrast_b200 import pointnet2_modules as ours
    _, ref = reference_modules(O.install)
    cls = "PointnetSAModuleVotes" if kind == "sa" else "PointnetFPModule"
    torch.manual_seed(seed)
    a = getattr(ref, cls)(**{k: list(v) if isinstance(v, list) else v for k, v in kw.items()})
    torch.manual_seed(seed)
    b = getattr(ours, cls)(**{k: list(v) if isinstance(v, list) else v for k, v in kw.items()})
    return a, b


@pytest.mark.parametrize("kind,name", [("sa", k) for k in SA] + [("fp", k) for k in FP])
def test_parameters_and_buffers_match_the_original(kind, name):
    a, b = _pair(kind, (SA if kind == "sa" else FP)[name])
    pa, pb = list(a.named_parameters()), list(b.named_parameters())
    assert [(n, t.shape, t.dtype) for n, t in pa] == [(n, t.shape, t.dtype) for n, t in pb]
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert sa[k].dtype == sb[k].dtype and torch.equal(sa[k], sb[k]), k          # same seeded initial values
    assert [type(m) for m in a.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.BatchNorm2d))] == \
        [type(m) for m in b.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.BatchNorm2d))]
    b.load_state_dict(sa)                                                           # an original checkpoint loads, and back
    a.load_state_dict(b.state_dict())


def test_constructor_edits_the_callers_list():
    from pointcontrast_b200 import pointnet2_modules as ours
    mlp = [1, 64, 64, 128]
    ours.PointnetSAModuleVotes(npoint=16, radius=0.2, nsample=8, mlp=mlp)
    assert mlp == [4, 64, 64, 128]


@pytest.mark.parametrize("bad", [dict(pooling="avg"), dict(pooling="rbf"), dict(sample_uniformly=True), dict(ret_unique_cnt=True),
                                 dict(npoint=None), dict(bn=False), dict(use_xyz=False), dict(mlp=[1, 48, 64, 128]), dict(mlp=[1, 64])])
def test_unsupported_options_raise(bad):
    from pointcontrast_b200 import pointnet2_modules as ours
    kw = dict(npoint=16, radius=0.2, nsample=8, mlp=[1, 64, 64, 128])
    kw.update(bad)
    with pytest.raises(NotImplementedError, match=next(iter(bad)) if "mlp" not in bad else "mlp"):
        ours.PointnetSAModuleVotes(**kw)
    with pytest.raises(NotImplementedError, match="bn"):
        ours.PointnetFPModule(mlp=[512, 256], bn=False)
    with pytest.raises(NotImplementedError, match="mlp"):
        ours.PointnetFPModule(mlp=[131, 64])
