"""Host checks of pointcontrast_b200/det_heads.py (no GPU): the new entry points are exported and reject bad arguments before touching a
device; VotingModule and ProposalModule have the original's parameters and buffers (names, order, shapes, dtypes, seeded values);
unsupported options raise; install() registers the names votenet.py imports."""
import sys

import numpy as np
import pytest
import torch

from oracle import pointnet2_cpu as O
from tests.test_oracle_det_heads import _original

ENTRY_POINTS = ("pcb_vote_epilogue", "pcb_vote_epilogue_grad", "pcb_proposal_epilogue", "pcb_proposal_epilogue_grad")


def test_entry_points_are_exported():
    from pointcontrast_b200 import _lib
    for name in ENTRY_POINTS:
        assert name in _lib.EXPORTS and getattr(_lib.lib, name)


def test_bad_arguments_return_status_2():
    from pointcontrast_b200 import _lib
    from pointcontrast_b200._lib import PcbStrided
    L = _lib.lib
    big = 1 << 31
    ms = np.ones((10, 3), np.float32)
    ms_big = np.ones((65, 3), np.float32)
    p = 1 << 20                                                   # a non-NULL pointer that is never dereferenced
    grads = (PcbStrided * 9)()
    rcs = [L.pcb_vote_epilogue(None, None, 256, None, 259, 2, 8, 1, 256, None, None, None),             # NULL pointers
           L.pcb_vote_epilogue(p, p, 256, p, 259, 0, 8, 1, 256, p, p, None),                            # B < 1
           L.pcb_vote_epilogue(p, p, 256, p, 259, big, 8, 1, 256, p, p, None),                          # B S V >= 2^31
           L.pcb_vote_epilogue(p, p, 128, p, 259, 2, 8, 1, 256, p, p, None),                            # ldf < C
           L.pcb_vote_epilogue(p, p, 256, p, 259, 2, 8, 2, 256, p, p, None),                            # ldz < (3 + C) V
           L.pcb_vote_epilogue_grad(None, None, 2, 8, 1, 256, None, None, 288, 288, None, 256, None, None),  # NULL planes
           L.pcb_vote_epilogue_grad(None, None, 2, 8, 1, 256, p, p, 288, 256, None, 256, None, None),       # Cpad < (3 + C) V
           L.pcb_vote_epilogue_grad(None, None, 2, 8, 1, 256, p, p, 256, 288, None, 256, None, None),       # ldz < Cpad
           L.pcb_vote_epilogue_grad(None, None, 2, 8, 1, 256, p, p, 288, 288, p, 128, None, None),          # ldd < C
           L.pcb_proposal_epilogue(p, 128, p, 2, 16, 12, 10, 0.26, ms.ctypes.data, p, p, None, None),       # NULL output
           L.pcb_proposal_epilogue(p, 128, p, 2, 16, 12, 10, 0.26, None, p, p, p, None),                    # NULL mean_size
           L.pcb_proposal_epilogue(p, 128, p, 2, 16, 12, 65, 0.26, ms_big.ctypes.data, p, p, p, None),     # NS > 64
           L.pcb_proposal_epilogue(p, 64, p, 2, 16, 12, 10, 0.26, ms.ctypes.data, p, p, p, None),          # ldz < X
           L.pcb_proposal_epilogue(p, 128, p, 2, 0, 12, 10, 0.26, ms.ctypes.data, p, p, p, None),          # K < 1
           L.pcb_proposal_epilogue_grad(None, 2, 16, 12, 10, 10, 0.26, ms.ctypes.data, p, p, None, 96, 96, None, None),   # NULL grads
           L.pcb_proposal_epilogue_grad(grads, 2, 16, 12, 10, 10, 0.26, ms.ctypes.data, None, None, None, 96, 96, None, None),
           L.pcb_proposal_epilogue_grad(grads, 2, 16, 12, 10, 10, 0.26, ms.ctypes.data, p, p, None, 96, 64, None, None),  # Xpad < X
           L.pcb_proposal_epilogue_grad(grads, 2, 16, 12, 10, 10, 0.26, ms.ctypes.data, p, p, None, 64, 96, None, None),  # ldz < Xpad
           L.pcb_proposal_epilogue_grad(grads, 2, 16, 12, 10, 10, 0.26, ms.ctypes.data, p, None, None, 96, 96, None, None)]  # hi, no lo
    assert rcs == [_lib.ERR_ARG] * len(rcs)


def _pair(kind, args, seed=3):
    """(the staged original module, ours), each constructed with args after the same manual_seed."""
    from pointcontrast_b200 import det_heads as ours
    ref = _original("voting_module" if kind == "VotingModule" else "proposal_module")
    torch.manual_seed(seed)
    a = getattr(ref, kind)(*args)
    torch.manual_seed(seed)
    b = getattr(ours, kind)(*args)
    return a, b


MS = np.random.default_rng(0).uniform(0.3, 2.0, (18, 3))
CASES = {"voting_v1": ("VotingModule", (1, 256)), "voting_v2": ("VotingModule", (2, 256)),
         "proposal_scannet": ("ProposalModule", (18, 1, 18, MS, 256, "seed_fps")),
         "proposal_sunrgbd": ("ProposalModule", (10, 12, 10, MS[:10], 256, "vote_fps"))}


@pytest.mark.parametrize("name", list(CASES))
def test_parameters_and_buffers_match_the_original(name):
    a, b = _pair(*CASES[name])
    pa, pb = list(a.named_parameters()), list(b.named_parameters())
    assert [(n, t.shape, t.dtype) for n, t in pa] == [(n, t.shape, t.dtype) for n, t in pb]
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert sa[k].dtype == sb[k].dtype and torch.equal(sa[k], sb[k]), k          # same seeded initial values
    kinds = (torch.nn.Conv1d, torch.nn.BatchNorm1d, torch.nn.Conv2d, torch.nn.BatchNorm2d)
    assert [type(m) for m in a.modules() if isinstance(m, kinds)] == [type(m) for m in b.modules() if isinstance(m, kinds)]
    b.load_state_dict(sa)                                                           # an original checkpoint loads, and back
    a.load_state_dict(b.state_dict())
    if name.startswith("proposal"):
        assert next(iter(dict(b.named_children()))) == "vote_aggregation"


def test_unsupported_options_raise():
    from pointcontrast_b200 import det_heads as ours
    with pytest.raises(NotImplementedError, match="seed_feature_dim"):
        ours.VotingModule(1, 200)
    with pytest.raises(NotImplementedError, match="seed_feat_dim"):
        ours.ProposalModule(10, 12, 10, MS[:10], 256, "vote_fps", seed_feat_dim=100)
    with pytest.raises(NotImplementedError, match="sampling"):
        ours.ProposalModule(10, 12, 10, MS[:10], 256, "grid")
    vm = ours.VotingModule(1, 64)
    vm.bn2.momentum = None
    with pytest.raises(NotImplementedError, match="momentum=None"):
        vm(torch.zeros(1, 8, 3), torch.zeros(1, 64, 8))
    pm = ours.ProposalModule(10, 12, 10, MS[:10], 16, "vote_fps")
    pm.bn1.momentum = None
    with pytest.raises(NotImplementedError, match="momentum=None"):
        pm(torch.zeros(1, 32, 3), torch.zeros(1, 256, 32), {})


def test_install_registers_the_four_names():
    from pointcontrast_b200 import det_heads, pointnet2_modules
    names = ("voting_module", "models.voting_module", "proposal_module", "models.proposal_module")
    saved = dict(sys.modules)
    try:
        assert det_heads.install() is det_heads
        for name in names:
            assert sys.modules[name] is det_heads
        assert sys.modules["models"].voting_module is det_heads and sys.modules["models"].proposal_module is det_heads
        assert sys.modules["pointnet2_modules"] is pointnet2_modules
    finally:
        for k in [k for k in sys.modules if k not in saved]:
            del sys.modules[k]
        sys.modules.update(saved)
        if "models" in saved:
            for name in ("voting_module", "proposal_module"):
                if hasattr(saved["models"], name) and getattr(saved["models"], name) is det_heads:
                    delattr(saved["models"], name)
