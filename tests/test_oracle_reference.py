"""The oracle against what the original PointContrast code computed (model graph, hardest-contrastive loss, PointInfoNCE training
iteration).  The original's outputs on these seeded inputs are stored under tests/golden/ (tests/golden/make_reference_golden.py
runs the original code to produce them)."""
import json
import os
import types

import numpy as np
import torch

from oracle import loss_cpu, me_cpu
from tests import refload

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HARDEST_NUM_POS = (1024, 5000)
NCE_NPOS = (64, 1 << 20)                 # with and without the npos subsample (`lib/ddp_trainer.py:411-415`)


def reference_structure():
    return json.loads(np.load(os.path.join(GOLDEN, "reference_model_structure.npz"))["json"].tobytes())


def reference_losses():
    return np.load(os.path.join(GOLDEN, "reference_losses.npz"))


def hardest_inputs():
    g = torch.Generator().manual_seed(0)
    N0, N1, P = 700, 650, 3000
    F0 = torch.nn.functional.normalize(torch.randn(N0, 32, generator=g, dtype=torch.float64), dim=1)
    F1 = torch.nn.functional.normalize(torch.randn(N1, 32, generator=g, dtype=torch.float64), dim=1)
    F1[:300] = F0[:300] + 0.05 * torch.randn(300, 32, generator=g, dtype=torch.float64)
    rng = np.random.default_rng(0)
    i0 = np.sort(rng.integers(0, 300, P))
    pairs = np.stack([i0, np.clip(i0 + rng.integers(-1, 2, P), 0, N1 - 1)], 1)
    return F0, F1, pairs


class Net(torch.nn.Module):                      # stand-in for Res16UNet: per-row features from (feats, coords)
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.lin = torch.nn.Linear(7, 32).double()

    def forward(self, s):
        x = torch.cat([s.F.double(), torch.sin(s.C.double() * 0.37)], 1)
        return types.SimpleNamespace(F=torch.nn.functional.normalize(self.lin(x), dim=1))


def nce_inputs():
    from pointcontrast_b200 import synth
    batch = synth.collate_pairs([synth.synth_pair(3, scale=0.1), synth.synth_pair(4, scale=0.1)])
    inp = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in batch.items()}
    inp["pcd0"], inp["pcd1"] = inp["sinput0_C"], inp["sinput1_C"]                  # only .shape[0] is read (`:400`)
    return inp, batch


def test_reference_res16unet34c_builds_on_oracle():
    """The original's Res16UNet34C (stored structure) has the expected shape, and this repository's model file built on the
    oracle has exactly that structure."""
    from tests.helpers import model_backend
    ref = reference_structure()
    assert ref["n_params"] == 37_847_808
    kinds = [m["kind"] for m in ref["modules"]]
    assert (kinds.count("conv"), kinds.count("transpose"), kinds.count("bn")) == (59, 4, 62)
    moms = sorted(m["momentum"] for m in ref["modules"] if m["kind"] == "bn")
    assert moms.count(0.1) == 46 and moms.count(0.05) == 16          # SURVEY 8a row B1
    sd = {k: tuple(s) for k, s in ref["state_dict"]}
    assert sd["conv0p1s1.kernel"] == (27, 3, 32)
    assert sd["final.kernel"] == (1, 96, 32) and sd["final.bias"] == (1, 32)
    assert sd["block2.0.downsample.0.kernel"] == (1, 32, 64)
    assert "bn0.bn.running_mean" in sd and "block8.1.norm2.bn.weight" in sd
    with model_backend(me_cpu) as mod:
        net = mod.Res16UNet34C(3, 32, refload.default_config(), D=3)
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref["state_dict"]


def test_hardest_loss_oracle_matches_reference_function():
    gold = reference_losses()
    F0, F1, pairs = hardest_inputs()
    N0, N1, P = len(F0), len(F1), len(pairs)
    for num_pos in HARDEST_NUM_POS:
        ref_pos, ref_neg = gold[f"hardest_{num_pos}"]
        np.random.seed(7)
        sel0 = np.random.choice(N0, 256, replace=False)
        sel1 = np.random.choice(N1, 256, replace=False)
        pos_sel = np.random.choice(P, num_pos, replace=False) if P > num_pos else None
        pos, neg = loss_cpu.hardest_contrastive_loss(F0, F1, pairs, sel0, sel1, pos_sel)
        assert abs(float(pos) - ref_pos) <= 1e-12 * abs(ref_pos) and abs(float(neg) - ref_neg) <= 1e-12 * abs(ref_neg)


def test_point_nce_oracle_matches_reference_train_iter():
    """Rows L1 + L2: the original's `PointNCELossTrainer._train_iter` (`lib/ddp_trainer.py:380-440`, `NCESoftmaxLoss` from
    `lib/criterion.py`), run on the CPU with a small stand-in model (stored loss and gradient), against
    `loss_cpu.select_positives` + `point_nce_loss` fed with the same RNG draws."""
    gold = reference_losses()
    inp, batch = nce_inputs()
    nq = len(np.unique(batch["correspondences"][:, 0]))
    for npos in NCE_NPOS:
        ref_loss, ref_grad = float(gold[f"nce_loss_{npos}"]), torch.from_numpy(gold[f"nce_grad_{npos}"])
        torch.manual_seed(11); np.random.seed(12)
        uniform = torch.distributions.Uniform(0, 1).sample([nq])
        sampled = np.random.choice(nq, npos, replace=False) if npos < nq else None
        net2 = Net()
        F0 = net2(me_cpu.SparseTensor(inp["sinput0_F"], coords=inp["sinput0_C"])).F
        F1 = net2(me_cpu.SparseTensor(inp["sinput1_F"], coords=inp["sinput1_C"])).F
        q, k = loss_cpu.select_positives(batch["correspondences"], uniform, npos, sampled)
        assert len(q) == min(npos, nq)
        loss = loss_cpu.point_nce_loss(F0, F1, q, k, 0.4)
        loss.backward()
        assert abs(float(loss) - ref_loss) < 1e-12 * abs(ref_loss), (float(loss), ref_loss)
        assert torch.allclose(net2.lin.weight.grad, ref_grad, rtol=1e-10, atol=1e-14)
