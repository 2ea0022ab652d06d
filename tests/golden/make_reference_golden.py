"""Generates tests/golden/reference_model_structure.npz and tests/golden/reference_losses.npz from the original PointContrast
code (its `pretrain/pointcontrast` tree, imported unmodified on top of the CPU oracle):

    python tests/golden/make_reference_golden.py /path/to/PointContrast

Stored: the original Res16UNet34C's structure (state-dict shapes, convolution offsets / stride / bias, BatchNorm momentum / eps)
and the outputs of its `contrastive_hardest_negative_loss` and `PointNCELossTrainer._train_iter` on the seeded inputs of
tests/test_oracle_reference.py.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import me_cpu                      # noqa: E402
from tests import refload                      # noqa: E402
from tests import test_oracle_reference as T   # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def structure(pkg):
    net = pkg.load_model("Res16UNet34C")(3, 32, refload.default_config(), D=3)
    mods = []
    for name, m in net.named_modules():
        if isinstance(m, (me_cpu.MinkowskiConvolution, me_cpu.MinkowskiConvolutionTranspose)):
            mods.append(dict(name=name, kind="transpose" if isinstance(m, me_cpu.MinkowskiConvolutionTranspose) else "conv",
                             offsets=np.asarray(m.kernel_generator.offsets).tolist(), stride=list(m.stride), has_bias=bool(m.has_bias)))
        elif isinstance(m, me_cpu.MinkowskiBatchNorm):
            mods.append(dict(name=name, kind="bn", momentum=m.bn.momentum, eps=m.bn.eps))
        else:
            mods.append(dict(name=name, kind="other"))
    return dict(state_dict=[[k, list(v.shape)] for k, v in net.state_dict().items()], modules=mods,
                n_params=sum(p.numel() for p in net.parameters()))


def main(ref_root):
    refload.REF_PC = os.path.join(os.path.abspath(ref_root), "pretrain", "pointcontrast")
    assert refload.available(), refload.REF_PC
    st = structure(refload.load_reference_model_module(me_cpu.install))
    np.savez_compressed(os.path.join(HERE, "reference_model_structure.npz"),      # the structure as JSON bytes
                        json=np.frombuffer(json.dumps(st, separators=(",", ":")).encode(), dtype=np.uint8))
    tr = refload.load_reference_trainer_module(me_cpu.install)
    out = {}
    obj = tr.HardestContrastiveLossTrainer.__new__(tr.HardestContrastiveLossTrainer)
    obj.pos_thresh, obj.neg_thresh = 0.1, 1.4
    F0, F1, pairs = T.hardest_inputs()
    for num_pos in T.HARDEST_NUM_POS:
        np.random.seed(7)
        pos, neg = obj.contrastive_hardest_negative_loss(F0, F1, torch.from_numpy(pairs), num_pos=num_pos, num_hn_samples=256)
        out[f"hardest_{num_pos}"] = np.array([float(pos), float(neg)])
    torch.Tensor.cuda = lambda self, *a, **k: self           # the original's hard-coded .cuda() calls, on the CPU
    torch.nn.Module.cuda = lambda self, *a, **k: self
    inp = T.nce_inputs()[0]

    class It:
        def next(self):
            return inp

    import types
    for npos in T.NCE_NPOS:
        net = T.Net()
        obj = tr.PointNCELossTrainer.__new__(tr.PointNCELossTrainer)
        obj.model, obj.cur_device, obj.T, obj.npos = net, "cpu", 0.4, npos
        obj.optimizer = types.SimpleNamespace(zero_grad=lambda: None, step=lambda: None)
        obj.config = refload.Cfg(misc=dict(num_gpus=1))
        torch.manual_seed(11); np.random.seed(12)
        out[f"nce_loss_{npos}"] = np.float64(obj._train_iter(It(), [tr.AverageMeter(), tr.Timer(), tr.Timer()]))
        out[f"nce_grad_{npos}"] = net.lin.weight.grad.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "reference_losses.npz"), **out)
    print("wrote", sorted(out), "n_params", st["n_params"])


if __name__ == "__main__":
    main(sys.argv[1])
