"""Which term sets the whole-network gradient error of the tensor-core path?

Runs the MODULAR path (one autograd node per op, `me.SIMT_OPS` selects per op class the exact-fp32 SIMT kernel instead of
the bf16x3-split tensor-core kernel) on small scene pairs and reports, per variant, the relative error of every parameter
gradient against the fp64 oracle (median / max over the 187 parameters) next to the plain-fp32 CPU floor.

    python profiles/grad_precision_ab.py [scale] > grad_precision_ab.json

Variants: all tensor-core | forward exact | data-gradient exact | weight-gradient exact | fwd+dgrad exact | all exact |
all tensor-core with ATen's BatchNorm (fp32, Welford) in place of bn.cu (E[x^2]-E[x]^2 in fp32 chunks + fp64 finalize).
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import loss_cpu, me_cpu as OR            # noqa: E402   (checker only)
from tests import refload                            # noqa: E402
from tests.helpers import det_init, model_backend, rel_err     # noqa: E402


def main():
    from pointcontrast_b200 import fused, losses, me, synth
    from pointcontrast_b200.model import load_model
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 0.15
    batch = synth.collate_pairs([synth.synth_pair(3, scale=scale), synth.synth_pair(4, scale=scale * 0.9)])
    cfg = refload.default_config()
    net0 = load_model("Res16UNet34C")(3, 32, cfg, D=3)
    det_init(net0, 1)
    state = {k: v.clone() for k, v in net0.state_dict().items()}
    rng = np.random.default_rng(0)
    pairs = batch["correspondences"]
    nq = len(np.unique(pairs[:, 0]))
    q, k = loss_cpu.select_positives(pairs, rng.random(nq).astype(np.float32), 4096, rng.choice(nq, 4096, replace=False) if nq > 4096 else None)

    def oracle(dtype):
        with model_backend(OR) as mod:
            onet = mod.Res16UNet34C(3, 32, cfg, D=3).to(dtype)
            onet.load_state_dict({kk: (v.to(dtype) if v.dtype.is_floating_point else v) for kk, v in state.items()})
            onet.train()
            Fo = [onet(OR.SparseTensor(torch.from_numpy(batch[f"sinput{v}_F"]).to(dtype), coords=torch.from_numpy(batch[f"sinput{v}_C"]))).F for v in "01"]
        loss_cpu.point_nce_loss(Fo[0], Fo[1], q, k, 0.4).backward()
        return [p.grad.clone() for p in onet.parameters()], [f.detach() for f in Fo]

    g64, F64 = oracle(torch.float64)
    g32, _ = oracle(torch.float32)
    names = [n for n, _ in net0.named_parameters()]
    floor = np.array([rel_err(a, b) for a, b in zip(g32, g64)])
    out = {"rows": [len(batch["sinput0_C"]), len(batch["sinput1_C"])], "fp32_cpu_floor": {"median": float(np.median(floor)), "max": float(floor.max())},
           "variants": {}}

    def run(tag, simt_ops, aten_bn=False, use_fused=False, fp16=False):
        net = load_model("Res16UNet34C")(3, 32, cfg, D=3)
        net.load_state_dict(state)
        net = net.cuda().train()
        me.SIMT_OPS = set(simt_ops)
        fused.ENABLED = use_fused
        saved_fmt, me.FWD_FP16 = me.FWD_FP16, fp16
        old_fwd = me.MinkowskiBatchNorm.forward
        if aten_bn:
            def fwd(self, inp):
                return me.SparseTensor(self.bn(inp.F), coords_key=inp.coords_key, coords_manager=inp.coords_man)
            me.MinkowskiBatchNorm.forward = fwd
        try:
            F = [net(me.SparseTensor(torch.from_numpy(batch[f"sinput{v}_F"]), coords=torch.from_numpy(batch[f"sinput{v}_C"])).to("cuda")).F for v in "01"]
            losses.point_nce_loss(F[0], F[1], q.cuda(), k.cuda(), 0.4).backward()
        finally:
            me.SIMT_OPS = set(); fused.ENABLED = True; me.MinkowskiBatchNorm.forward = old_fwd; me.FWD_FP16 = saved_fmt
        err = np.array([rel_err(p.grad, g) for p, g in zip(net.parameters(), g64)])
        ferr = max(float((F[i].detach().double().cpu() - F64[i]).abs().max() / F64[i].pow(2).mean().sqrt()) for i in range(2))
        w = int(np.argmax(err))
        out["variants"][tag] = {"grad_err_median": float(np.median(err)), "grad_err_max": float(err.max()), "worst": names[w], "feature_err": ferr}
        print(tag, out["variants"][tag], file=sys.stderr, flush=True)

    run("tensor-core fwd+dgrad+wgrad (modular)", [])
    run("fused executor, bf16 hi/lo planes everywhere", [], use_fused=True)
    run("fused executor, fp16 hi/lo activations + forward weights (default)", [], use_fused=True, fp16=True)
    run("exact fwd", ["fwd"])
    run("exact dgrad", ["dgrad"])
    run("exact wgrad", ["wgrad"])
    run("exact fwd+dgrad", ["fwd", "dgrad"])
    run("exact dgrad+wgrad", ["dgrad", "wgrad"])
    run("exact all", ["fwd", "dgrad", "wgrad"])
    run("tensor-core, ATen BatchNorm", [], aten_bn=True)
    run("exact all, ATen BatchNorm", ["fwd", "dgrad", "wgrad"], aten_bn=True)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
