"""Generates tests/golden/loss_curve_100.npz  (~6 minutes of CPU):

    python tests/golden/make_loss_curve.py

100 SGD steps (lr 0.1, momentum 0.8, wd 1e-4, ExponentialLR 0.99 per step, PointInfoNCE T = 0.4) of Res16UNet34C on two small
synthetic scene-pair batches, on the CPU oracle (oracle/me_cpu.py + oracle/loss_cpu.py) in fp64 and in fp32, with deterministic
weights (tests/helpers.det_init seed 11) and positive draws from numpy default_rng(5).  Stored: both loss curves.
tests/test_gpu_trainer.py::test_loss_curve_100_steps replays the same steps on the GPU and compares."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import loss_cpu, me_cpu as OR            # noqa: E402
from pointcontrast_b200 import synth                 # noqa: E402
from tests import refload                            # noqa: E402
from tests.helpers import det_init, model_backend    # noqa: E402

STEPS, SEEDS, SCALE, INIT_SEED, DRAW_SEED = 100, (60, 61, 62, 63), 0.12, 11, 5


def setup():
    batches = [synth.collate_pairs([synth.synth_pair(SEEDS[2 * s], scale=SCALE), synth.synth_pair(SEEDS[2 * s + 1], scale=SCALE)]) for s in range(2)]
    rng = np.random.default_rng(DRAW_SEED)
    draws = []
    for step in range(STEPS):
        pairs = batches[step % 2]["correspondences"]
        nq = len(np.unique(pairs[:, 0]))
        draws.append(loss_cpu.select_positives(pairs, rng.random(nq).astype(np.float32), 4096, rng.choice(nq, 4096, replace=False) if nq > 4096 else None))
    return batches, draws


def run_oracle(batches, draws, state, dtype):
    cfg = refload.default_config()
    with model_backend(OR) as mod:
        onet = mod.Res16UNet34C(3, 32, cfg, D=3).to(dtype)
        onet.load_state_dict({k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in state.items()})
        onet.train()
        oopt = torch.optim.SGD(onet.parameters(), lr=0.1, momentum=0.8, weight_decay=1e-4)
        sch = torch.optim.lr_scheduler.ExponentialLR(oopt, 0.99)
        inputs = [[OR.SparseTensor(torch.from_numpy(b[f"sinput{v}_F"]).to(dtype), coords=torch.from_numpy(b[f"sinput{v}_C"])) for v in "01"] for b in batches]
        curve = []
        for step in range(STEPS):
            q, k = draws[step]
            oopt.zero_grad()
            Fo = [onet(OR.SparseTensor(s.F, coords_key=s.coords_key, coords_manager=s.coords_man)).F for s in inputs[step % 2]]
            lo = loss_cpu.point_nce_loss(Fo[0], Fo[1], q, k, 0.4)
            lo.backward(); oopt.step(); sch.step()
            curve.append(float(lo.detach()))
            if step % 10 == 0:
                print(dtype, step, curve[-1], flush=True)
    return curve


def main():
    torch.set_num_threads(min(os.cpu_count() or 1, 16))
    from pointcontrast_b200.model import load_model
    net = load_model("Res16UNet34C")(3, 32, refload.default_config(), D=3)
    det_init(net, INIT_SEED)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    batches, draws = setup()
    c64 = run_oracle(batches, draws, state, torch.float64)
    c32 = run_oracle(batches, draws, state, torch.float32)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loss_curve_100.npz")
    np.savez_compressed(out, oracle_fp64=np.array(c64), oracle_fp32=np.array(c32), steps=STEPS, seeds=np.array(SEEDS), scale=SCALE,
                        init_seed=INIT_SEED, draw_seed=DRAW_SEED)
    print("wrote", out)


if __name__ == "__main__":
    main()
