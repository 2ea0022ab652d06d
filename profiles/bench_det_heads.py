"""VoteNet's voting module and proposal head on the library (det_heads, DESIGN.md 8f-18) against the original's torch modules, timed as
the other profiles time (CUDA events, warmed, windows >= 1 s, the routes alternating, the smaller of two rounds):
  * each head's forward + backward at the training scripts' sizes (ScanNet B = 32, SUN RGB-D B = 64; 1024 seeds, 256 proposals), the
    proposal head after its vote aggregation (a stand-in returns the aggregated xyz and features, so both routes time the same layers);
    the original at torch's defaults (TF32 on in cuDNN, what users get) and with TF32 off;
  * a whole VoteNet training step (unmodified votenet.py, sparse-conv backbone, det_loss, forward + backward) with and without
    det_heads.install(), everything else on the library in both;
  * the heads' outputs of both routes at the timed size (same weights, TF32 off): the largest difference over the largest value.
The original modules are the ones __graft_entry__.build() staged under oracle/_ref/votenet/models.  Prints one JSON line with the GPU
name and power limit read in the same call.

    python profiles/bench_det_heads.py
"""
import importlib
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointcontrast_b200 import det_heads, det_loss, detection, me, pointnet2, pointnet2_modules, synth  # noqa: E402
from oracle import stage_ref  # noqa: E402
from profiles.bench_pointnet2 import gpu_info, time_ms  # noqa: E402

# name: (NH, NS, C, scenes per batch, points per scene) -- train_scannet.sh / train_sunrgbd.sh
DATASETS = {"scannet": (1, 18, 18, 32, 40000), "sunrgbd": (12, 10, 10, 64, 20000)}
S, K = 1024, 256


def load_votenet(ours):
    """The staged models/votenet.py (fresh import) on the library's me, PointNet++ operators and modules and det_loss; det_heads as
    its heads when `ours`, the original voting_module.py / proposal_module.py otherwise."""
    if not stage_ref.available("votenet"):
        raise SystemExit("the original is not staged under oracle/_ref/votenet (run __graft_entry__.build())")
    try:                      # the original's plotting helpers import cv2 and never call it here
        importlib.import_module("cv2")
    except Exception:
        sys.modules["cv2"] = types.ModuleType("cv2")
    from oracle import det_eval_ref
    det_eval_ref.load()
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k in (
            "pointnet2_utils", "pointnet2_modules", "pytorch_utils", "backbone_module", "proposal_module", "voting_module", "loss_helper",
            "dump_helper")]:
        del sys.modules[k]
    me.install()
    pointnet2.install()
    for p in (stage_ref.path("votenet"), stage_ref.path("votenet", "models", "backbone", "pointnet2")):   # pointnet2_utils' imports
        if p not in sys.path:
            sys.path.insert(0, p)
    pointnet2_modules.install()
    if ours:
        det_heads.install()
    det_loss.install()
    return importlib.import_module("models.votenet"), importlib.import_module("voting_module"), importlib.import_module("proposal_module")


class _Aggregation(torch.nn.Module):
    def __init__(self, out):
        super().__init__()
        self.out = out

    def forward(self, *args):
        return self.out


def routes(fn_ours, fn_ref):
    """Mean ms of ours, the original with TF32 on and with TF32 off, alternating over two rounds (the smaller of each)."""
    res = {"ours": [], "original_tf32": [], "original_fp32": []}
    for _ in range(2):
        res["ours"].append(time_ms(fn_ours))
        for name, on in (("original_tf32", True), ("original_fp32", False)):
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
            res[name].append(time_ms(fn_ref))
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, True          # torch's defaults
    return {k: round(min(v), 3) for k, v in res.items()}


def max_rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def bench_heads(vm, pm):
    out = {}
    for name, (NH, NS, C, B, _) in DATASETS.items():
        ms = np.random.default_rng(0).uniform(0.3, 2.0, (NS, 3))
        g = torch.Generator(device="cuda").manual_seed(1)
        xyz = torch.rand(B, S, 3, device="cuda", generator=g) * 6 - 3
        f = torch.randn(B, S, 256, device="cuda", generator=g).transpose(1, 2).requires_grad_()     # point-major, as the backbones give
        a, b = vm.VotingModule(1, 256).cuda().train(), det_heads.VotingModule(1, 256).cuda().train()
        b.load_state_dict(a.state_dict())

        def vote(mod):
            def run():
                mod.zero_grad(set_to_none=True)
                vx, vf = mod(xyz, f)
                (vx.square().sum() + vf.square().sum()).backward()
            return run
        res = {"voting": routes(vote(b), vote(a))}
        agg = (torch.rand(B, K, 3, device="cuda", generator=g) * 6 - 3).requires_grad_()
        af = torch.relu(torch.randn(B, K, 128, device="cuda", generator=g)).transpose(1, 2).requires_grad_()
        stand_in = _Aggregation((agg, af, torch.zeros(B, K, dtype=torch.int32, device="cuda")))
        pa = pm.ProposalModule(C, NH, NS, ms, K, "vote_fps").cuda().train()
        pb = det_heads.ProposalModule(C, NH, NS, ms, K, "vote_fps").cuda().train()
        pb.load_state_dict(pa.state_dict())
        pa.vote_aggregation = pb.vote_aggregation = stand_in

        def prop(mod):
            def run():
                mod.zero_grad(set_to_none=True)
                ep = mod(None, None, {})
                sum(ep[k].square().sum() for k in det_heads.DECODE).backward()
            return run
        res["proposal"] = routes(prop(pb), prop(pa))
        # agreement at the timed size: one training-mode forward each from the same weights and statistics, TF32 off
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        a2, b2 = vm.VotingModule(1, 256).cuda().train(), det_heads.VotingModule(1, 256).cuda().train()
        b2.load_state_dict(a2.state_dict())
        pa2 = pm.ProposalModule(C, NH, NS, ms, K, "vote_fps").cuda().train()
        pb2 = det_heads.ProposalModule(C, NH, NS, ms, K, "vote_fps").cuda().train()
        pb2.load_state_dict(pa2.state_dict())
        pa2.vote_aggregation = pb2.vote_aggregation = stand_in
        with torch.no_grad():
            va, vb = a2(xyz, f), b2(xyz, f)
            ea, eb = pa2(None, None, {}), pb2(None, None, {})
        res["max_rel_diff"] = {"vote_xyz": max_rel(vb[0], va[0]), "vote_features": max_rel(vb[1], va[1]),
                               **{k: max_rel(eb[k], ea[k]) for k in det_heads.DECODE}}
        torch.backends.cudnn.allow_tf32 = True
        out[name] = res
    return out


def bench_votenet():
    """A training step of the unmodified VoteNet (sparse-conv backbone, det_loss) at each script's shape, with the original heads and
    with det_heads.install(); cuDNN at torch's defaults."""
    labels = ("center_label", "heading_class_label", "heading_residual_label", "size_class_label", "size_residual_label", "sem_cls_label",
              "box_label_mask", "vote_label", "vote_label_mask")
    out = {}
    for name, (NH, NS, C, B, N) in DATASETS.items():
        ms = np.random.default_rng(6).uniform(0.3, 2.0, (NS, 3))
        cfg = type("Cfg", (), dict(num_heading_bin=NH, num_size_cluster=NS, num_class=C, mean_size_arr=ms))()
        ep = synth.synth_votenet_loss_batch(41, B, N, S, K, 1, NH, ms, C)
        pts = torch.from_numpy(ep["point_clouds"]).cuda()
        b = detection.voxelize_batch({"point_clouds": pts}, 0.025)
        inputs = {k: b[k] for k in ("point_clouds", "voxel_coords", "voxel_inds", "voxel_feats")}
        lab = {k: torch.from_numpy(ep[k]).cuda() for k in labels}
        steps, nets = {}, {}
        for ours in (False, True):
            votenet = load_votenet(ours)[0]
            torch.manual_seed(0)
            net = votenet.VoteNet(C, NH, NS, ms, input_feature_dim=0, num_proposal=K, vote_factor=1, sampling="seed_fps",
                                  backbone="sparseconv").cuda().train()
            nets[ours] = net

            def step(net=net):
                net.zero_grad(set_to_none=True)
                end_points = net(dict(inputs))
                end_points.update(lab)
                loss, _ = det_loss.get_loss(end_points, cfg)
                loss.backward()
            steps[ours] = step
        nets[True].load_state_dict(nets[False].state_dict())
        res = {"ours": [], "original_heads": []}
        for _ in range(2):
            res["ours"].append(time_ms(steps[True]))
            res["original_heads"].append(time_ms(steps[False]))
        out[name] = {k: round(min(v), 2) for k, v in res.items()}
        out[name]["voxels"] = int(inputs["voxel_coords"].shape[0])
    return out


def main():
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    _, vm, pm = load_votenet(False)
    result = {"gpu": gpu_info(), "unit": "ms per forward + backward (min of two alternating rounds)", "heads": bench_heads(vm, pm),
              "votenet_step_sparseconv": bench_votenet()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
