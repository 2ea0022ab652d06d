"""Writes tests/golden/detection_loss.npz from the original VoteNet criterion, run unmodified on the CPU in fp64:

    python tests/golden/make_detection_loss_golden.py <root>      (<root>: the original repository)

Loads `models/loss_helper.py` (with `lib/utils/nn_distance.py`) by path.  The original calls `.cuda()` and `torch.cuda.FloatTensor`;
here `.cuda()` returns the tensor itself, `torch.cuda.FloatTensor(*shape)` is `torch.zeros(*shape)`, and the default dtype is float64,
so `torch.Tensor(OBJECTNESS_CLS_WEIGHTS)`, `torch.zeros` and the one-hot buffers are fp64 as well.  Every input is fp64 (mean_size_arr
as the original rounds it, through fp32).  Autograd of `loss` gives the gradients of the nine differentiable inputs.

Cases: ScanNet (NH 1, NS 18, C 18) and SUN RGB-D (NH 12, NS 10, C 10) shapes, vote_factor 1 and 3, each a small seeded batch of
`synth.synth_votenet_loss_batch` (2 scenes, 16 seeds, 24 proposals, 16 label slots) with planted cases in scene 0:
  * proposal 0 exactly equidistant (squared distance 1/16) to label slots 0 and 1: the argmin tie goes to slot 0;
  * seed 0 exactly equidistant in L1 (1/4) to two different GT votes; seed 1's vote exactly on its first GT vote (zero |x|' );
  * proposal 1 near the origin, so assigned to a padded zero slot; proposals 2 and 3 in the gray zone (0.45 from a box);
and scene 1 with no positive proposal (every proposal more than 0.6 from every slot), so its label sums are 0 and the 1e-6 terms count.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "detection_loss.npz")
ROOT = os.path.dirname(os.path.dirname(HERE))
DATASETS = {"scannet": (1, 18, 18), "sunrgbd": (12, 10, 10)}        # NH, NS, C
GRAD_INPUTS = ("vote_xyz", "seed_xyz", "center", "objectness_scores", "heading_scores", "heading_residuals_normalized", "size_scores",
               "size_residuals_normalized", "sem_cls_scores")
OUTPUTS = ("vote_loss", "objectness_loss", "center_loss", "heading_cls_loss", "heading_reg_loss", "size_cls_loss", "size_reg_loss",
           "sem_cls_loss", "box_loss", "loss", "pos_ratio", "neg_ratio", "obj_acc")


def case(dname, V, seed):
    """The numpy end_points of one case (fp32 / int as the dataset and network give them), planted as the module docstring says."""
    sys.path.insert(0, ROOT)
    from pointcontrast_b200 import synth
    NH, NS, C = DATASETS[dname]
    rng = np.random.default_rng(seed)
    mean_size = rng.uniform(0.3, 2.0, (NS, 3))
    ep = synth.synth_votenet_loss_batch(seed, 2, 2000, 16, 24, V, NH, mean_size, C, max_obj=16)
    # scene 0: slots 0 / 1 at dyadic centres, proposal 0 halfway between them
    ep["center_label"][0, 0] = (1.0, 1.0, 0.5)
    ep["center_label"][0, 1] = (1.5, 1.0, 0.5)
    ep["box_label_mask"][0, :2] = 1
    for j in range(2, ep["center_label"].shape[1]):                    # keep every other box clear of the planted proposals
        if np.abs(ep["center_label"][0, j] - (1.25, 1.0, 0.5)).max() < 1.5 and ep["box_label_mask"][0, j]:
            ep["center_label"][0, j, 0] += 3.0
    ep["aggregated_vote_xyz"][0, 0] = (1.25, 1.0, 0.5)
    ep["aggregated_vote_xyz"][0, 1] = (0.03125, 0.0, 0.0)
    ep["aggregated_vote_xyz"][0, 2] = (1.0 - 0.45, 1.0, 0.5)
    ep["aggregated_vote_xyz"][0, 3] = (1.5 + 0.45, 1.0, 0.5)
    # seeds 0 and 1: dyadic points with dyadic votes
    i0, i1 = ep["seed_inds"][0, 0], ep["seed_inds"][0, 1]
    for i, p in ((i0, (1.0, 2.0, 0.5)), (i1, (2.0, 1.0, 0.25))):
        ep["point_clouds"][0, i] = p
        ep["vote_label_mask"][0, i] = 1
    ep["vote_label"][0, i0] = (0.25, 0, 0, -0.25, 0, 0, 0.25, 0, 0)
    ep["vote_label"][0, i1] = (0.5, 0.25, 0, 0.5, 0.25, 0, 0.5, 0.25, 0)
    ep["seed_xyz"][0, 0] = ep["point_clouds"][0, i0]
    ep["seed_xyz"][0, 1] = ep["point_clouds"][0, i1]
    ep["vote_xyz"][0, 0:V] = ep["seed_xyz"][0, 0]                        # L1 1/4 to GT votes 0 and 1
    ep["vote_xyz"][0, V:2 * V] = ep["seed_xyz"][0, 1] + 0.125
    ep["vote_xyz"][0, V] = ep["seed_xyz"][0, 1] + np.float32([0.5, 0.25, 0])   # exactly on GT vote 0
    # scene 1: no positive proposal -- every proposal far from every slot (padded slots included)
    slots = ep["center_label"][1][:, None, :]
    far = ep["aggregated_vote_xyz"][1]
    for k in range(far.shape[0]):
        while np.sqrt(((far[k] - slots[:, 0]) ** 2).sum(-1)).min() <= 0.7:
            far[k] = rng.uniform(-3, 3, 3).astype(np.float32)
    return ep, mean_size


def load(root):
    base = os.path.join(root, "downstream", "votenet_det_new")
    sys.path[:0] = [base]
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.cuda.FloatTensor = lambda *shape: torch.zeros(*shape)
    torch.set_default_dtype(torch.float64)
    from models import loss_helper
    return loss_helper


class Config:
    def __init__(self, NH, NS, C, mean_size):
        self.num_heading_bin, self.num_size_cluster, self.num_class, self.mean_size_arr = NH, NS, C, mean_size


def run(loss_helper, ep, mean_size, dname):
    NH, NS, C = DATASETS[dname]
    t = {}
    for k, v in ep.items():
        t[k] = torch.from_numpy(np.asarray(v, np.float64) if v.dtype == np.float32 else v.astype(np.int64))
        if k in GRAD_INPUTS:
            t[k].requires_grad_(True)
    loss, out = loss_helper.get_loss(dict(t), Config(NH, NS, C, mean_size))
    loss.backward()
    res = {k: float(out[k]) for k in OUTPUTS}
    res.update({k: out[k].detach().numpy() for k in ("objectness_label", "objectness_mask", "object_assignment")})
    res.update({"grad_" + k: t[k].grad.numpy() for k in GRAD_INPUTS})
    return res


def main(root):
    loss_helper = load(root)
    z = {}
    for n, (dname, V) in enumerate((d, V) for d in DATASETS for V in (1, 3)):
        ep, mean_size = case(dname, V, 100 + n)
        name = f"{dname}_v{V}"
        res = run(loss_helper, ep, mean_size, dname)
        assert res["object_assignment"][0, 0] == 0 and res["objectness_label"][0, 0] == 1
        assert res["object_assignment"][0, 1] >= ep["box_label_mask"][0].sum()
        assert res["objectness_mask"][0, 2] == 0 and res["objectness_mask"][0, 3] == 0
        assert res["objectness_label"][1].sum() == 0
        for k, v in ep.items():
            if k != "point_clouds":                                      # the criterion does not read it
                z[f"{name}/in/{k}"] = v
        z[f"{name}/mean_size"] = mean_size
        for k, v in res.items():
            z[f"{name}/out/{k}"] = np.asarray(v)
        print(name, {k: round(res[k], 6) for k in OUTPUTS})
    np.savez_compressed(OUT, **z)
    print("wrote", OUT)


if __name__ == "__main__":
    main(sys.argv[1])
