"""fp64 torch-CPU restatement of VoteNet's voting module and proposal head (`models/voting_module.py` VotingModule,
`models/proposal_module.py` ProposalModule's layers after the vote aggregation, and decode_scores), the checker of
pointcontrast_b200/det_heads.py.  Gradients come from autograd in fp64.

Each head is conv1 -> BatchNorm -> ReLU, conv2 -> BatchNorm -> ReLU, conv3 (1x1 convolutions with bias) over point-major rows, BatchNorm
over all rows (biased variance to normalise, unbiased into the running statistics).  Then:
  * voting: vote_xyz[b, s V + v] = seed_xyz[b, s] + z[b S + s, v (3 + C) : v (3 + C) + 3], vote_features = seed features + the rest;
  * decode_scores: the column slices of z, center = aggregated_vote_xyz + z[2:5], heading_residuals = heading_residuals_normalized *
    pi / NH, size_residuals = size_residuals_normalized * mean_size (rounded to fp32, as the original takes it).
"""
import numpy as np
import torch

from oracle.pointnet2_mlp_cpu import _bn

D = torch.float64
DECODE = ("objectness_scores", "center", "heading_scores", "heading_residuals_normalized", "heading_residuals", "size_scores",
          "size_residuals_normalized", "size_residuals", "sem_cls_scores")


def head_params(sd, prefix=""):
    """{conv1, conv2, conv3: {W [Cout, Cin], b}, bn1, bn2: {weight, bias, running_mean, running_var}} in fp64 (the weights and biases as
    leaves requiring grad) from a head's state_dict."""
    g = lambda k: sd[prefix + k].detach().cpu().to(D).clone()             # noqa: E731
    p = {}
    for c in ("conv1", "conv2", "conv3"):
        p[c] = dict(W=g(c + ".weight").flatten(1).requires_grad_(), b=g(c + ".bias").requires_grad_())
    for c in ("bn1", "bn2"):
        p[c] = dict(weight=g(c + ".weight").requires_grad_(), bias=g(c + ".bias").requires_grad_(), running_mean=g(c + ".running_mean"),
                    running_var=g(c + ".running_var"))
    return p


def grads(p):
    """The parameter gradients in the modules' registration order: conv1 (weight, bias), conv2, conv3, bn1 (weight, bias), bn2."""
    return [p[c][k].grad for c in ("conv1", "conv2", "conv3") for k in ("W", "b")] + \
        [p[c][k].grad for c in ("bn1", "bn2") for k in ("weight", "bias")]


def layers(x, p, train, momentum=0.1, eps=1e-5):
    """x fp64 [n, Cin] -> z [n, Cout3] of conv1/bn1/relu, conv2/bn2/relu, conv3; updates the running statistics in training."""
    for c, bn in (("conv1", "bn1"), ("conv2", "bn2")):
        x = torch.relu(_bn(x @ p[c]["W"].T + p[c]["b"], p[bn], train, momentum, eps, (0,)))
    return x @ p["conv3"]["W"].T + p["conv3"]["b"]


def voting(seed_xyz, seed_features, p, vote_factor, train, momentum=0.1):
    """seed_xyz [B, S, 3], seed_features [B, C, S] -> (vote_xyz [B, S V, 3], vote_features [B, C, S V])."""
    B, S, _ = seed_xyz.shape
    C, V = seed_features.shape[1], vote_factor
    X = seed_features.transpose(1, 2).reshape(B * S, C)
    z = layers(X, p, train, momentum).view(B, S, V, 3 + C)
    vote_xyz = (seed_xyz[:, :, None] + z[..., :3]).reshape(B, S * V, 3)
    vote_features = (X.view(B, S, 1, C) + z[..., 3:]).reshape(B, S * V, C).transpose(1, 2)
    return vote_xyz, vote_features


def decode(z, agg, NH, NS, mean_size):
    """z [B, K, X] (decode_scores' net_transposed), aggregated_vote_xyz [B, K, 3] -> {name: tensor} of the nine end_points."""
    B, K, _ = z.shape
    s0 = 5 + 2 * NH
    c0 = s0 + 4 * NS
    hrn = z[:, :, 5 + NH:s0]
    srn = z[:, :, s0 + NS:c0].reshape(B, K, NS, 3)
    out = dict(objectness_scores=z[:, :, 0:2], center=agg + z[:, :, 2:5], heading_scores=z[:, :, 5:5 + NH],
               heading_residuals_normalized=hrn, heading_residuals=hrn * (np.pi / NH), size_scores=z[:, :, s0:s0 + NS],
               size_residuals_normalized=srn, size_residuals=srn * torch.as_tensor(np.asarray(mean_size, np.float32)).to(z.dtype),
               sem_cls_scores=z[:, :, c0:])
    return {k: out[k] for k in DECODE}


def proposal(agg, features, p, NH, NS, mean_size, train, momentum=0.1):
    """The proposal head after the vote aggregation: aggregated_vote_xyz [B, K, 3], features [B, 128, K] -> decode()'s end_points."""
    B, C, K = features.shape
    z = layers(features.transpose(1, 2).reshape(B * K, C), p, train, momentum).view(B, K, -1)
    return decode(z, agg, NH, NS, mean_size)
