"""fp64 torch-CPU restatement of VoteNet's PointnetSAModuleVotes / PointnetFPModule shared MLPs (`pointnet2_modules.py`,
`pytorch_utils.SharedMLP`), the checker of pointcontrast_b200/pointnet2_modules.py.  Gradients come from autograd in fp64.

The set-abstraction MLP is written the way the library computes it, which is the same function as the original's:
  * the relative coordinates are fp32, formed as the original forms them (its index ops take fp32 xyz);
  * layer 0 projects before grouping: z0 = (F W_f^T)[j] + rel W_x^T, rel = (xyz[j] - new_xyz[i]) [/ radius];
  * BatchNorm over all B npoint nsample rows (biased variance to normalise, unbiased into the running statistics), then ReLU;
  * the max pool is a selection: per (centre, channel) the sample holding the largest z when gamma >= 0 and the smallest when gamma < 0
    (first among equals: torch's max_pool2d rule), normalised alone.  BatchNorm is monotone in z with the sign of gamma and ReLU is
    monotone, so this is the maximum of the normalised values; `sel` may be given to replay another implementation's choice where two
    samples lie within rounding of each other.
"""
import torch

D = torch.float64


def _bn(z, bn, train, momentum, eps, dims):
    """BatchNorm over `dims` of z (channels last); updates bn's running statistics (fp64 copies in `bn`) in training."""
    if train:
        mean = z.mean(dims)
        var = z.var(dims, unbiased=False)
        n = z.numel() // z.shape[-1]
        with torch.no_grad():
            bn["running_mean"].mul_(1 - momentum).add_(momentum * mean.detach())
            bn["running_var"].mul_(1 - momentum).add_(momentum * var.detach() * n / (n - 1))
    else:
        mean, var = bn["running_mean"], bn["running_var"]
    return (z - mean) / torch.sqrt(var + eps) * bn["weight"] + bn["bias"]


def layer_params(mlp, prefix):
    """[{W [Cout, Cin], weight, bias, running_mean, running_var}] in fp64 (weights as leaves requiring grad) from a module's state."""
    sd = mlp.state_dict() if hasattr(mlp, "state_dict") else mlp
    out, i = [], 0
    while f"{prefix}layer{i}.conv.weight" in sd:
        g = lambda k: sd[f"{prefix}layer{i}.{k}"].detach().cpu().to(D).clone()         # noqa: E731
        p = dict(W=g("conv.weight").flatten(1), weight=g("bn.bn.weight"), bias=g("bn.bn.bias"), running_mean=g("bn.bn.running_mean"),
                 running_var=g("bn.bn.running_var"))
        for k in ("W", "weight", "bias"):
            p[k].requires_grad_()
        out.append(p)
        i += 1
    return out


def sa_forward(xyz, features, inds, idx, layers, radius, normalize_xyz, train, momentum=0.1, eps=1e-5, sel=None):
    """xyz fp64 [B, N, 3], features fp64 [B, C, N] or None, inds [B, npoint], idx [B, npoint, S] (int) ->
    (new_xyz [B, npoint, 3], pooled [B, npoint, C_L], sel [B, npoint, C_L], per-layer z list)."""
    B, N, _ = xyz.shape
    inds, idx = inds.long(), idx.long()
    bi = torch.arange(B)[:, None]
    new_xyz = xyz[bi, inds]                                               # [B, M, 3]
    x32 = xyz.float()                                                     # rel in fp32 as the original forms it: subtract, then divide
    rel = x32[bi[:, :, None], idx] - x32[bi, inds][:, :, None]            # [B, M, S, 3]
    if normalize_xyz:
        rel = rel / radius
    rel = rel.to(D)
    W0 = layers[0]["W"]
    z = rel @ W0[:, :3].T
    if features is not None:
        P = features.transpose(1, 2) @ W0[:, 3:].T                        # [B, N, C0]: projected before grouping
        z = z + P[bi[:, :, None], idx]
    zs = []
    for k, p in enumerate(layers):
        if k:
            z = a @ p["W"].T
        zs.append(z)
        a = torch.relu(_bn(z, p, train, momentum, eps, (0, 1, 2)))
    gamma = layers[-1]["weight"].detach()
    if sel is None:
        key = torch.where(gamma >= 0, z.detach(), -z.detach())
        sel = torch.argmax(key, dim=2)                                    # first maximum
    pooled = torch.gather(a, 2, sel.long()[:, :, None, :]).squeeze(2)
    return new_xyz, pooled, sel, zs


def fp_forward(known_feats, unknow_feats, idx, weight, layers, train, momentum=0.1, eps=1e-5):
    """known_feats fp64 [B, C2, m], unknow_feats [B, C1, n] or None, idx / weight [B, n, 3] -> [B, n, C_L] (point-major)."""
    B = known_feats.shape[0]
    kf = known_feats.transpose(1, 2)
    bi = torch.arange(B)[:, None, None]
    x = (kf[bi, idx.long()] * weight.to(D)[..., None]).sum(2)             # [B, n, C2]
    if unknow_feats is not None:
        x = torch.cat([x, unknow_feats.transpose(1, 2)], 2)
    for p in layers:
        x = torch.relu(_bn(x @ p["W"].T, p, train, momentum, eps, (0, 1)))
    return x
