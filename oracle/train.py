"""ORACLE - TEST INFRASTRUCTURE ONLY.  The training-mode cost volume (models/cost_volume.py:64-101 under autograd),
restated in plain torch next to oracle/hotpath.cost_volume, whose warp and group correlation it reuses.  The visibility
CNN is a callable, so that train-mode BatchNorm (batch statistics, running-statistics update) runs as in the reference;
vis_cnn_train is that CNN as a function of a flat state dict.  dtype follows the inputs: in fp64 this is the truth the
CUDA op's gradients are held against.  With oracle.hotpath.USE_ATEN_KERNELS the warp is F.grid_sample, the reference's
own sampler, and under torch.set_default_device("cuda") the whole restatement runs on the GPU (the training benchmark's
reference arm).  Self-contained: it does not import the reference."""
import torch
import torch.nn.functional as F

from oracle import hotpath as O


def vis_cnn_train(entropy, sd, p, momentum=0.1, eps=1e-5):
    """cost_volume.py:37 in train() mode: BatchNorm normalises with the batch statistics and updates sd's running_mean /
    running_var in place (momentum 0.1, unbiased variance), as nn.BatchNorm2d does"""
    x = entropy
    for i in range(3):
        b = f"{p}vis.{i}.bn."
        x = F.conv2d(x, sd[f"{p}vis.{i}.conv.weight"], padding=1)
        x = F.relu(F.batch_norm(x, sd[b + "running_mean"], sd[b + "running_var"], sd[b + "weight"], sd[b + "bias"],
                                training=True, momentum=momentum, eps=eps))
    return torch.sigmoid(F.conv2d(x, sd[f"{p}vis.3.weight"], sd[f"{p}vis.3.bias"]))


def cost_volume(features, proj_matrices, depth_values, vis, G):
    """cost_volume.py:64-101: features [B,V,C,H,W], proj_matrices [B,V,2,4,4], depth_values [B,D,H,W], vis a callable on
    the [B,1,H,W] entropy of each source view (in view order) -> volume_mean [B,G,D,H,W].  Differentiable with respect to
    the features and whatever vis closes over; the entropy is taken of the detached similarity (cost_volume.py:91)."""
    ref_feat, src_feats = features[:, 0], torch.unbind(features[:, 1:], dim=1)
    projs = torch.unbind(proj_matrices, 1)
    ref_new = O.compose_projection(projs[0])
    volume_sum, vis_sum = 0.0, 0.0
    for src_feat, src_proj in zip(src_feats, projs[1:]):
        warped, _ = O.homo_warp(src_feat, O.compose_projection(src_proj), ref_new, depth_values)
        in_prod = O.group_correlation(ref_feat, warped, G)
        p = F.softmax(in_prod.sum(dim=1).detach(), dim=1)
        w = vis((-p * torch.log(p + 1e-7)).sum(dim=1, keepdim=True))
        volume_sum = volume_sum + in_prod * w.unsqueeze(1)
        vis_sum = vis_sum + w
    return volume_sum / (vis_sum.unsqueeze(1) + 1e-6)
