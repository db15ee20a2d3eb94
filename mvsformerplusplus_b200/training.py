"""Training through the cost volume (models/cost_volume.py:64-101 under autograd) on the CUDA library.

  cost_volume(features, proj_matrices, depth_values, vis, G=8)  -> volume_mean [B,G,D,H,W], differentiable with respect to
                                                                  the features and the parameters of `vis`
  install_training(model)  rebinds forward of each model.fusions[i] of a reference-constructed DINOv2MVSNet so that its
                           cost volume runs on this op; the rest of the stage (cost_reg, softmax, depth) and the rest of
                           the model stay the reference's torch code

The warped source volumes are never stored: the forward is the eval path's warp + group correlation + view aggregation,
and the backward (mvsf_warp_corr_aggregate_backward) recomputes the samples.  What autograd keeps for the op is the fp32
channels-last features, the visibility weights, the volume, the homographies and the hypotheses."""
import types

import torch
import torch.nn.functional as F

from . import _lib
from .config import stage_list
from .hotpath import _f32c, _require_cuda


class _Aggregate(torch.autograd.Function):
    """volume [B,D,H,W,G] = sum_v vis_v * corr_v / (sum_v vis_v + 1e-6) of every sample, from feat [B,V,H,W,C] fp32
    channels-last and vis [B,V-1,H,W]; corr[b] is pass A's stored correlations of sample b (spill plan) or None (the
    aggregation gathers again)"""

    @staticmethod
    def forward(ctx, feat, vis, homs, depth, corr, G):
        B, V, H, W, C = feat.shape
        D = depth.shape[1]
        volume = torch.empty((B, D, H, W, G), device=feat.device, dtype=torch.float32)
        for b in range(B):
            if corr[b] is not None:
                _lib.call("mvsf_corr_aggregate", corr[b], vis[b], volume[b], V, G, D, H, W)
            else:
                _lib.call("mvsf_warp_corr_aggregate", feat[b], homs[b], depth[b], vis[b], volume[b], V, C, G, D, H, W)
        ctx.save_for_backward(feat, vis, volume, homs, depth)
        ctx.G = G
        return volume

    @staticmethod
    def backward(ctx, grad):
        feat, vis, volume, homs, depth = ctx.saved_tensors
        B, V, H, W, C = feat.shape
        D = depth.shape[1]
        grad_feat = torch.empty_like(feat)
        grad_vis = torch.empty_like(vis)
        for b in range(B):   # one sample's upstream gradient made contiguous at a time
            _lib.call("mvsf_warp_corr_aggregate_backward", feat[b], homs[b], depth[b], vis[b], volume[b], grad[b].contiguous(),
                      grad_feat[b], grad_vis[b], V, C, ctx.G, D, H, W)
        return grad_feat, grad_vis, None, None, None, None


def cost_volume(features, proj_matrices, depth_values, vis, G=8, spill_budget_bytes=0):
    """models/cost_volume.py:64-101 in train or eval mode.  features [B,V,C,H,W] (any float dtype, may require grad),
    proj_matrices [B,V,2,4,4], depth_values [B,D,H,W] (or [B,D]), vis a callable such as the reference's StageNet.vis,
    called once per source view in view order on the [B,1,H,W] entropy map, as the reference does.  -> volume_mean
    [B,G,D,H,W] fp32, a channels-last view.  Runs in fp32 with autocast disabled (cost_volume.py:64).

    spill_budget_bytes: the per-sample size up to which pass A may store the per-view group correlations for the
    aggregation (mvsf_warp_corr_plan).  The default 0 always gathers twice: at the fine stages that buffer is as large
    as the warped volumes this op exists not to keep."""
    _require_cuda(features, "cost_volume(features)")
    B, V, C, H, W = features.shape
    if V != proj_matrices.shape[1]:
        raise AssertionError("Different number of images and projection matrices")
    if G > C:
        raise AssertionError("G must <= C!")
    dev = features.device
    f32 = dict(device=dev, dtype=torch.float32)
    with torch.autocast("cuda", enabled=False):
        # differentiable cast + layout change: a no-op for fp32 channels-last features (FMT_with_pathway's output)
        feat = features.permute(0, 1, 3, 4, 2).to(torch.float32).contiguous()
        proj = _f32c(proj_matrices.detach())
        depth = _f32c(depth_values.detach())
        if depth.dim() == 2:
            depth = depth.view(B, -1, 1, 1).expand(B, depth.shape[1], H, W).contiguous()
        D = depth.shape[1]
        homs = torch.empty((B, (V - 1) * 12), **f32)
        kinv = torch.empty(9, **f32)
        entropy = torch.empty((B, V - 1, H, W), **f32)
        spill = _lib.lib().mvsf_warp_corr_plan(C, G, D, H, W, V, int(spill_budget_bytes)) == 0
        corr = [None] * B
        fd = feat.detach()
        for b in range(B):
            _lib.call("mvsf_compose_geometry", proj[b], V, homs[b], kinv)
            if spill:
                corr[b] = torch.empty((V - 1, D, H, W, G), **f32)
                _lib.call("mvsf_warp_corr_entropy_store", fd[b], homs[b], depth[b], entropy[b], corr[b], V, C, G, D, H, W)
            else:
                _lib.call("mvsf_warp_corr_entropy", fd[b], homs[b], depth[b], entropy[b], V, C, G, D, H, W)
        weights = torch.cat([vis(entropy[:, v:v + 1]) for v in range(V - 1)], 1).to(torch.float32).contiguous()
        volume = _Aggregate.apply(feat, weights, homs, depth, corr, G)
    return volume.permute(0, 4, 1, 2, 3)


def _check_stage(stage, i):
    from .params import Bag
    if getattr(stage, "fusion_type", "cnn") != "cnn":
        raise NotImplementedError(f"install_training: stage {i}: only fusion_type 'cnn' is implemented, got {stage.fusion_type!r}")
    if stage.depth_type != "ce":
        raise NotImplementedError(f"install_training: stage {i}: only depth_type 'ce' is implemented, got {stage.depth_type!r}")
    G = stage_list(stage.args["base_ch"], stage.stage_idx)
    if G != 8:
        raise NotImplementedError(f"install_training: stage {i}: only G = 8 groups (base_ch) is implemented, got {G}")
    if any(isinstance(m, Bag) for m in stage.vis.modules()):
        raise NotImplementedError(f"install_training: stage {i} is this package's eval-mode StageNet (its vis is a parameter "
                                  "container); install_training binds a reference-constructed model")


def _stage_forward(self, features, proj_matrices, depth_values, tmp, position3d=None):
    """StageNet.forward (models/cost_volume.py:51-133, depth_type 'ce') with the cost volume on the CUDA library"""
    G = stage_list(self.args["base_ch"], self.stage_idx)
    volume_mean = cost_volume(features, proj_matrices, depth_values, self.vis, G=G)
    cost_reg = self.cost_reg(volume_mean, position3d)
    prob_volume_pre = cost_reg.squeeze(1)
    prob_volume = F.softmax(prob_volume_pre, dim=1)
    if self.training:
        _, idx = torch.max(prob_volume, dim=1)
        depth = torch.gather(depth_values, dim=1, index=idx.unsqueeze(1)).squeeze(1)
    else:
        dv = depth_values.view(*depth_values.shape, 1, 1) if depth_values.dim() <= 2 else depth_values
        depth = torch.sum(F.softmax(prob_volume_pre * tmp, dim=1) * dv, 1)
    photometric_confidence = prob_volume.max(1)[0]
    return {"depth": depth, "prob_volume": prob_volume, "photometric_confidence": photometric_confidence.detach(),
            "depth_values": depth_values, "prob_volume_pre": prob_volume_pre}


def install_training(model):
    """Rebinds forward of each model.fusions[i] of a reference-constructed DINOv2MVSNet (models/networks/
    DINOv2_mvsformer_model.py) to a forward whose cost volume (cost_volume.py:64-101) runs on cost_volume() above, in
    train() and eval().  The module objects and their parameters are kept, so optimiser groups, state_dict(), DDP wrapping
    and checkpoints are unchanged.  Raises NotImplementedError for fusion_type != 'cnn', depth_type != 'ce', G != 8 and
    for this package's own StageNet.  Returns model."""
    for i, stage in enumerate(model.fusions):
        _check_stage(stage, i)
    for stage in model.fusions:
        stage.forward = types.MethodType(_stage_forward, stage)
    return model
