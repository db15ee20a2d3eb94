"""Synthetic inputs for the hot path (SURVEY.md §8(d), Appendix C).

Feature pyramids are seeded normal tensors (optionally low-pass filtered so that they behave like
image features instead of white noise), cameras are the look-at ring of Appendix C in the reference's
``proj_matrices`` layout (datasets/general_eval.py:213-242: slot 0 = 4x4 extrinsic, slot 1[:3,:3] =
intrinsic scaled per stage), and ``depth_values`` follows datasets/general_eval.py:223.
Weights are seeded and BatchNorm statistics are randomised so logits are not flat (SURVEY.md §7.3-4).
All generation is done with torch CPU generators, so the same seed gives the same tensors everywhere.
"""
import math
import re

import torch
import torch.nn.functional as F

VIEW_ORDER = [0, 1, -1, 2, -2, 3, -3, 4, -4, 5, -5, 6, -6, 7, -7]


def lookat_camera(i, H, W, focal_full=2776.6, width_full=1536.0, radius=650.0, theta_step=0.1, jitter=0.0):
    th = theta_step * i * (1.0 + jitter)
    C = torch.tensor([radius * math.sin(th), 10.0 * i, radius - radius * math.cos(th)], dtype=torch.float64)
    z = torch.tensor([0.0, 0.0, radius], dtype=torch.float64) - C
    z = z / z.norm()
    x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64), z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    R = torch.stack([x, y, z])
    E = torch.eye(4, dtype=torch.float64)
    E[:3, :3] = R
    E[:3, 3] = -R @ C
    f = focal_full * W / width_full
    K = torch.tensor([[f, 0.0, W / 2.0], [0.0, f, H / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    return E, K


def make_proj_matrices(V, H, W, batch=1, jitter=0.0, **cam_kw):
    """-> {'stage1'..'stage4': [B,V,2,4,4] float32}; stage k intrinsics rows 0-1 scaled 1/8,1/4,1/2,1."""
    out = {}
    for s, sc in enumerate([8.0, 4.0, 2.0, 1.0]):
        P = torch.zeros(batch, V, 2, 4, 4, dtype=torch.float64)
        for b in range(batch):
            for vi in range(V):
                E, K = lookat_camera(VIEW_ORDER[vi], H, W, jitter=jitter, **cam_kw)
                K = K.clone()
                K[:2] /= sc
                P[b, vi, 0] = E
                P[b, vi, 1, :3, :3] = K
        out[f"stage{s + 1}"] = P.float()
    return out


def make_depth_values(numdepth=192, depth_min=425.0, interval=2.65, batch=1):
    return (depth_min + interval * torch.arange(numdepth, dtype=torch.float32)).unsqueeze(0).repeat(batch, 1)


def make_features(V, H, W, feat_chs=(64, 32, 16, 8), seed=1234, batch=1, smooth=True):
    """{'stage1'..'stage4': [B,V,C_s,H_s,W_s]} at 1/8,1/4,1/2,1 resolution."""
    g = torch.Generator().manual_seed(seed)
    feats = {}
    for s, (c, sc) in enumerate(zip(feat_chs, [8, 4, 2, 1])):
        h, w = H // sc, W // sc
        f = torch.randn(batch * V, c, h, w, generator=g)
        if smooth:  # separable 5-tap binomial low-pass, renormalised to unit variance
            k = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0]) / 16.0
            f = F.conv2d(F.pad(f, (2, 2, 0, 0), mode="replicate"), k.view(1, 1, 1, 5).repeat(c, 1, 1, 1), groups=c)
            f = F.conv2d(F.pad(f, (0, 0, 2, 2), mode="replicate"), k.view(1, 1, 5, 1).repeat(c, 1, 1, 1), groups=c)
            f = f / f.std()
        feats[f"stage{s + 1}"] = f.view(batch, V, c, h, w).contiguous()
    return feats


def make_images(V, H, W, seed=2024):
    """[V,3,H,W] image-like inputs of the FPN encoder: a smooth random field (binomial low-pass applied twice) plus a
    little texture, per channel zero-mean and unit-variance."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, 3, H, W, generator=g)
    k = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0]) / 16.0
    for _ in range(2):
        x = F.conv2d(F.pad(x, (2, 2, 0, 0), mode="replicate"), k.view(1, 1, 1, 5).repeat(3, 1, 1, 1), groups=3)
        x = F.conv2d(F.pad(x, (0, 0, 2, 2), mode="replicate"), k.view(1, 1, 5, 1).repeat(3, 1, 1, 1), groups=3)
    x = x / x.std() + 0.2 * torch.randn(V, 3, H, W, generator=g)
    x = x - x.mean(dim=(2, 3), keepdim=True)
    return (x / x.std(dim=(2, 3), keepdim=True)).contiguous()


def randomize_state_dict(module, seed=7, prob_gain=1.0):
    """Seeded re-initialisation of a parameter container (params.build_hotpath_params or the
    reference modules themselves - same key names): seeded normal weights (1/sqrt(fan_in)), randomised BatchNorm
    affine/statistics, LayerNorm affine, LayerScale/gamma, and up-scales the final ``prob`` weights so the
    softmax over depth is not flat."""
    g = torch.Generator().manual_seed(seed)
    sd = module.state_dict()
    new = {}
    for k in sorted(sd.keys()):
        v = sd[k]
        if k.endswith("num_batches_tracked"):
            new[k] = v.clone()
            continue
        r = torch.randn(v.shape, generator=g)
        if k.endswith("running_mean"):
            new[k] = 0.2 * r
        elif k.endswith("running_var"):
            new[k] = 0.5 + torch.rand(v.shape, generator=g)
        elif ".bn." in k or re.search(r"cost_reg\.conv(7|9|11)\.1\.", k) or re.search(r"(^|\.)decoder\.out[0-3]\.1\.", k) \
                or re.search(r"(^|\.)decoder_vit\.(proj|upsampler0|upsampler1)\.1\.", k):
            new[k] = (1.0 + 0.2 * r) if k.endswith("weight") else 0.1 * r
        elif "norm" in k or ".down.1." in k or ".up.1." in k:
            new[k] = (1.0 + 0.1 * r) if k.endswith("weight") else 0.05 * r
        elif k.endswith("gamma") or k.endswith("gamma1") or k.endswith("gamma2"):
            new[k] = 1.0 + 0.1 * r
        elif k.endswith("bias"):
            new[k] = 0.05 * r
        elif v.dim() >= 2:
            fan_in = v[0].numel()
            new[k] = r * (1.0 / math.sqrt(fan_in))
            if "pe_proj" in k:
                new[k] = new[k] * 0.5
            if "cost_reg.prob.weight" in k:
                new[k] = new[k] * prob_gain
        else:
            new[k] = v.clone()
        new[k] = new[k].to(v.dtype)
    module.load_state_dict(new, strict=True)
    return new
