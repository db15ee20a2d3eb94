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


def _smooth_field(g, H, W, passes):
    """seeded [H,W] field, binomial low-pass `passes` times, zero mean and unit variance"""
    x = torch.randn(1, 1, H, W, generator=g, dtype=torch.float64)
    k = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0], dtype=torch.float64) / 16.0
    for _ in range(passes):
        x = F.conv2d(F.pad(x, (2, 2, 0, 0), mode="replicate"), k.view(1, 1, 1, 5))
        x = F.conv2d(F.pad(x, (0, 0, 2, 2), mode="replicate"), k.view(1, 1, 5, 1))
    x = x[0, 0] - x.mean()
    return x / x.std().clamp_min(1e-12)


def make_fusion_scene(N, H, W, seed=77, n_src=4, theta_step=0.12, radius=650.0):
    """A scene for depth-map fusion (test.py:387-517): N cameras of the look-at ring, the true depth of an analytic
    surface (a tilted plane with a sphere in front of it) ray-cast per view, then seeded damage so that every decision
    of the filters goes both ways: smooth depth noise whose amplitude varies from nothing to a few thresholds, blobs of
    gross outliers, low-confidence regions, zero-depth holes, and a last camera with 1.6 x the focal length, which sees a
    part of what the others see, so that reprojections leave its image.
    -> dict(depths [N,H,W], confs [N,H,W], cams [N,2,4,4], images [N,3,H,W] in [0,1] on the k/255 grid, pairs
    [(ref, [src, ...]), ...] with the n_src nearest views of the ring first, depth_true [N,H,W]); float32, CPU."""
    g = torch.Generator().manual_seed(seed)
    order = [VIEW_ORDER[i % len(VIEW_ORDER)] + (i // len(VIEW_ORDER)) * 0.37 for i in range(N)]
    cams = torch.zeros(N, 2, 4, 4, dtype=torch.float64)
    depth_true = torch.zeros(N, H, W, dtype=torch.float64)
    normal = torch.tensor([0.25, 0.12, -1.0], dtype=torch.float64)
    normal = normal / normal.norm()
    on_plane = torch.tensor([0.0, 0.0, radius + 30.0], dtype=torch.float64)
    centre, rad = torch.tensor([25.0, -15.0, radius], dtype=torch.float64), 0.18 * radius * W / 1536.0 * 1536.0 / 2776.6
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64) + 0.5, torch.arange(W, dtype=torch.float64) + 0.5, indexing="ij")
    pix = torch.stack([xs, ys, torch.ones_like(xs)], -1)
    for i in range(N):
        E, K = lookat_camera(order[i], H, W, radius=radius, theta_step=theta_step,
                             focal_full=2776.6 * (1.6 if i == N - 1 and N > 2 else 1.0))
        cams[i, 0], cams[i, 1, :3, :3], cams[i, 1, 3, 3] = E, K, 1.0
        R, t = E[:3, :3], E[:3, 3]
        C = -R.T @ t
        d = (pix @ torch.linalg.inv(K).T) @ R            # world direction of unit camera depth
        plane = ((on_plane - C) @ normal) / (d @ normal)
        oc = C - centre
        a, b, c = (d * d).sum(-1), 2.0 * (d @ oc), oc @ oc - rad * rad
        disc = b * b - 4.0 * a * c
        sphere = torch.where(disc > 0, (-b - disc.clamp_min(0).sqrt()) / (2.0 * a), torch.full_like(a, float("inf")))
        sphere = torch.where(sphere > 0, sphere, torch.full_like(a, float("inf")))
        depth_true[i] = torch.minimum(plane, sphere)
    depths, confs = depth_true.clone(), torch.zeros(N, H, W, dtype=torch.float64)
    images = torch.zeros(N, 3, H, W, dtype=torch.float64)
    for i in range(N):
        amp = (0.006 * (_smooth_field(g, H, W, 6) + 0.6)).clamp_min(0.0)          # relative; thresholds are 0.0015 .. 0.01
        depths[i] *= 1.0 + amp * _smooth_field(g, H, W, 2)
        blobs = _smooth_field(g, H, W, 5) > 1.5
        depths[i] = torch.where(blobs, depths[i] * (1.0 + 0.08 * _smooth_field(g, H, W, 3)), depths[i])
        confs[i] = (0.72 + 0.3 * _smooth_field(g, H, W, 4) + 0.05 * torch.randn(H, W, generator=g, dtype=torch.float64)).clamp(0.0, 1.0)
        depths[i] = torch.where(_smooth_field(g, H, W, 4) > 1.9, torch.zeros_like(depths[i]), depths[i])
        for c in range(3):
            images[i, c] = torch.round((0.5 + 0.25 * _smooth_field(g, H, W, 3)).clamp(0.0, 1.0) * 255.0)
    pairs = []
    for i in range(N):
        others = sorted((j for j in range(N) if j != i), key=lambda j: (abs(order[j] - order[i]), j))
        pairs.append((i, others[:n_src]))
    return dict(depths=depths.float(), confs=confs.float(), cams=cams.float(), images=(images.float() / 255.0), pairs=pairs,
                depth_true=depth_true.float())


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
