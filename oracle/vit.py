"""ORACLE - TEST INFRASTRUCTURE ONLY.  DinoVisionTransformer.forward_interval_features of models/dino/dinov2.py:249-266
(ViT-B/14 as DINOv2_mvsformer_model.py:40-41 builds it: patch conv, cls token, interpolated pos_embed, 12 pre-norm blocks
of softmax attention with LayerScale, eps-1e-6 LayerNorms, cross_interval_layers 3, eval mode) restated with plain torch
ops on a state dict, in the dtype of the input (fp32 or fp64), on any device.  Pinned to the reference's own module by
tests/golden/vit_*.npz (tests/test_vit_cpu.py).
"""
import math

import torch
import torch.nn.functional as F

NHEAD, PATCH, EPS = 12, 14, 1e-6


def _t(sd, k, x):
    return sd[k].to(dtype=x.dtype, device=x.device)


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), _t(sd, p + "weight", x), _t(sd, p + "bias", x), EPS)


def _linear(x, sd, p):
    return F.linear(x, _t(sd, p + "weight", x), _t(sd, p + "bias", x))


def pos_embed_for(pos_embed, gh, gw, dtype):
    """interpolate_pos_encoding (dinov2.py:176-200) for a gh x gw grid: unchanged for the 37 x 37 grid of a square image,
    else bicubic with scale_factor ((gh + 0.1) / 37, (gw + 0.1) / 37), computed in `dtype` -> [1, gh gw + 1, dim]."""
    pos = pos_embed.to(dtype)
    N = pos.shape[1] - 1
    if gh * gw == N and gh == gw:
        return pos
    s = math.sqrt(N)
    grid = pos[:, 1:].reshape(1, int(s), int(s), -1).permute(0, 3, 1, 2)
    patch = F.interpolate(grid, scale_factor=((gh + 0.1) / s, (gw + 0.1) / s), mode="bicubic")
    assert patch.shape[-2:] == (gh, gw)
    return torch.cat([pos[:, :1], patch.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], 1)


def block(x, sd, p):
    """block.py:85-120 (eval): x + ls1 * attn(norm1(x)), then + ls2 * mlp(norm2(x)); attention scale head_dim ** -0.5"""
    n, N, C = x.shape
    qkv = _linear(_ln(x, sd, p + "norm1."), sd, p + "attn.qkv.").reshape(n, N, 3, NHEAD, C // NHEAD).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    a = torch.softmax((q * (C // NHEAD) ** -0.5) @ k.transpose(-2, -1), dim=-1)
    o = (a @ v).transpose(1, 2).reshape(n, N, C)
    x = x + _t(sd, p + "ls1.gamma", x) * _linear(o, sd, p + "attn.proj.")
    h = F.gelu(_linear(_ln(x, sd, p + "norm2."), sd, p + "mlp.fc1."))
    return x + _t(sd, p + "ls2.gamma", x) * _linear(h, sd, p + "mlp.fc2.")


def vit_interval_features(img, sd, p="vit."):
    """img [n,3,14 gh,14 gw] -> [block 3 output, block 7 output, norm(block 11 output)], each [n, gh gw, 768] without the
    cls token"""
    n, _, H, W = img.shape
    gh, gw = H // PATCH, W // PATCH
    x = F.conv2d(img, _t(sd, p + "patch_embed.proj.weight", img), _t(sd, p + "patch_embed.proj.bias", img), stride=PATCH)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat([_t(sd, p + "cls_token", x).expand(n, -1, -1), x], 1)
    x = x + pos_embed_for(sd[p + "pos_embed"].to(x.device), gh, gw, x.dtype)
    out = []
    for i in range(12):
        x = block(x, sd, f"{p}blocks.{i}.")
        if i in (3, 7):
            out.append(x[:, 1:])
    out.append(_ln(x, sd, p + "norm.")[:, 1:])
    return out
