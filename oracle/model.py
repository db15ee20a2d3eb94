"""ORACLE - TEST INFRASTRUCTURE ONLY.  The eval forward of DINOv2MVSNet (models/networks/DINOv2_mvsformer_model.py:68-179),
images to depth maps, composed from the restatements of its parts (oracle/vit.py, vit_decoder.py, fpn.py, hotpath.py)
with F.interpolate for the resizes, in the dtype of the inputs (fp32 or fp64), on the CPU.  Pinned to the reference's own
DINOv2MVSNet.forward by tests/golden/model_*.npz (tests/test_model_cpu.py).
"""
import torch
import torch.nn.functional as F

from oracle import fpn as OF
from oracle import hotpath as O
from oracle import vit as OVT
from oracle import vit_decoder as OV


def vit_size(H, W, rescale):
    """DINOv2_mvsformer_model.py:72: the ViT input size, a multiple of the patch size"""
    return int(H * rescale // 14 * 14), int(W * rescale // 14 * 14)


def extract_features(imgs, sd, rescale):
    """DINOv2_mvsformer_model.py:75-98 (eval branch): imgs [B,V,3,H,W] -> the FPN pyramid {stage1..4: [B,V,C,h,w]}.
    vit_feat is b-major [B V, 64, H/8, W/8] and view vi of every batch item gets vit_feat[vi] (:88), batch item 0's."""
    B, V, _, H, W = imgs.shape
    vh, vw = vit_size(H, W, rescale)
    vit_imgs = F.interpolate(imgs.reshape(B * V, 3, H, W), (vh, vw), mode="bicubic", align_corners=False)
    vit_out = [v.reshape(B, V, -1, 768) for v in OVT.vit_interval_features(vit_imgs, sd)]
    vit_feat = OV.vit_decoder(vit_out, sd, [B, V, vh // 14, vw // 14, 768])
    if vit_feat.shape[2] != H // 8 or vit_feat.shape[3] != W // 8:
        vit_feat = F.interpolate(vit_feat, size=(H // 8, W // 8), mode="bilinear", align_corners=False)
    feats = [[], [], [], []]
    for vi in range(V):
        c01, c11, c21, c31 = OF.fpn_encoder(imgs[:, vi], sd)
        c31 = c31 + vit_feat[vi].unsqueeze(0)
        for k, f in enumerate(OF.fpn_decoder(c01, c11, c21, c31, sd)):
            feats[k].append(f)
    return {f"stage{k + 1}": torch.stack(feats[k], dim=1) for k in range(4)}


def model_forward(imgs, proj_matrices, depth_values, sd, args, tmp=(5.0, 5.0, 5.0, 1.0)):
    """DINOv2MVSNet.forward in eval mode -> the reference's output dict, plus "features_fpn" (the pyramid before FMT)
    and "features" (after FMT)"""
    with torch.no_grad():
        fpn = extract_features(imgs, sd, args["rescale"])
        out = O.hotpath_forward(fpn, proj_matrices, depth_values, sd, args, tmp=tmp)
    out["features_fpn"] = fpn
    return out
