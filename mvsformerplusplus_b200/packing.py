"""Packs a reference state_dict (hot-path keys) into the flat fp32 weight layouts libmvsf_b200 documents in
include/mvsf_b200.h / csrc/*.cu.  BatchNorm (eval mode, eps 1e-5) is folded into the preceding conv in fp64.
This runs once at install time; nothing here is on the per-frame path."""
import torch

BN_EPS = 1e-5


def _d(t):
    return t.detach().double().cpu()


def _fold_bn(sd, p):
    scale = _d(sd[p + "weight"]) / torch.sqrt(_d(sd[p + "running_var"]) + BN_EPS)
    shift = _d(sd[p + "bias"]) - _d(sd[p + "running_mean"]) * scale
    return scale, shift


def _cat(parts, pad_to=4):
    flat = torch.cat([x.reshape(-1).double() for x in parts])
    if flat.numel() % pad_to:
        flat = torch.cat([flat, torch.zeros(pad_to - flat.numel() % pad_to, dtype=torch.float64)])
    return flat.float().contiguous()


def pack_vis(sd, p):
    """p = 'fusions.{s}.vis.'  -> w1[9][16] b1[16] w2[16 ic][9][16 oc] b2[16] w3[16][9][8] b3[8] w4[8] b4[1]"""
    parts = []
    for i, (cin, cout) in enumerate([(1, 16), (16, 16), (16, 8)]):
        w = _d(sd[f"{p}{i}.conv.weight"])  # [cout, cin, 3, 3]
        scale, shift = _fold_bn(sd, f"{p}{i}.bn.")
        w = w * scale.view(-1, 1, 1, 1)
        parts.append(w.permute(1, 2, 3, 0).reshape(cin, 9, cout))  # [ic][tap][oc]
        parts.append(shift)
    parts.append(_d(sd[p + "3.weight"]).reshape(8))
    parts.append(_d(sd[p + "3.bias"]).reshape(1))
    out = _cat(parts)
    assert out.numel() == 3652, out.numel()  # 3649 + pad
    return out


COSTREG_UNET_CONV_WTS = 290304          # floats of the conv part of pack_costreg_unet (csrc/costreg_unet.cu NCONV)
COSTREG_UNET_SMALL_WTS = (496, 292)     # floats of its small part by kind (csrc/costreg_unet.cu NSMALL)


def pack_costreg_unet(sd, p):
    """p = 'fusions.{s}.cost_reg.'  -> (kind, conv, small); kind 0 = CostRegNet, 1 = CostRegNet3D.  conv: per layer
    conv1 ... conv6, conv7, conv9, conv11 the weights [27 taps][ci][co] with BN scale folded (the input of
    mvsf_costreg_unet_pack_tc).  small, the wts argument: per layer the folded shift [co]; then the prob conv, [27][8]
    (kind 0) or w[8], b (kind 1)."""
    is3d = (p + "conv7.0.weight") in sd
    conv, small = [], []
    for name in ("conv1", "conv2", "conv3", "conv4", "conv5", "conv6"):
        w = _d(sd[f"{p}{name}.conv.weight"])  # [cout, cin, 3,3,3]
        scale, shift = _fold_bn(sd, f"{p}{name}.bn.")
        w = w * scale.view(-1, 1, 1, 1, 1)
        conv.append(w.permute(2, 3, 4, 1, 0).reshape(27, w.shape[1], w.shape[0]))  # [tap][ci][co]
        small.append(shift)
    for name in ("conv7", "conv9", "conv11"):
        if is3d:
            w = _d(sd[f"{p}{name}.0.weight"])  # [cin, cout, 3,3,3]
            scale, shift = _fold_bn(sd, f"{p}{name}.1.")
        else:
            w = _d(sd[f"{p}{name}.conv.weight"])
            scale, shift = _fold_bn(sd, f"{p}{name}.bn.")
        w = w * scale.view(1, -1, 1, 1, 1)
        conv.append(w.permute(2, 3, 4, 0, 1).reshape(27, w.shape[0], w.shape[1]))  # [tap][ci][co]
        small.append(shift)
    pw = _d(sd[p + "prob.weight"])
    if is3d:
        small += [pw.reshape(8), _d(sd[p + "prob.bias"]).reshape(1)]
    else:
        small.append(pw[0].permute(1, 2, 3, 0).reshape(27, 8))  # [tap][ci]
    kind = 1 if is3d else 0
    conv, small = _cat(conv), _cat(small)
    sizes = conv.numel(), small.numel()
    assert sizes == (COSTREG_UNET_CONV_WTS, COSTREG_UNET_SMALL_WTS[kind]), sizes
    return kind, conv, small


def costreg_tr_wts(layers):
    """floats of the (gemm, small) parts of pack_costreg_tr (csrc/costreg_tr.cu tr_gemm_floats / tr_small_floats)"""
    return 32768 + 49152 * layers, 672 + 768 * layers


def pack_costreg_tr(sd, p, layers):
    """p = 'fusions.{s}.cost_reg.' -> (gemm, small), the two fp32 parts of mvsf_costreg_tr_forward's weights (layout
    in csrc/costreg_tr.cu).  gemm, as [N][K] rows: down [64][256], per layer qkv [192][64], proj, linear1, linear2, then
    up [256][64].  small, the wts argument: pe_proj, the down bias and LayerNorm, per layer proj bias, gamma1, norm1,
    linear1 bias, linear2 bias, gamma2, norm2; the up bias (repeated per voxel), its LayerNorm and prob."""
    wd = _d(sd[p + "down.0.weight"])  # [64, 8, 2,4,4] -> [64][kd][kh][kw][ci]
    g = [wd.permute(0, 2, 3, 4, 1).reshape(64, 256)]
    small = [_d(sd[p + "pe_proj.weight"]).reshape(8, 24), _d(sd[p + "down.0.bias"]),
             _d(sd[p + "down.1.weight"]), _d(sd[p + "down.1.bias"])]
    for i in range(layers):
        q = f"{p}attention_layers.{i}."
        g += [_d(sd[q + k]) for k in ("attn.qkv.weight", "attn.proj.weight", "ffn.linear1.weight",
                                      "ffn.linear2.weight")]
        small += [_d(sd[q + "attn.proj.bias"]), _d(sd[q + "gamma1"]).reshape(1).expand(64), _d(sd[q + "norm1.weight"]),
                  _d(sd[q + "norm1.bias"]), _d(sd[q + "ffn.linear1.bias"]), _d(sd[q + "ffn.linear2.bias"]),
                  _d(sd[q + "gamma2"]).reshape(1).expand(64), _d(sd[q + "norm2.weight"]), _d(sd[q + "norm2.bias"])]
    wu = _d(sd[p + "up.0.weight"])  # [64 ci, 8 co, 2,4,4] -> [kd][kh][kw][co][ci] = [256][64]
    g.append(wu.permute(2, 3, 4, 1, 0).reshape(256, 64))
    small += [_d(sd[p + "up.0.bias"]).repeat(32), _d(sd[p + "up.1.weight"]), _d(sd[p + "up.1.bias"]),
              _d(sd[p + "prob.weight"]).reshape(8), _d(sd[p + "prob.bias"]).reshape(1)]
    g, small = _cat(g, pad_to=8), _cat(small, pad_to=8)
    sizes = g.numel(), small.numel()
    assert sizes == costreg_tr_wts(layers), sizes
    return g, small


def fold_conv_bn(sd, conv, bn, bias=None):
    """Conv2d weight [co, ci, k, k] (+ optional conv bias) followed by eval BatchNorm -> (w [k*k][ci][co], shift [co]) in
    fp64: BN(conv(x) + b) = conv_{w * scale}(x) + (b - mean) * scale + beta."""
    w = _d(sd[conv])
    scale, shift = _fold_bn(sd, bn)
    if bias is not None:
        shift = shift + _d(sd[bias]) * scale
    w = w * scale.view(-1, 1, 1, 1)
    return w.permute(2, 3, 1, 0).reshape(w.shape[2] * w.shape[3], w.shape[1], w.shape[0]), shift


FPN_ENCODER_CONV_WTS = 132800   # floats of the conv part of pack_fpn_encoder (csrc/fpn.cu enc_conv_off(11))
FPN_ENCODER_SMALL_WTS = 1528    # floats of its small part (csrc/fpn.cu enc_bias_off(11))


def pack_fpn_encoder(sd, p="encoder."):
    """models/module.py:208-239 -> (conv, small), the two fp32 parts of the encoder's weights (layout documented in
    include/mvsf_b200.h, mvsf_fpn_encoder_forward).  conv: the weights [k*k][ci][co] with BN folded of conv01 ...
    conv31, the layers that run on the tensor cores (the input of mvsf_fpn_pack_tc).  small, the wts argument: conv00's
    weights and shift (computed in SIMT), then the shifts [co] of conv01 ... conv31."""
    from .params import FPN_ENCODER_LAYERS
    conv, small = [], []
    for i, (name, *_) in enumerate(FPN_ENCODER_LAYERS):
        w, shift = fold_conv_bn(sd, f"{p}{name}.conv.weight", f"{p}{name}.bn.")
        (small if i == 0 else conv).append(w)
        small.append(shift)
    conv, small = _cat(conv), _cat(small)
    sizes = conv.numel(), small.numel()
    assert sizes == (FPN_ENCODER_CONV_WTS, FPN_ENCODER_SMALL_WTS), sizes
    return conv, small


FPN_DECODER_CONV_WTS = 32256    # floats of the conv part of pack_fpn_decoder (csrc/fpn.cu dec_conv_off(3))
FPN_DECODER_SMALL_WTS = 7992    # floats of its small part (csrc/fpn.cu dec_inner_off(3))


def pack_fpn_decoder(sd, p="decoder."):
    """models/module.py:242-270 -> (conv, small), the two fp32 parts of the decoder's weights (conv bias and BN folded;
    layout documented in include/mvsf_b200.h, mvsf_fpn_decoder_forward).  conv: out_k [9][64][c_k], k = 1..3 (the input
    of mvsf_fpn_pack_tc).  small, the wts argument: out0 [64][64] + shift; per level k = 1..3: inner_k [cl][64] +
    bias[64], out_k's shift [c_k]."""
    small = list(fold_conv_bn(sd, p + "out0.0.weight", p + "out0.1.", p + "out0.0.bias"))
    conv = []
    for k in (1, 2, 3):
        wi = _d(sd[f"{p}inner{k}.weight"])  # [64, cl, 1, 1]
        w, shift = fold_conv_bn(sd, f"{p}out{k}.0.weight", f"{p}out{k}.1.", f"{p}out{k}.0.bias")
        small += [wi.reshape(wi.shape[0], wi.shape[1]).t(), _d(sd[f"{p}inner{k}.bias"]), shift]
        conv.append(w)
    conv, small = _cat(conv), _cat(small)
    sizes = conv.numel(), small.numel()
    assert sizes == (FPN_DECODER_CONV_WTS, FPN_DECODER_SMALL_WTS), sizes
    return conv, small


FMT_GEMM_WTS = 196608   # floats of the GEMM part of pack_fmt (csrc/fmt.cu NG)
FMT_SMALL_WTS = 17856   # floats of its small part (csrc/fmt.cu NS)


def pack_fmt(sd, p="FMT_module."):
    """-> (gemm, small), the two fp32 parts of mvsf_fmt_forward's weights (layout in csrc/fmt.cu).  gemm, per block as
    [N][K] rows: [q; k; v] [192][64], proj, fc1, fc2.  small, the wts argument: per block norm1 w, b, proj bias, ls1,
    norm2 w, b, fc1 bias, fc2 bias, ls2; then dim_reduction_1..3 [co][ci] and smooth_1..3 [tap][ci][co]."""
    g, small = [], []
    for i in range(4):
        q = f"{p}FMT.layers.{i}."
        g += [torch.cat([_d(sd[q + "attn.q_proj.weight"]), _d(sd[q + "attn.k_proj.weight"]),
                         _d(sd[q + "attn.v_proj.weight"])], 0),
              _d(sd[q + "attn.proj.weight"]), _d(sd[q + "mlp.fc1.weight"]), _d(sd[q + "mlp.fc2.weight"])]
        small += [_d(sd[q + k]) for k in ("norm1.weight", "norm1.bias", "attn.proj.bias", "ls1.gamma", "norm2.weight",
                                          "norm2.bias", "mlp.fc1.bias", "mlp.fc2.bias", "ls2.gamma")]
    for k in (1, 2, 3):
        w = _d(sd[f"{p}dim_reduction_{k}.weight"])
        small.append(w.reshape(w.shape[0], w.shape[1]))
    for k in (1, 2, 3):
        w = _d(sd[f"{p}smooth_{k}.weight"])  # [co, ci, 3, 3] -> [tap][ci][co]
        small.append(w.permute(2, 3, 1, 0).reshape(9, w.shape[1], w.shape[0]))
    g, small = _cat(g, pad_to=8), _cat(small, pad_to=8)
    assert g.numel() == FMT_GEMM_WTS and small.numel() == FMT_SMALL_WTS, (g.numel(), small.numel())
    return g, small


VIT_DECODER_BLOCKS = tuple(f"self_attn_blocks.{i}." for i in range(2)) + tuple(f"cross_attn_blocks.{i}." for i in range(3))
VIT_DECODER_GEMM_WTS = 37814272   # floats of the GEMM part of pack_vit_decoder (csrc/vit_decoder.cu NG)
VIT_DECODER_SMALL_WTS = 49608     # floats of its small-parameter part (csrc/vit_decoder.cu N_WTS)


def deconv_class_taps(py):
    """ConvTranspose2d(k4, s2, p1) in gather form along one axis: output 2 y + py reads input y + d with kernel index k,
    for the class's two taps (d, k) (csrc/vit_decoder.cu deconv_taps)."""
    return ((0, 1), (-1, 3)) if py == 0 else ((0, 2), (1, 0))


def pack_vit_decoder(sd, p=""):
    """models/module.py:273-364 -> (gemm, small), the two fp32 parts of mvsf_vit_decoder_forward's weights (layout in
    csrc/vit_decoder.cu).  gemm, the GEMM weights as [N][K] rows: per block (self0, self1, cross0, cross1, cross2)
    [q; k; v] [2304][768], proj, fc1, fc2; the 3x3 proj conv [256][tap * 768 + ci] (tap = ky * 3 + kx) and, per parity
    class (py, px) of the two transposed convs, [co][tap * ci_n + ci] over the class's 2 x 2 gather taps; BN scale
    folded into every conv.  small, the wts argument: per block norm1 w, b, proj bias, ls1, norm2 w, b, fc1 bias, fc2
    bias, ls2; norm_layers; prev_values (padded to 8); the folded conv biases [256], [128], [64]."""
    g, small = [], []
    for b in VIT_DECODER_BLOCKS:
        q = p + b
        g += [torch.cat([_d(sd[q + "attn.q_proj.weight"]), _d(sd[q + "attn.k_proj.weight"]),
                         _d(sd[q + "attn.v_proj.weight"])], 0),
              _d(sd[q + "attn.proj.weight"]), _d(sd[q + "mlp.fc1.weight"]), _d(sd[q + "mlp.fc2.weight"])]
        small += [_d(sd[q + k]) for k in ("norm1.weight", "norm1.bias", "attn.proj.bias", "ls1.gamma", "norm2.weight",
                                          "norm2.bias", "mlp.fc1.bias", "mlp.fc2.bias", "ls2.gamma")]
    scale, shift = _fold_bn(sd, p + "proj.1.")
    w = _d(sd[p + "proj.0.weight"]) * scale.view(-1, 1, 1, 1)          # [256, 768, 3, 3]
    g.append(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))
    biases = [shift + _d(sd[p + "proj.0.bias"]) * scale]
    for name in ("upsampler0", "upsampler1"):
        scale, shift = _fold_bn(sd, f"{p}{name}.1.")
        w = _d(sd[f"{p}{name}.0.weight"]) * scale.view(1, -1, 1, 1)    # [ci, co, 4, 4]
        for py in (0, 1):
            for px in (0, 1):
                taps = [w[:, :, ky, kx] for _, ky in deconv_class_taps(py) for _, kx in deconv_class_taps(px)]
                g.append(torch.stack(taps, 0).permute(2, 0, 1).reshape(w.shape[1], -1))   # [co][tap][ci]
        biases.append(shift + _d(sd[f"{p}{name}.0.bias"]) * scale)
    for i in range(2):
        small += [_d(sd[f"{p}norm_layers.{i}.weight"]), _d(sd[f"{p}norm_layers.{i}.bias"])]
    small += [torch.stack([_d(sd[f"{p}prev_values.{i}"]).reshape(()) for i in range(2)]), torch.zeros(6, dtype=torch.float64)]
    g, small = _cat(g), _cat(small + biases, pad_to=8)
    assert g.numel() == VIT_DECODER_GEMM_WTS and small.numel() == VIT_DECODER_SMALL_WTS, (g.numel(), small.numel())
    return g, small


VIT_GEMM_WTS = 85426176   # floats of the GEMM part of pack_vit (csrc/vit.cu NG)
VIT_SMALL_WTS = 141312    # floats of its small-parameter part (csrc/vit.cu NS)


def pack_vit(sd, p=""):
    """models/dino/dinov2.py (ViT-B/14) -> (gemm, small), the two fp32 parts of mvsf_vit_forward's weights (layout in
    csrc/vit.cu).  gemm: patch_embed.proj [768][640] (k = c * 196 + ky * 14 + kx, zero from 588), then per block qkv
    [2304][768], proj, fc1, fc2 as [N][K] rows.  small, the wts argument: per block norm1 w, b, qkv bias, proj bias, ls1,
    norm2 w, b, fc1 bias, fc2 bias, ls2, and patch bias, cls token, norm w, b."""
    pw = _d(sd[p + "patch_embed.proj.weight"]).reshape(768, 588)
    g = [torch.cat([pw, torch.zeros(768, 640 - 588, dtype=torch.float64)], 1)]
    small = []
    for i in range(12):
        q = f"{p}blocks.{i}."
        g += [_d(sd[q + k]) for k in ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight")]
        small += [_d(sd[q + k]) for k in ("norm1.weight", "norm1.bias", "attn.qkv.bias", "attn.proj.bias", "ls1.gamma",
                                          "norm2.weight", "norm2.bias", "mlp.fc1.bias", "mlp.fc2.bias", "ls2.gamma")]
    small += [_d(sd[p + "patch_embed.proj.bias"]), _d(sd[p + "cls_token"]), _d(sd[p + "norm.weight"]),
              _d(sd[p + "norm.bias"])]
    g, small = _cat(g), _cat(small, pad_to=8)
    assert g.numel() == VIT_GEMM_WTS and small.numel() == VIT_SMALL_WTS, (g.numel(), small.numel())
    return g, small


def vit_pos_embed(pos_embed, gh, gw):
    """DinoVisionTransformer.interpolate_pos_encoding (dinov2.py:176-200) for a gh x gw patch grid (image 14 gh x 14 gw),
    with the reference's own F.interpolate call on the fp32 parameter, so the result is bit-identical on the same device:
    pos_embed [1, 1370, 768] -> fp32 [gh * gw + 1, 768] (row 0 = cls).  Unchanged when the grid is the 37 x 37 one the
    parameter was trained at (npatch == 1369 and image H == W); otherwise bicubic with scale_factor
    ((gh + 0.1) / 37, (gw + 0.1) / 37) - not the size ratio, which gives different values."""
    import math
    import torch.nn.functional as F
    pos = pos_embed.detach()
    npatch, N = gh * gw, pos.shape[1] - 1
    if npatch == N and gh == gw:
        return pos.float().reshape(N + 1, -1).contiguous()
    pos = pos.float()
    dim = pos.shape[-1]
    s = int(math.sqrt(N))
    w0, h0 = gh + 0.1, gw + 0.1   # the reference calls the image height w and the width h
    with torch.autocast(pos.device.type, enabled=False):
        patch = F.interpolate(pos[:, 1:].reshape(1, s, s, dim).permute(0, 3, 1, 2),
                              scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)), mode="bicubic")
    assert patch.shape[-2:] == (gh, gw), patch.shape
    patch = patch.permute(0, 2, 3, 1).reshape(-1, dim)
    return torch.cat([pos[0, :1], patch], 0).contiguous()
