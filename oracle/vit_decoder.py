"""ORACLE - TEST INFRASTRUCTURE ONLY.  CrossVITDecoder.forward of models/module.py:273-364 (shipped decoder_cfg: linear
attention, ffn, LayerScale, pre-norm CrossBlocks with pre_norm_query, combine norms, conv head with BN + SiLU, eval
mode) restated with plain torch ops on a state dict, in the dtype of the inputs (fp32 or fp64), on any device.  Pinned to
the reference's own module by tests/golden/vit_decoder_*.npz (tests/test_vit_decoder_cpu.py).
"""
import torch
import torch.nn.functional as F

NHEAD = 12


def _t(sd, k, x):
    return sd[k].to(dtype=x.dtype, device=x.device)


def _linear(x, sd, p, bias=True):
    return F.linear(x, _t(sd, p + "weight", x), _t(sd, p + "bias", x) if bias else None)


def _ln(x, sd, p, eps):
    return F.layer_norm(x, (x.shape[-1],), _t(sd, p + "weight", x), _t(sd, p + "bias", x), eps)


def linear_attention(x, kv, sd, p):
    """attention.py:261-291 CrossLinearAttention: q from x, k = v input from kv (no bias), elu + 1, Z = 1/(q.sum_s k + eps)"""
    B, N, C = x.shape
    q = _linear(x, sd, p + "q_proj.", False).reshape(B, N, NHEAD, C // NHEAD)
    k = _linear(kv, sd, p + "k_proj.", False).reshape(B, kv.shape[1], NHEAD, C // NHEAD)
    v = _linear(kv, sd, p + "v_proj.", False).reshape(B, kv.shape[1], NHEAD, C // NHEAD)
    q, k = F.elu(q) + 1, F.elu(k) + 1
    KV = torch.einsum("nshd,nshm->nhmd", k, v)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", q, k.sum(dim=1)) + 1e-6)
    out = torch.einsum("nlhd,nhmd,nlh->nlhm", q, KV, Z).reshape(B, N, C)
    return _linear(out, sd, p + "proj.")


def cross_block(x, sd, p, key=None):
    """block.py:336-346, pre-norm with pre_norm_query=True: the key / value input is the raw `key`, or norm1(x) for self
    attention"""
    xn = _ln(x, sd, p + "norm1.", 1e-5)
    kv = xn if key is None else key
    x = x + _t(sd, p + "ls1.gamma", x) * linear_attention(xn, kv, sd, p + "attn.")
    h = F.gelu(_linear(_ln(x, sd, p + "norm2.", 1e-5), sd, p + "mlp.fc1."))
    return x + _t(sd, p + "ls2.gamma", x) * _linear(h, sd, p + "mlp.fc2.")


def _conv_bn_silu(x, sd, p, transposed):
    w, b = _t(sd, p + "0.weight", x), _t(sd, p + "0.bias", x)
    y = F.conv_transpose2d(x, w, b, stride=2, padding=1) if transposed else F.conv2d(x, w, b, padding=1)
    t = lambda k: _t(sd, p + "1." + k, y)
    return F.silu(F.batch_norm(y, t("running_mean"), t("running_var"), t("weight"), t("bias"), False, 0.0, 1e-5))


def vit_decoder(x, sd, vit_shape, p="decoder_vit."):
    """module.py:315-364: x = [x0, x1, x2], each [B,V,h*w,768] -> [B*V,64,4h,4w]"""
    B, V, H, W, C = vit_shape
    prev = [_t(sd, f"{p}prev_values.{i}", x[0]) for i in range(2)]
    ref = [x[0][:, 0]]
    for i in (1, 2):
        s = cross_block(ref[-1], sd, f"{p}self_attn_blocks.{i - 1}.")
        ref.append(_ln(prev[i - 1] * s + x[i][:, 0], sd, f"{p}norm_layers.{i - 1}.", 1e-6))
    srcs = []
    for v in range(1, V):
        s = cross_block(x[0][:, v], sd, f"{p}cross_attn_blocks.0.", key=ref[0])
        for i in (1, 2):
            q = _ln(prev[i - 1] * s + x[i][:, v], sd, f"{p}norm_layers.{i - 1}.", 1e-6)
            s = cross_block(q, sd, f"{p}cross_attn_blocks.{i}.", key=ref[i])
        srcs.append(s)
    t = torch.stack([ref[-1]] + srcs, dim=1).reshape(B * V, H, W, C).permute(0, 3, 1, 2)
    t = _conv_bn_silu(t, sd, p + "proj.", False)
    t = _conv_bn_silu(t, sd, p + "upsampler0.", True)
    return _conv_bn_silu(t, sd, p + "upsampler1.", True)
