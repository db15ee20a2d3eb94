"""Shared helpers of the ViT-decoder tests: the shipped decoder config, weights of the vit_decoder_*.npz fixtures
re-created from their seeds, and oracle-backed modules with the reference's parameter names."""
import copy

import torch
import torch.nn as nn

from mvsformerplusplus_b200 import synth
from mvsformerplusplus_b200.params import Bag, build_fpn_decoder, build_fpn_encoder, build_vit_decoder
from oracle import fpn as OF
from oracle import vit_decoder as OV
from oracle.gen_golden_vit_decoder import CASES, make_tokens  # noqa: F401  (fixture inputs are re-drawn from seeds)

# config/mvsformer++.json arch.args: the keys CrossVITDecoder reads
SHIPPED_ARGS = dict(vit_ch=768, out_ch=64, dino_cfg=dict(
    use_flash2_dino=False, softmax_scale=None, train_avg_length=762, cross_interval_layers=3,
    decoder_cfg=dict(init_values=1.0, prev_values=0.5, d_model=768, nhead=12, attention_type="Linear", ffn_type="ffn",
                     softmax_scale="entropy_invariance", train_avg_length=762, self_cross_types=None, post_norm=False,
                     pre_norm_query=True, no_combine_norm=False)))


def shipped_args(**decoder_cfg):
    a = copy.deepcopy(SHIPPED_ARGS)
    a["dino_cfg"]["decoder_cfg"].update(decoder_cfg)
    return a


def vit_params():
    """Parameter container with the reference's decoder_vit.* keys (models/module.py:273-313)."""
    m = Bag()
    m.decoder_vit = build_vit_decoder(Bag())
    return m.eval()


def vit_state_dict(seed):
    """The seeded weights oracle/gen_golden_vit_decoder.py gave the reference module (same keys -> same draws)."""
    return synth.randomize_state_dict(vit_params(), seed=seed)


def sub_sd(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def tcs_tiles(M, N):
    """tiles of one streamed-weight GEMM: 128-row M tiles x N tiles of 128 columns (64 when N % 128 != 0), walked by
    min(tiles, SMs) persistent CTAs (csrc/linear_tc.cu:749-750, :796)"""
    return -(-M // 128) * (N // (128 if N % 128 == 0 else 64))


def decoder_gemm_tiles(B, V, h, w):
    """tiles of the streamed GEMMs of one ViT-decoder forward (csrc/vit_decoder.cu:236-266 head, :95-116 token linears
    of the source-view batch, M = (V - 1) h w tokens)"""
    L, D = h * w, 768
    t = {"head_conv": tcs_tiles(B * V * L, 256)}
    for cls in range(4):
        t[f"upsampler0_class{cls}"] = tcs_tiles(B * V * L, 128)
        t[f"upsampler1_class{cls}"] = tcs_tiles(B * V * 4 * L, 64)
    for name, n in (("q", D), ("proj", D), ("fc1", 4 * D), ("fc2", D)):
        t[f"source_{name}"] = tcs_tiles((V - 1) * L, n)
    return t


def cuda_decoder(sd, dev):
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    m = CrossVITDecoder(shipped_args())
    m.load_state_dict(sub_sd(sd, "decoder_vit."), strict=True)
    return m.to(dev).eval()


class OracleViTDecoder(nn.Module):
    """Runs oracle/vit_decoder.py on its own parameters (the reference's names): the unswapped module of a stub."""

    def __init__(self):
        super().__init__()
        build_vit_decoder(self)

    def forward(self, x, Fmats=None, vit_shape=None):
        return OV.vit_decoder(x, self.state_dict(), vit_shape, p="")


class OracleFPNEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        build_fpn_encoder(self)

    def forward(self, x):
        return OF.fpn_encoder(x, self.state_dict(), p="")


class OracleFPNDecoder(nn.Module):
    def __init__(self):
        super().__init__()
        build_fpn_decoder(self)

    def forward(self, *c):
        return OF.fpn_decoder(*c, self.state_dict(), p="")
