"""Shared helpers of the FPN tests: weights of the fpn_*.npz fixtures re-created from their seeds, their inputs."""
import torch
import torch.nn as nn

from mvsformerplusplus_b200 import synth
from mvsformerplusplus_b200.params import Bag, build_fpn_decoder, build_fpn_encoder
from oracle.gen_golden_fpn import fixture_crop  # noqa: F401  (what a fixture keeps of an output)

FPN_CASES = ("fpn_n2_64x96", "fpn_n1_40x72")


def fpn_params():
    """Parameter container with the reference's encoder.* / decoder.* keys (models/module.py:208-255)."""
    m = Bag()
    m.encoder = build_fpn_encoder(Bag())
    m.decoder = build_fpn_decoder(Bag())
    return m.eval()


def fpn_state_dict(seed):
    """The seeded weights oracle/gen_golden_fpn.py gave the reference modules (same keys and shapes -> same draws)."""
    return synth.randomize_state_dict(fpn_params(), seed=seed)


def fpn_inputs(gold, meta):
    """Inputs of a fixture: the stored images and vit_feat re-drawn from its seed."""
    g = torch.Generator().manual_seed(meta["vseed"])
    vit = torch.randn(meta["N"], 64, meta["H"] // 8, meta["W"] // 8, generator=g)
    return gold["x"], vit


def sub_sd(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


# ---- tile coverage of the 13 tensor-core convolutions (csrc/fpn.cu, csrc/conv2d_tc.cuh)
# name, CI, CO, KS, S, TR, NS, output scale (1 = full resolution), source: csrc/fpn.cu:223-233 (kEnc[1..10], EncL: S = 2
# for layers 2, 5, 8, TR = 8 from layer 8 on; kDec, DecL: TR = 8 for out1), with the source that fills each layer's tile
FPN_TC_LAYERS = (
    ("conv01", 8, 8, 5, 1, 16, 8, 1, "conv00"), ("downsample1", 8, 16, 5, 2, 16, 16, 2, "nhwc"),
    ("conv10", 16, 16, 3, 1, 16, 16, 2, "nhwc"), ("conv11", 16, 16, 3, 1, 16, 16, 2, "nhwc"),
    ("downsample2", 16, 32, 5, 2, 16, 32, 4, "nhwc"), ("conv20", 32, 32, 3, 1, 16, 32, 4, "nhwc"),
    ("conv21", 32, 32, 3, 1, 16, 32, 4, "nhwc"), ("downsample3", 32, 64, 3, 2, 8, 32, 8, "nhwc"),
    ("conv30", 64, 64, 3, 1, 8, 32, 8, "nhwc"), ("conv31", 64, 64, 3, 1, 8, 32, 8, "nhwc"),
    ("out1", 64, 32, 3, 1, 8, 32, 4, "intra32"), ("out2", 64, 16, 3, 1, 16, 16, 2, "intra16"),
    ("out3", 64, 8, 3, 1, 16, 8, 1, "intra8"),
)


def conv_smem(CI, CO, KS, S, TR, NS, src):
    """dynamic shared memory of one conv2d_tc_kernel launch: Conv::SMEM (csrc/conv2d_tc.cuh:25-31) + Src::EXTRA
    (Conv00Src, csrc/fpn.cu:52-53; IntraSrc, :101; NhwcSrc has none)"""
    halo = (KS - 1) // S
    pr, pc = TR + halo, 32 + halo
    plane = pr * pc * 16
    ng = 1 if CI < 16 else CI // 16
    smem = S * S * (CI // 8) * 2 * plane + KS * KS * ng * 64 * NS
    if src == "conv00":
        smem += (3 * (pr + 6) * (pc + 6) + 49 * 3 * 8 + 8) * 4
    elif src.startswith("intra"):
        smem += (int(src[5:]) * 64 + 64) * 4
    return smem


def fpn_coverage(N, H, W, sms, smem_per_sm, max_threads_per_sm=2048):
    """{layer: (tiles, grid bound, right edge ragged, bottom edge ragged)} of an FPN run on N images of H x W.  The grid
    launch_conv picks is min(tiles, resident CTAs per SM * SMs / N blocks) (conv2d_tc.cuh:176-178); the bound counts
    the resident CTAs from the thread and shared-memory limits only (1 KB of each CTA's shared memory is the runtime's),
    and registers can only lower it, so tiles > bound means some CTA runs a second tile (conv2d_tc.cuh:61)."""
    out = {}
    for name, CI, CO, KS, S, TR, NS, scale, src in FPN_TC_LAYERS:
        OH, OW = H // scale, W // scale
        tiles = N * -(-OW // 32) * -(-OH // TR)
        per_sm = min(max_threads_per_sm // 256, smem_per_sm // (conv_smem(CI, CO, KS, S, TR, NS, src) + 1024))
        bound = max(1, per_sm * sms // (CO // NS))
        out[name] = (tiles, bound, OW % 32 != 0, OH % TR != 0)
    return out


class Pyramid(nn.Module):
    """encoder -> conv31 + vit_feat -> decoder, the glue of DINOv2_mvsformer_model.py:85-98 for one view at a time."""

    def __init__(self, encoder, decoder):
        super().__init__()
        self.encoder, self.decoder = encoder, decoder

    def forward(self, imgs, vit_feat):   # imgs [B,V,3,H,W], vit_feat [V,64,H/8,W/8]
        feats = [[], [], [], []]
        for vi in range(imgs.shape[1]):
            c01, c11, c21, c31 = self.encoder(imgs[:, vi])
            c31 = c31 + vit_feat[vi].unsqueeze(0)
            for k, f in enumerate(self.decoder.forward(c01, c11, c21, c31)):
                feats[k].append(f)
        return {f"stage{k + 1}": torch.stack(feats[k], dim=1) for k in range(4)}
