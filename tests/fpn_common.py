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
