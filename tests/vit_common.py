"""Shared helpers of the ViT tests: the shipped dino_cfg, weights of the vit_*.npz fixtures re-created from their seeds,
and a parameter container with the reference's vit.* keys."""
import copy

import torch.nn as nn

from mvsformerplusplus_b200.params import Bag, build_vit
from oracle.gen_golden_vit import CASES, make_images, vit_weights  # noqa: F401  (fixture inputs are re-drawn from seeds)

# config/mvsformer++.json arch.args.dino_cfg (decoder_cfg is passed through to the ViT and ignored there)
DINO_CFG = dict(use_flash2_dino=False, softmax_scale=None, train_avg_length=762, cross_interval_layers=3,
                decoder_cfg=dict(init_values=1.0, prev_values=0.5, d_model=768, nhead=12, attention_type="Linear"))
VIT_KW = dict(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp")


def dino_cfg(**kw):
    c = copy.deepcopy(DINO_CFG)
    c.update(kw)
    return c


def vit_params():
    """Parameter container with the reference's vit.* keys (models/dino/dinov2.py:43-165)."""
    m = Bag()
    m.vit = build_vit(Bag())
    return m.eval()


def vit_state_dict(seed, harsh=False):
    """The seeded weights oracle/gen_golden_vit.py gave the reference module (same keys -> same draws)."""
    return vit_weights(vit_params(), seed, harsh)


def sub_sd(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def cuda_vit(sd, dev):
    from mvsformerplusplus_b200 import vit_base
    m = vit_base(**VIT_KW, **dino_cfg())
    m.load_state_dict(sub_sd(sd, "vit."), strict=True)
    return m.to(dev).eval()


class OracleViT(nn.Module):
    """Runs oracle/vit.py on its own parameters (the reference's names): the unswapped module of a stub."""

    def __init__(self):
        super().__init__()
        build_vit(self)
        self.embed_dim, self.patch_size = 768, 14

    def forward_interval_features(self, x, masks=None):
        from oracle import vit as OVT
        return OVT.vit_interval_features(x, self.state_dict(), p="")
