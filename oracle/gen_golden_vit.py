"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the ViT fixtures by executing the REFERENCE's own
vit_base(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp", **dino_cfg)
(models/dino/dinov2.py, imported read-only, shipped config/mvsformer++.json) on seeded images.  Writes only

  tests/golden/vit_n2_3x4.npz, vit_n3_2x5.npz, vit_harsh_n1_4x4.npz   the three interval features
  tests/golden/vit_state_dict_keys.txt       vit.* keys of a reference DINOv2MVSNet

and leaves every other fixture alone.  Re-run:  python oracle/gen_golden_vit.py
Weights: synth.randomize_state_dict(seed=wseed) over a module whose child `vit` is the ViT, then vit_weights() re-draws
pos_embed and cls_token at O(0.5) (synth gives them ~1e-3 / ~0.04) and, for the harsh case, adds outlier channels
(DINOv2-style massive activations) and sharpens one block's attention.  Images are synth.make_images draws re-created
from the seeds in each fixture's meta, so only outputs are stored.
"""
import os
import sys

import torch
import torch.nn as nn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fixture, reference  # noqa: E402

CASES = {
    "vit_n2_3x4": dict(n=2, gh=3, gw=4, xseed=81, wseed=82, harsh=False),          # 42 x 56, H != W
    "vit_n3_2x5": dict(n=3, gh=2, gw=5, xseed=83, wseed=84, harsh=False),          # 28 x 70
    "vit_harsh_n1_4x4": dict(n=1, gh=4, gw=4, xseed=85, wseed=86, harsh=True),     # 56 x 56: H == W, bicubic pos path
}
OUTLIER_CHANNELS = (3, 97, 410, 767)


def vit_weights(module, wseed, harsh=False):
    """Seeded weights of a module whose child `vit` has the reference's ViT keys; loads them and returns the state dict.
    harsh: the fc2 bias of block 1 puts +-400 on four channels of the residual stream (the "massive activations" DINOv2
    carries through its later blocks), and block 2's q / k weights are scaled by 3, so its logits reach tens and some
    attention rows are sharply peaked."""
    sd = synth.randomize_state_dict(module, seed=wseed)
    g = torch.Generator().manual_seed(wseed + 1000)
    sd["vit.pos_embed"] = 0.5 * torch.randn(sd["vit.pos_embed"].shape, generator=g)
    sd["vit.cls_token"] = 0.5 * torch.randn(sd["vit.cls_token"].shape, generator=g)
    if harsh:
        for k, ch in enumerate(OUTLIER_CHANNELS):
            sd["vit.blocks.1.mlp.fc2.bias"][ch] += 400.0 * (-1) ** k
        sd["vit.blocks.2.attn.qkv.weight"][:1536] *= 3.0
    module.load_state_dict(sd, strict=True)
    return sd


def make_images(c):
    return synth.make_images(c["n"], 14 * c["gh"], 14 * c["gw"], seed=c["xseed"])


def reference_vit_base(root=None):
    """the reference's vit_base, from the models/ package under root (default: the one reference.root finds), and the
    shipped arch.args"""
    reference.import_models(root)
    from models.dino.dinov2 import vit_base
    return vit_base, reference.config()


def main():
    vit_base, cfg = reference_vit_base()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out_dir = os.path.join(REPO, "tests", "golden")
    for name, c in CASES.items():
        m = nn.Module()
        m.vit = vit_base(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp",
                         **cfg.get("dino_cfg", {}))
        m.eval()
        vit_weights(m, c["wseed"], c["harsh"])
        with torch.no_grad():
            outs = m.vit.forward_interval_features(make_images(c))
        blob = {f"out{i}": o.contiguous().numpy() for i, o in enumerate(outs)}
        fixture.save(os.path.join(out_dir, name + ".npz"), blob, c)
        print(name, [tuple(o.shape) for o in outs], [float(o.abs().max()) for o in outs])

    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    model = DINOv2MVSNet(cfg)
    with open(os.path.join(out_dir, "vit_state_dict_keys.txt"), "w") as f:
        for k, v in model.state_dict().items():
            if k.startswith("vit."):
                f.write(f"{k} {tuple(v.shape)}\n")


if __name__ == "__main__":
    main()
