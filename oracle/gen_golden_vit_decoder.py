"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the ViT-decoder fixtures by executing the REFERENCE's own CrossVITDecoder
(models/module.py:273-364, imported read-only, shipped config/mvsformer++.json) on seeded token maps.  Writes only

  tests/golden/vit_decoder_b1v3_4x6.npz, vit_decoder_b2v2_3x5.npz, vit_decoder_harsh_b1v2_4x4.npz   the output
  tests/golden/vit_decoder_state_dict_keys.txt       decoder_vit.* keys of a reference DINOv2MVSNet

and leaves every other fixture alone.  Re-run:  python oracle/gen_golden_vit_decoder.py
Weights: synth.randomize_state_dict(seed=wseed) over a module whose child `decoder_vit` is the decoder.  Inputs are
torch.randn draws re-drawn bit for bit from the seeds in each fixture's meta (make_tokens), so only outputs are stored.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle.ref_hotpath import reference_root  # noqa: E402

CASES = {
    "vit_decoder_b1v3_4x6": dict(B=1, V=3, h=4, w=6, xseed=51, wseed=52, harsh=False),
    "vit_decoder_b2v2_3x5": dict(B=2, V=2, h=3, w=5, xseed=61, wseed=62, harsh=False),   # odd grid, batch offset
    "vit_decoder_harsh_b1v2_4x4": dict(B=1, V=2, h=4, w=4, xseed=71, wseed=72, harsh=True),
}
OUTLIER_CHANNELS = (3, 97, 410, 767)


def make_tokens(c):
    """[x0, x1, x2], each [B,V,h*w,768].  harsh: the block-8 tokens x1 scaled by 40 with a few outlier channels of
    magnitude ~300 in x1 and x2 (dinov2.py:259 notes that the features of blocks 8-10 are very large)."""
    g = torch.Generator().manual_seed(c["xseed"])
    x = [torch.randn(c["B"], c["V"], c["h"] * c["w"], 768, generator=g) for _ in range(3)]
    if c["harsh"]:
        x[1] = 40.0 * x[1]
        for k, ch in enumerate(OUTLIER_CHANNELS):
            x[1][..., ch] += 300.0 * (-1) ** k
            x[2][..., ch] -= 150.0 * (-1) ** k
    return x


def reference_decoder_cls(root):
    sys.path.insert(0, root)
    import models.dino.layers.attention as A
    A.FLASH_AVAILABLE = False
    from models.module import CrossVITDecoder
    cfg = json.load(open(os.path.join(root, "config", "mvsformer++.json")))["arch"]["args"]
    return CrossVITDecoder, cfg


def main():
    root = reference_root()
    if root is None:
        raise SystemExit("reference sources not found")
    CrossVITDecoder, cfg = reference_decoder_cls(root)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out_dir = os.path.join(REPO, "tests", "golden")
    for name, c in CASES.items():
        m = nn.Module()
        m.decoder_vit = CrossVITDecoder(cfg)
        m.eval()
        synth.randomize_state_dict(m, seed=c["wseed"])
        x = make_tokens(c)
        with torch.no_grad():
            out = m.decoder_vit(x, vit_shape=[c["B"], c["V"], c["h"], c["w"], 768])
        blob = dict(out=out.contiguous().numpy(), meta=np.frombuffer(json.dumps(c).encode(), dtype=np.uint8))
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **blob)
        print(name, tuple(out.shape), float(out.abs().max()))

    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    model = DINOv2MVSNet(cfg)
    with open(os.path.join(out_dir, "vit_decoder_state_dict_keys.txt"), "w") as f:
        for k, v in model.state_dict().items():
            if k.startswith("decoder_vit."):
                f.write(f"{k} {tuple(v.shape)}\n")


if __name__ == "__main__":
    main()
