"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the FPN fixtures by executing the REFERENCE's own FPNEncoder /
FPNDecoder (models/module.py:208-270, imported read-only) on seeded synthetic images, with a seeded `vit_feat` added to
conv31 between the two modules as DINOv2_mvsformer_model.py:88 does.  Writes only

  tests/golden/fpn_n2_64x96.npz, tests/golden/fpn_n1_40x72.npz   the images x and the eight outputs (fixture_crop)
  tests/golden/fpn_state_dict_keys.txt                          encoder.* / decoder.* keys of a reference DINOv2MVSNet

and leaves every other fixture alone.  Re-run:  python oracle/gen_golden_fpn.py
Weights: synth.randomize_state_dict(seed=wseed) over a module with `encoder` and `decoder` children (tests rebuild them
from the seed stored in each fixture's meta).
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
    "fpn_n2_64x96": dict(N=2, H=64, W=96, iseed=31, vseed=32, wseed=33),
    "fpn_n1_40x72": dict(N=1, H=40, W=72, iseed=41, vseed=42, wseed=43),   # 5 x 9 at 1/8: odd sizes at every level
}


def fixture_crop(name, t):
    """What a fixture keeps of an output [N,C,h,w]: the last image of the batch (so a batch offset is exercised), the
    1/8-resolution maps whole and the finer maps as their bottom-right quarter, which still holds the image's bottom and
    right borders.  Keeps the files small."""
    t = t[-1]
    if name not in ("conv31", "out0"):
        t = t[:, t.shape[1] // 2:, t.shape[2] // 2:]
    return t


def make_inputs(c):
    x = synth.make_images(c["N"], c["H"], c["W"], seed=c["iseed"])
    g = torch.Generator().manual_seed(c["vseed"])
    vit = torch.randn(c["N"], 64, c["H"] // 8, c["W"] // 8, generator=g)
    return x, vit


def main():
    root = reference_root()
    if root is None:
        raise SystemExit("reference sources not found")
    sys.path.insert(0, root)
    import models.dino.layers.attention as A
    A.FLASH_AVAILABLE = False
    from models.module import FPNDecoder, FPNEncoder
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out_dir = os.path.join(REPO, "tests", "golden")
    chs = [8, 16, 32, 64]
    for name, c in CASES.items():
        m = nn.Module()
        m.encoder, m.decoder = FPNEncoder(chs), FPNDecoder(chs)
        m.eval()
        synth.randomize_state_dict(m, seed=c["wseed"])
        x, vit = make_inputs(c)
        with torch.no_grad():
            c01, c11, c21, c31 = m.encoder(x)
            outs = m.decoder(c01, c11, c21, c31 + vit)   # the decoder input is conv31 + vit_feat
        # vit_feat is a plain torch.randn draw (bit-reproducible from vseed); x involves CPU convolutions, so it is stored
        full = dict(conv01=c01, conv11=c11, conv21=c21, conv31=c31, **{f"out{k}": o for k, o in enumerate(outs)})
        blob = dict(x=x.numpy(), **{k: fixture_crop(k, v).contiguous().numpy() for k, v in full.items()})
        blob["meta"] = np.frombuffer(json.dumps(c).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **blob)
        print(name, {k: float(np.abs(v).max()) for k, v in blob.items() if k != "meta"})

    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    cfg = json.load(open(os.path.join(root, "config", "mvsformer++.json")))["arch"]["args"]
    model = DINOv2MVSNet(cfg)
    with open(os.path.join(out_dir, "fpn_state_dict_keys.txt"), "w") as f:
        for k, v in model.state_dict().items():
            if k.startswith("encoder.") or k.startswith("decoder."):
                f.write(f"{k} {tuple(v.shape)}\n")


if __name__ == "__main__":
    main()
