"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the whole-model fixtures by executing the REFERENCE's own DINOv2MVSNet
(models/networks/DINOv2_mvsformer_model.py, imported read-only, shipped config/mvsformer++.json) in eval mode on the CPU,
images to depth maps.  Writes only

  tests/golden/model_b1v3_96x128.npz   B=1, V=3: ViT grid 3 x 4
  tests/golden/model_b2v2_64x96.npz    B=2, V=2: ViT grid 2 x 3, different images per batch item, so the batch quirk of
                                       DINOv2_mvsformer_model.py:88 (every batch item gets batch item 0's vit_feat) is pinned

and leaves every other fixture alone.  Re-run:  python oracle/gen_golden_model.py
Weights: oracle/gen_golden_vit.vit_weights(model, wseed), i.e. synth.randomize_state_dict over the whole model and the ViT's
pos_embed / cls_token re-drawn at O(0.5); any module with the reference's keys re-creates them from the seed.  Inputs are
re-created from the seeds in each fixture's meta (make_inputs), so only outputs are stored: refined_depth,
photometric_confidence, per-stage depth and confidence, a seeded sample of each stage's prob_volume, and the stage-1
features before FMT.
"""
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fixture, reference  # noqa: E402
from oracle.gen_golden_vit import vit_weights  # noqa: E402

CASES = {
    "model_b1v3_96x128": dict(B=1, V=3, H=96, W=128, numdepth=192, iseed=301, wseed=302),
    "model_b2v2_64x96": dict(B=2, V=2, H=64, W=96, numdepth=48, iseed=311, wseed=312),
}
TMP = [5.0, 5.0, 5.0, 1.0]
PROB_SAMPLES = 4096


def make_inputs(c):
    """imgs [B,V,3,H,W] (distinct draws per batch item), proj_matrices (the same look-at ring for every batch item),
    depth_values [B, numdepth]"""
    imgs = synth.make_images(c["B"] * c["V"], c["H"], c["W"], seed=c["iseed"]).view(c["B"], c["V"], 3, c["H"], c["W"])
    proj = synth.make_proj_matrices(c["V"], c["H"], c["W"], batch=c["B"], theta_step=0.12)
    dv = synth.make_depth_values(c["numdepth"], 425.0, 2.65 * 192 / c["numdepth"], batch=c["B"])
    return imgs, proj, dv


def prob_sample_index(c, s, numel):
    """the flat indices of stage s's prob_volume a fixture keeps"""
    g = torch.Generator().manual_seed(1000 * c["iseed"] + s)
    return torch.randint(0, numel, (min(PROB_SAMPLES, numel),), generator=g)


def fixture_outputs(c, out, features_fpn):
    """what a fixture keeps of an output dict (shared by the generator and the tests)"""
    blob = {"refined_depth": out["refined_depth"], "photometric_confidence": out["photometric_confidence"],
            "features_fpn.stage1": features_fpn["stage1"]}
    for s in range(1, 5):
        so = out[f"stage{s}"]
        blob[f"stage{s}.depth"] = so["depth"]
        blob[f"stage{s}.photometric_confidence"] = so["photometric_confidence"]
        pv = so["prob_volume"].reshape(-1)
        blob[f"stage{s}.prob_volume_sample"] = pv[prob_sample_index(c, s, pv.numel()).to(pv.device)]
    return blob


def reference_model():
    reference.import_models()
    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    cfg = reference.config()
    cfg["vit_path"] = ""   # the weights are seeded; nothing is read
    return DINOv2MVSNet, cfg


def main():
    DINOv2MVSNet, cfg = reference_model()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out_dir = os.path.join(REPO, "tests", "golden")
    for name, c in CASES.items():
        torch.manual_seed(0)
        model = DINOv2MVSNet(cfg).eval()
        vit_weights(model, c["wseed"])
        imgs, proj, dv = make_inputs(c)
        cap, fmt_forward = {}, model.FMT_module.forward

        def capture(features):   # the reference calls FMT_module.forward directly, so a forward hook would not run
            cap["fpn"] = {k: v.clone() for k, v in features.items()}
            return fmt_forward(features)
        model.FMT_module.forward = capture
        with torch.no_grad():
            out = model(imgs, proj, dv, tmp=TMP)
        blob = {k: v.contiguous().numpy() for k, v in fixture_outputs(c, out, cap["fpn"]).items()}
        fixture.save(os.path.join(out_dir, name + ".npz"), blob, c)
        print(name, "refined_depth", float(out["refined_depth"].min()), float(out["refined_depth"].max()),
              "confidence mean", float(out["photometric_confidence"].mean()))


if __name__ == "__main__":
    main()
