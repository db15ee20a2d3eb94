"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates tests/golden/*.npz by executing the REFERENCE's own
modules (found and imported read-only by oracle/reference.py) on seeded synthetic inputs.  The fixtures pin
oracle/hotpath.py (tests/test_oracle_golden.py) and, on the GPU box, the CUDA path (tests/test_gpu_parity.py).
Re-run:  python oracle/gen_golden.py

The reference has no tests/golden vectors of its own (SURVEY.md §4), so these reference-executed outputs
are the pin.  Reference code is imported, never copied.
"""
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from mvsformerplusplus_b200.config import default_args  # noqa: E402
from oracle import fixture  # noqa: E402
from oracle.ref_hotpath import RefHotPath, import_reference, reference_hotpath  # noqa: E402

CASES = {
    # name: (V, H, W, feature seed, weight seed)
    "hotpath_v3_96x128": dict(V=3, H=96, W=128, fseed=1234, wseed=7, numdepth=192),
    "hotpath_v4_64x96": dict(V=4, H=64, W=96, fseed=99, wseed=11, numdepth=48),
}


def make_case(c, args):
    feats = synth.make_features(c["V"], c["H"], c["W"], seed=c["fseed"])
    proj = synth.make_proj_matrices(c["V"], c["H"], c["W"], theta_step=0.12)
    dv = synth.make_depth_values(c["numdepth"], 425.0, 2.65 * 192 / c["numdepth"])
    return feats, proj, dv


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    R = import_reference()
    args = default_args()
    out_dir = os.path.join(REPO, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    tmp = [5.0, 5.0, 5.0, 1.0]

    for name, c in CASES.items():
        torch.manual_seed(0)
        model = RefHotPath(R, args).eval()
        synth.randomize_state_dict(model, seed=c["wseed"])
        feats, proj, dv = make_case(c, args)
        out = reference_hotpath(R, model, args, feats, proj, dv, tmp)
        blob = {}
        for s in range(4):
            so = out[f"stage{s + 1}"]
            for k in ("depth", "photometric_confidence", "depth_values", "prob_volume_pre"):  # prob_volume = softmax(pre)
                blob[f"stage{s + 1}.{k}"] = so[k][0].numpy()
            blob[f"stage{s + 1}.entropy"] = out["captured"][f"stage{s + 1}.entropy"][0].numpy()
            blob[f"stage{s + 1}.vis_weight"] = out["captured"][f"stage{s + 1}.vis_weight"][0].numpy()
            if s < 2:
                blob[f"stage{s + 1}.volume_mean"] = out["captured"][f"stage{s + 1}.volume_mean"][0].numpy()
        blob["refined_depth"] = out["refined_depth"][0].numpy()
        blob["photometric_confidence"] = out["photometric_confidence"][0].numpy()
        blob["fmt.stage1"] = out["features"]["stage1"][0].numpy()
        # full-resolution FMT outputs are large: keep view 1 (first source view) of stages 2-4 only
        for k in ("stage2", "stage3", "stage4"):
            blob[f"fmt.{k}.view1"] = out["features"][k][0, 1].numpy()
        fixture.save(os.path.join(out_dir, name + ".npz"), blob, c)
        print(name, "refined_depth range", float(out["refined_depth"].min()), float(out["refined_depth"].max()),
              "stage4 conf mean", float(out["stage4"]["photometric_confidence"].mean()))

    # ---- warp seam alone, including out-of-image taps and per-pixel hypotheses (warping.py:69-109)
    g = torch.Generator().manual_seed(5)
    H, W, C, D = 12, 16, 8, 4
    src = torch.randn(1, C, H, W, generator=g)
    pm = synth.make_proj_matrices(3, H * 8, W * 8, theta_step=0.5)["stage1"]  # wide baseline -> taps leave the image
    from oracle.hotpath import compose_projection
    refp, srcp = compose_projection(pm[:, 0]), compose_projection(pm[:, 2])
    dvals = 425.0 + 500.0 * torch.rand(1, D, H, W, generator=g)
    warped, mask = R["homo_warp"](src, srcp, refp, dvals)
    fixture.save(os.path.join(out_dir, "warp_seam.npz"), dict(src=src.numpy(), src_proj=srcp.numpy(), ref_proj=refp.numpy(),
                                                              depth_values=dvals.numpy(), warped=warped.numpy(), mask=mask.numpy()))
    print("warp_seam: fraction masked", float(mask.float().mean()))


if __name__ == "__main__":
    main()
