"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the depth-map fusion fixtures by executing the REFERENCE's own
misc/fusion.py (imported read-only; oracle/_ref/misc/fusion.py where build() copied it) on the seeded synthetic scenes of
synth.make_fusion_scene.  The glue between its functions (test.py:395-412 for pcd, :453-483 for dpcd) is restated in
reference_filter below, because test.py parses the command line on import.  Writes only

  tests/golden/fusion_n6_40x72.npz     6 views, 4 sources, odd size; reference views 0 and 5 (5 has the long focal length)
  tests/golden/fusion_n11_32x48.npz    11 views, 10 sources; reference view 0

each with the scene (depths, confs, cams, images as uint8) and, per method m in (pcd, dpcd) and stored reference view r,
m_mask_r (bits), m_depth_r (averaged depth, [H,W]) and m_points_r (world points of the masked pixels, [M,3]).
Re-run:  python oracle/gen_golden_fusion.py

misc/fusion.py builds its pixel grid with `.cuda()` (fusion.py:9-10).  To run it on a machine without a GPU, on_cpu()
replaces torch.Tensor.cuda by the identity for the duration of the call and restores it afterwards.
"""
import contextlib
import importlib.util
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402

CASES = {
    "fusion_n6_40x72": dict(N=6, H=40, W=72, n_src=4, seed=77, refs=[0, 5]),
    "fusion_n11_32x48": dict(N=11, H=32, W=48, n_src=10, seed=78, refs=[0]),
}
DEFAULTS = dict(conf=0.5, thres_view=2, thres_disp=1.0, dist_base=4.0, rel_diff_base=1300.0)   # test.py:64-66,84-85


def reference_fusion_module():
    """The reference's misc/fusion.py as a module, or None where the reference is not available."""
    for root in (os.environ.get("MVSF_REFERENCE"), os.path.join(REPO, "oracle", "_ref"), "/root/reference"):
        path = os.path.join(root, "misc", "fusion.py") if root else None
        if path and os.path.isfile(path):
            spec = importlib.util.spec_from_file_location("mvsf_reference_fusion", path)
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            return mod
    return None


@contextlib.contextmanager
def on_cpu():
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = orig


def reference_filter(fusion, method, ref, srcs, depths, confs, cams, conf=0.5, thres_view=2, thres_disp=1.0, dist_base=4.0,
                     rel_diff_base=1300.0):
    """One reference view through the reference's functions on the tensors' device -> mask [H,W] bool, averaged depth
    [H,W], points [3,H,W].  The scene tensors are not modified."""
    ref_depth, ref_cam, ref_conf = depths[ref][None, None], cams[ref][None], confs[ref][None]
    src_depths, src_cams, src_confs = depths[srcs][None, :, None].clone(), cams[srcs][None], confs[srcs][None]
    prob_mask = ref_conf > conf
    if method == "pcd":
        for k in range(src_depths.size(1)):
            src_depths[:, k] *= (src_confs[:, k] > conf).float()
        reproj_xyd, in_range = fusion.get_reproj(ref_depth, src_depths, ref_cam, src_cams)
        vis_masks, vis_mask = fusion.vis_filter(ref_depth, reproj_xyd, in_range, thres_disp, 0.01, thres_view)
        depth_avg = fusion.ave_fusion(ref_depth, reproj_xyd, vis_masks)
        mask = fusion.bin_op_reduce([prob_mask, vis_mask], torch.min)
    else:
        dy_range = src_depths.shape[1] + 1
        reproj_xyd = fusion.get_reproj_dynamic(ref_depth, src_depths, ref_cam, src_cams)
        vis_masks, vis_mask = fusion.vis_filter_dynamic(ref_depth, reproj_xyd, dist_base=dist_base, rel_diff_base=rel_diff_base)
        reproj_depth = reproj_xyd[:, :, -1]
        reproj_depth[~vis_mask.squeeze(2)] = 0
        sums, last = vis_masks.sum(dim=1), vis_mask.sum(dim=1)
        depth_avg = (torch.sum(reproj_depth, dim=1, keepdim=True) + ref_depth) / (last + 1)
        geo_mask = last >= dy_range
        for i in range(2, dy_range):
            geo_mask = torch.logical_or(geo_mask, sums[:, i - 2] >= i)
        mask = fusion.bin_op_reduce([prob_mask, geo_mask], torch.min)
    idx_img = fusion.get_pixel_grids(*depth_avg.size()[-2:]).unsqueeze(0)
    idx_cam = fusion.idx_img2cam(idx_img, depth_avg, ref_cam)
    points = fusion.idx_cam2world(idx_cam, ref_cam)[..., :3, 0].permute(0, 3, 1, 2)
    return mask[0, 0].bool(), depth_avg[0, 0], points[0]


def main():
    fusion = reference_fusion_module()
    if fusion is None:
        raise SystemExit("reference sources not found")
    out_dir = os.path.join(REPO, "tests", "golden")
    for name, c in CASES.items():
        sc = synth.make_fusion_scene(c["N"], c["H"], c["W"], seed=c["seed"], n_src=c["n_src"])
        blob = dict(depths=sc["depths"].numpy(), confs=sc["confs"].numpy(), cams=sc["cams"].numpy(),
                    images=torch.round(sc["images"] * 255).to(torch.uint8).numpy())
        meta = dict(c, pairs=sc["pairs"], **DEFAULTS)
        for method in ("pcd", "dpcd"):
            for r in c["refs"]:
                with on_cpu(), torch.no_grad():
                    mask, avg, pts = reference_filter(fusion, method, r, sc["pairs"][r][1], sc["depths"], sc["confs"], sc["cams"])
                blob[f"{method}_mask_{r}"] = np.packbits(mask.numpy())
                blob[f"{method}_depth_{r}"] = avg.numpy()
                blob[f"{method}_points_{r}"] = pts.permute(1, 2, 0)[mask].numpy()
                print(name, method, r, "kept", float(mask.float().mean()))
        blob["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **blob)
        print(name, os.path.getsize(os.path.join(out_dir, name + ".npz")), "bytes")


if __name__ == "__main__":
    main()
