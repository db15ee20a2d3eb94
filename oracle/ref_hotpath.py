"""ORACLE - TEST INFRASTRUCTURE ONLY.  Runs the REFERENCE's own modules (never this repo's kernels) through the glue of
models/networks/DINOv2_mvsformer_model.py:117-179.  Used by

  * oracle/gen_golden.py           - generates the hot-path fixtures under tests/golden/
  * bench.py --impl reference      - times the reference's own CPU implementation of the hot path
                                     (cpu_baseline.kind = "reference") when a copy of the reference's models/ package
                                     is available

The reference is located and imported by oracle/reference.py, never copied into tracked files.  Only tests/,
__graft_entry__ and bench.py's CPU legs may import this module.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import reference


def reference_root():
    """Directory that holds the reference's `models/` package, or None."""
    return reference.root("models")


def import_reference(root=None):
    reference.import_models(root)  # CPU: SDPA fallback with the same scale (attention.py:82-96,144-146)
    from models.FMT import FMT_with_pathway
    from models.cost_volume import StageNet
    from models.module import init_inverse_range, schedule_inverse_range
    from models.position_encoding import get_position_3d
    from models.warping import homo_warping_3D_with_mask
    return dict(FMT=FMT_with_pathway, StageNet=StageNet, init_inverse_range=init_inverse_range,
                schedule_inverse_range=schedule_inverse_range, get_position_3d=get_position_3d,
                homo_warp=homo_warping_3D_with_mask)


class RefHotPath(nn.Module):
    """Reference modules under the reference's attribute names (DINOv2_mvsformer_model.py:41,53)."""

    def __init__(self, R, args):
        super().__init__()
        self.FMT_module = R["FMT"](**args["FMT_config"])
        self.fusions = nn.ModuleList([R["StageNet"](args, args["ndepths"][i], i) for i in range(len(args["ndepths"]))])


def reference_hotpath(R, model, args, features, proj_matrices, depth_values, tmp, run_fmt=True, capture=True):
    """Glue of DINOv2_mvsformer_model.py:117-179, calling the reference's functions/modules only."""
    cap = {}

    def hook_vis(s):
        def fn(mod, inp, out):
            cap.setdefault(f"stage{s + 1}.entropy", []).append(inp[0][:, 0].clone())
            cap.setdefault(f"stage{s + 1}.vis_weight", []).append(out[:, 0].clone())
        return fn

    def hook_reg(s):
        def fn(mod, inp):
            cap[f"stage{s + 1}.volume_mean"] = inp[0].clone()
        return fn

    hs = []
    for s, st in enumerate(model.fusions if capture else []):   # capture=False: plain timing run, no clones
        hs.append(st.vis.register_forward_hook(hook_vis(s)))
        hs.append(st.cost_reg.register_forward_pre_hook(hook_reg(s)))
    with torch.no_grad():
        if run_fmt:
            features = model.FMT_module.forward(features)
        ndepths, ratios = args["ndepths"], args["depth_interals_ratio"]
        Hf, Wf = features[f"stage{len(ndepths)}"].shape[-2:]
        B = depth_values.shape[0]
        prob_maps = torch.zeros(B, Hf, Wf)
        outputs, so = {}, {}
        hmin = hmax = wmin = wmax = None
        for s in range(len(ndepths)):
            pm = proj_matrices[f"stage{s + 1}"]
            f = features[f"stage{s + 1}"]
            _, _, C, H, W = f.shape
            if s == 0:
                ds = R["init_inverse_range"](depth_values, ndepths[s], f.device, f.dtype, H, W)
            else:
                ds = R["schedule_inverse_range"](so["depth"], so["depth_values"], ndepths[s], ratios[s], H, W)
            p3d = None
            if args["cost_reg_type"][s] != "Normal" and args["use_pe3d"]:
                p3d, hmin, hmax, wmin, wmax = R["get_position_3d"](
                    B, H, W, pm[:, 0, 1, :3, :3], ds, depth_min=depth_values.min(), depth_max=depth_values.max(),
                    height_min=hmin, height_max=hmax, width_min=wmin, width_max=wmax, normalize=True)
            so = model.fusions[s].forward(f, pm, ds, tmp=tmp[s], position3d=p3d)
            outputs[f"stage{s + 1}"] = so
            conf = so["photometric_confidence"]
            if conf.shape[1] != Hf or conf.shape[2] != Wf:
                conf = F.interpolate(conf.unsqueeze(1), [Hf, Wf], mode="nearest").squeeze(1)
            prob_maps += conf
        outputs["refined_depth"] = so["depth"]
        outputs["photometric_confidence"] = prob_maps / len(ndepths)
    for h in hs:
        h.remove()
    for k in list(cap):
        if isinstance(cap[k], list):
            cap[k] = torch.stack(cap[k], 1)
    outputs["features"] = features
    outputs["captured"] = cap
    return outputs


