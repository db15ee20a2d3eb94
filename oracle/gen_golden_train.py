"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the training fixtures of the cost volume by executing the REFERENCE's own
StageNet (models/cost_volume.py, imported read-only through oracle/reference.py, shipped config/mvsformer++.json) in
train() mode on the CPU, one forward and backward of its CE loss (models/losses.py get_multi_stage_losses) against a
seeded depth_gt and mask.  Writes only

  tests/golden/train_cost_volume_stage1.npz   stage 1: C = 64, D = 32 (transformer regulariser), B = 1, V = 3
  tests/golden/train_cost_volume_stage4.npz   stage 4: C = 8, D = 4 (CostRegNet3D), B = 2, V = 4, H even

Each holds the inputs (features, proj_matrices, depth_values), the vis part of the stage's state dict before the step
(`sd.<key>`; cost_reg's weights re-create from the seed and only shape the stored volume gradient),
volume_mean and its gradient (hooks on cost_reg's input), the gradient of the features, the gradient of every vis
parameter (`grad.<key>`) and the vis BatchNorm running statistics after the step (`after.<key>`).
Re-run:  python oracle/gen_golden_train.py
"""
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fixture, reference  # noqa: E402
from oracle import hotpath as O  # noqa: E402

CASES = {
    "train_cost_volume_stage1": dict(stage=0, B=1, V=3, H=8, W=16, seed=401, wseed=402),
    "train_cost_volume_stage4": dict(stage=3, B=2, V=4, H=16, W=32, seed=411, wseed=412),
}
CHANNELS = (64, 32, 16, 8)
LOSS_ARGS = {"dlossw": [1.0, 1.0, 1.0, 1.0], "focal": False, "gamma": 2.0}   # arch.loss of the shipped config


def make_inputs(c, D):
    """features [B,V,C,H,W], proj_matrices [B,V,2,4,4] (the stage's intrinsics of the synth look-at ring), depth_values
    [B,D,H,W] (init_inverse_range over 425..931), depth_gt [B,H,W] inside that range and mask [B,H,W] (~80 % valid)"""
    s, B, V, H, W = c["stage"], c["B"], c["V"], c["H"], c["W"]
    g = torch.Generator().manual_seed(c["seed"])
    feats = torch.randn(B, V, CHANNELS[s], H, W, generator=g)
    scale = 2 ** (3 - s)
    proj = synth.make_proj_matrices(V, H * scale, W * scale, batch=B, theta_step=0.12)[f"stage{s + 1}"]
    dv = synth.make_depth_values(192, batch=B)
    depth_values = O.init_inverse_range(dv, D, H, W)
    depth_gt = 430.0 + 490.0 * torch.rand(B, H, W, generator=g)
    mask = (torch.rand(B, H, W, generator=g) < 0.8).float()
    return feats, proj, depth_values, depth_gt, mask


def reference_stage(c):
    reference.import_models()
    from models.cost_volume import StageNet
    args = reference.config()
    s = c["stage"]
    torch.manual_seed(0)
    stage = StageNet(args, args["ndepths"][s], s)
    synth.randomize_state_dict(stage, seed=c["wseed"])
    return stage.train(), args


def run(c):
    """-> the fixture's arrays"""
    stage, args = reference_stage(c)
    from models.losses import get_multi_stage_losses
    s = c["stage"]
    D = args["ndepths"][s]
    feats, proj, depth_values, depth_gt, mask = make_inputs(c, D)
    sd0 = {k: v.clone() for k, v in stage.state_dict().items() if k.startswith("vis.")}
    cap = {}

    def pre_hook(mod, inp):
        inp[0].register_hook(lambda g: cap.__setitem__("grad", g.clone()))
        cap["volume"] = inp[0].detach().clone()
    h = stage.cost_reg.register_forward_pre_hook(pre_hook)
    feats.requires_grad_(True)
    out = stage(feats, proj, depth_values, tmp=[5.0, 5.0, 5.0, 1.0][s])
    h.remove()
    key = f"stage{s + 1}"
    # depth_types indexed by stage: one stage's outputs, so a one-entry mapping
    losses = get_multi_stage_losses(LOSS_ARGS, {s: "ce"}, {key: out}, {key: depth_gt}, {key: mask},
                                    depth_values[:, 1, 0, 0] - depth_values[:, 0, 0, 0], args["inverse_depth"])
    loss = sum(losses.values())
    loss.backward()
    blob = dict(features=feats.detach(), proj_matrices=proj, depth_values=depth_values, depth_gt=depth_gt, mask=mask,
                volume_mean=cap["volume"], volume_mean_grad=cap["grad"], features_grad=feats.grad, loss=loss.detach())
    blob.update({f"sd.{k}": v for k, v in sd0.items()})
    for k, p in stage.vis.named_parameters():
        blob[f"grad.vis.{k}"] = p.grad
    for k, v in stage.vis.state_dict().items():
        if "running" in k:
            blob[f"after.vis.{k}"] = v
    return {k: v.contiguous().numpy() for k, v in blob.items()}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out_dir = os.path.join(REPO, "tests", "golden")
    for name, c in CASES.items():
        blob = run(c)
        fixture.save(os.path.join(out_dir, name + ".npz"), blob, c)
        print(name, "loss", float(blob["loss"]), "|grad features|max", float(abs(blob["features_grad"]).max()),
              "|grad volume|max", float(abs(blob["volume_mean_grad"]).max()))


if __name__ == "__main__":
    main()
