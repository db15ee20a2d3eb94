"""Shared pieces of the training tests: the training fixtures (oracle/gen_golden_train.py), a visibility CNN under the
reference's parameter names built from torch modules, and the fp64 restatement of a fixture's step."""
import torch
import torch.nn as nn

from oracle import train as OT
from tests.common import load_golden

CASES = ("train_cost_volume_stage1", "train_cost_volume_stage4")
# fixture (the reference in fp32 on the CPU) against the fp64 restatement: |a - b| <= TOL * max|b| per tensor.  About 3x
# the worst measured: 6.5e-6 (volume), 6.0e-6 (feature gradient), 2.0e-5 (vis parameter gradients), 1.4e-7 (running
# statistics); the reference's fp32 arithmetic and fp32 homography inverse are what is left
FIXTURE_TOL = 6e-5


class ConvBnReLU(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False)
        self.bn = nn.BatchNorm2d(cout)

    def forward(self, x):
        return torch.relu(self.bn(self.conv(x)))


def make_vis():
    """models/cost_volume.py:37 with the reference's parameter names (vis.0.conv.weight, vis.0.bn.*, ..., vis.3.*)"""
    return nn.Sequential(ConvBnReLU(1, 16), ConvBnReLU(16, 16), ConvBnReLU(16, 8), nn.Conv2d(8, 1, 1), nn.Sigmoid())


def fixture(name):
    """-> (arrays, meta, vis module loaded with the fixture's state dict, in train())"""
    g, meta = load_golden(name)
    vis = make_vis()
    vis.load_state_dict({k[len("sd.vis."):]: v for k, v in g.items() if k.startswith("sd.vis.")}, strict=True)
    return g, meta, vis.train()


def restated_step(g, dtype=torch.float64):
    """fp64 (or `dtype`) restatement of the fixture's step, driven by its stored volume gradient -> dict(volume,
    features_grad, vis grads {key: grad}, running statistics after the step {key: value})"""
    sd = {k[len("sd."):]: v.to(dtype).clone() for k, v in g.items() if k.startswith("sd.")}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if "running" not in k and "num_batches" not in k}
    feats = g["features"].to(dtype).requires_grad_(True)
    vol = OT.cost_volume(feats, g["proj_matrices"].to(dtype), g["depth_values"].to(dtype),
                         lambda e: OT.vis_cnn_train(e, sd, ""), G=8)
    vol.backward(g["volume_mean_grad"].to(dtype))
    return dict(volume=vol.detach(), features_grad=feats.grad, grads={k: p.grad for k, p in params.items()},
                running={k: v for k, v in sd.items() if "running" in k})


def rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-30)
