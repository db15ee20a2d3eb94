"""Shared helpers of the whole-model tests: the shipped arch.args, weights of the model_*.npz fixtures re-created from
their seeds, and the errors of an output dict against a fixture."""
import copy

import torch

from mvsformerplusplus_b200.config import default_args
from oracle.gen_golden_model import CASES, fixture_outputs, make_inputs  # noqa: F401  (inputs are re-drawn from seeds)
from oracle.gen_golden_vit import vit_weights
from tests.common import load_golden, max_abs, rel_linf
from tests.vit_decoder_common import SHIPPED_ARGS

# config/mvsformer++.json arch.args: the hot-path defaults, the ViT / decoder keys and the keys only the model reads
MODEL_ARGS = dict(default_args(), **copy.deepcopy(SHIPPED_ARGS), freeze_vit=True, rescale=0.4375, decoder_type="CrossVITDecoder",
                  vit_path="./pretrained_models/dinov2_vitb14_pretrain.pth")
DEPTH_BAR, PROB_BAR = 1e-3, 1e-4   # north-star: relative L-inf on depth, absolute on probabilities


def model_args(**kw):
    a = copy.deepcopy(MODEL_ARGS)
    a.update(kw)
    return a


def model_state_dict(wseed):
    """The seeded weights oracle/gen_golden_model.py gave the reference model (same keys and shapes -> same draws)."""
    from mvsformerplusplus_b200.hotpath import DINOv2MVSNet
    return vit_weights(DINOv2MVSNet(model_args()), wseed)


def fixture(name):
    gold, meta = load_golden(name)
    imgs, proj, dv = make_inputs(meta)
    return gold, meta, imgs, proj, dv


def fixture_errors(meta, out, features_fpn, gold):
    """errors of an output dict (any device) against a fixture: depth maps relative, probabilities and confidences
    absolute, stage-1 features relative to max(1, max|ref|)"""
    got = {k: v.detach().cpu() for k, v in fixture_outputs(meta, out, features_fpn).items()}
    e = {}
    for k, want in gold.items():
        if k.endswith("depth"):
            e[k] = rel_linf(got[k], want)
        elif k.startswith("features"):
            e[k] = max_abs(got[k], want) / max(1.0, float(want.abs().max()))
        else:
            e[k] = max_abs(got[k], want)
    return e


def bar(key):
    return DEPTH_BAR if key.endswith("depth") else PROB_BAR


def within_bars(e, floor=None):
    """the keys of e over their bar: the north-star bar, or 3x the fp32-versus-fp64 floor where that floor is above a
    third of it"""
    over = {}
    for k, v in e.items():
        b = bar(k)
        if floor is not None and floor.get(k, 0.0) > b / 3:
            b = 3.0 * floor[k]
        if not v < b:
            over[k] = (v, b)
    return over


def to_double(sd):
    return {k: (v.double() if torch.is_floating_point(v) else v) for k, v in sd.items()}


class ReferenceGlueModel(torch.nn.Module):
    """A reference-shaped DINOv2MVSNet: the reference's attribute names and its eval-forward glue in torch
    (DINOv2_mvsformer_model.py:68-98: bicubic resize, per-view FPN encoder and decoder calls, conv31 + vit_feat, torch.stack),
    then the FMT + cascade glue of cascade_forward.  Its seams are the oracle's modules until install(...) rebinds them:
    with install(model, feature_pyramid=True, vit_decoder=True, vit=True) it is the best path there was before
    DINOv2MVSNet."""

    def __init__(self, args):
        from mvsformerplusplus_b200.params import build_hotpath_params
        from tests.vit_common import OracleViT
        from tests.vit_decoder_common import OracleFPNDecoder, OracleFPNEncoder, OracleViTDecoder
        super().__init__()
        self.args = self.vit_args = args
        self.encoder, self.decoder = OracleFPNEncoder(), OracleFPNDecoder()
        self.vit, self.decoder_vit = OracleViT(), OracleViTDecoder()
        hp = build_hotpath_params(args)
        self.FMT_module, self.fusions = hp.FMT_module, hp.fusions

    @torch.no_grad()
    def extract_features(self, imgs):
        import torch.nn.functional as F
        from oracle.model import vit_size
        B, V, _, H, W = imgs.shape
        vh, vw = vit_size(H, W, self.vit_args["rescale"])
        vit_imgs = F.interpolate(imgs.reshape(B * V, 3, H, W), (vh, vw), mode="bicubic", align_corners=False)
        vit_out = [v.reshape(B, V, -1, 768) for v in self.vit.forward_interval_features(vit_imgs)]
        vit_feat = self.decoder_vit.forward(vit_out, vit_shape=[B, V, vh // 14, vw // 14, 768])
        feats = [[], [], [], []]
        for vi in range(V):
            c01, c11, c21, c31 = self.encoder(imgs[:, vi])
            c31 = c31 + vit_feat[vi].unsqueeze(0)
            for k, f in enumerate(self.decoder.forward(c01, c11, c21, c31)):
                feats[k].append(f)
        return {f"stage{k + 1}": torch.stack(feats[k], dim=1) for k in range(4)}

    @torch.no_grad()
    def forward(self, imgs, proj_matrices, depth_values, tmp=(5.0, 5.0, 5.0, 1.0)):
        from mvsformerplusplus_b200.hotpath import cascade_forward
        return cascade_forward(self.FMT_module, self.fusions, self.args, self.extract_features(imgs), proj_matrices,
                               depth_values, tmp)


def installed_glue_model(sd, dev):
    """ReferenceGlueModel with the weights sd, its seams rebound by install(feature_pyramid, vit_decoder, vit)"""
    from mvsformerplusplus_b200.hotpath import install
    m = ReferenceGlueModel(model_args())
    m.load_state_dict(sd, strict=True)
    return install(m.to(dev).eval(), feature_pyramid=True, vit_decoder=True, vit=True)


def cuda_model(sd, dev):
    from mvsformerplusplus_b200 import DINOv2MVSNet
    m = DINOv2MVSNet(model_args())
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()
