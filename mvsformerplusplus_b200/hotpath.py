"""Host side of the CUDA hot path: Python/PyTorch mirrors of the reference seams (SURVEY.md §8b) that
enqueue libmvsf_b200 kernels.  PyTorch is used for device memory, streams and module/state-dict plumbing only.

  StageNet.forward(features, proj_matrices, depth_values, tmp, position3d=None)   <- models/cost_volume.py:51-133
  FMT_with_pathway.forward(features)                                              <- models/FMT.py:164-206
  HotPathNet.forward_features(features, proj_matrices, depth_values, tmp)         <- DINOv2_mvsformer_model.py:117-179
  FPNEncoder.forward(x) / FPNDecoder.forward(conv01, conv11, conv21, conv31)     <- models/module.py:208-270
  install(model)  rebinds the two module seams of a reference-constructed DINOv2MVSNet        (test.py drop-in)
  install(model, feature_pyramid=True)  also rebinds model.encoder / model.decoder
  CrossVITDecoder.forward(x, Fmats=None, vit_shape=None)                          <- models/module.py:273-364
  install(model, vit_decoder=True)  also rebinds model.decoder_vit
  DinoVisionTransformer.forward_interval_features(x, masks=None)                  <- models/dino/dinov2.py:249-266
  install(model, vit=True)  also rebinds model.vit (vit_base(...), DINOv2_mvsformer_model.py:40-41)
  DINOv2MVSNet(args).forward(imgs, proj_matrices, depth_values, tmp)              <- DINOv2_mvsformer_model.py:68-179

Tensors crossing the seams keep the reference's logical shapes ([B,V,C,H,W] features, [B,D,H,W] volumes).  Feature
maps produced by FMT_with_pathway are channels-last in memory (a permuted view), which StageNet consumes
without a copy; any NCHW-contiguous input is converted by a transpose kernel.
"""
import math

import torch
import torch.nn as nn

from . import _lib, packing
from .config import load_args, stage_list, validate_args
from .params import build_fmt, build_fpn_decoder, build_fpn_encoder, build_stage, build_vit, build_vit_decoder


def _f32c(t):
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: expected a CUDA tensor (the hot path has no CPU fallback)")


def to_nhwc(x):
    """[N,C,H,W] (any strides) -> contiguous [N,H,W,C] buffer; zero-copy when x is already channels-last."""
    n, c, h, w = x.shape
    xp = x.permute(0, 2, 3, 1)
    if x.dtype == torch.float32 and xp.is_contiguous():
        return xp
    x = _f32c(x)
    out = torch.empty((n, h, w, c), device=x.device, dtype=torch.float32)
    _lib.call("mvsf_nchw_to_nhwc", x, out, n, c, h * w)
    return out


def to_nchw(x_nhwc):
    n, h, w, c = x_nhwc.shape
    out = torch.empty((n, c, h, w), device=x_nhwc.device, dtype=torch.float32)
    _lib.call("mvsf_nhwc_to_nchw", x_nhwc, out, n, c, h * w)
    return out


def _pack_f16(entry, flat, *args, query=None):
    """fp32 parameter blob on the device -> the fp16 buffer that the library's pack entry point
    mvsf_<entry>(*args, flat, out, size, stream) fills (install time, once).  query = (name, *query_args):
    mvsf_<name>(*query_args, &size) gives the buffer's size in bytes.  Without a query the buffer is the hi | lo split
    of the whole blob, 2 n halves, and size = n."""
    if query is None:
        size, halves = flat.numel(), 2 * flat.numel()
    else:
        size = _lib.size("mvsf_" + query[0], *query[1:])
        halves = size // 2
    out = torch.empty(halves, device=flat.device, dtype=torch.float16)
    _lib.call("mvsf_" + entry, *args, flat, out, size)
    return out


def split_weights_f16(flat):
    """fp32 weight blob on the device -> fp16 [hi | lo] blob for the wgmma GEMMs (install time, once)."""
    assert flat.numel() % 8 == 0
    return _pack_f16("split_weights_f16", flat)


def pack_unet_tc(kind, conv):
    """fp32 U-Net conv weights (the conv part of packing.pack_costreg_unet) on the device -> fp16 hi/lo weight slabs of
    the wgmma implicit-GEMM convolutions (install time, once)."""
    return _pack_f16("costreg_unet_pack_tc", conv, kind, query=("costreg_unet_tc_bytes",))


@torch.no_grad()
def homo_warping_3D_with_mask(src_fea, src_proj, ref_proj, depth_values):
    """Drop-in for the reference's finest seam, models/warping.py:69-109 (called at cost_volume.py:72):
    src_fea [B,C,H,W], src_proj / ref_proj [B,4,4] (already composed K@E), depth_values [B,D,H,W] or [B,D]
    -> (warped_src_fea [B,C,D,H,W] fp32, mask [B,D,H,W] bool; True where the sample falls outside the source image or
    behind the camera).  The hot path never materialises this volume (the warp is fused with the correlation);
    this standalone op exists for seam-level parity and for callers of the reference function."""
    _require_cuda(src_fea, "homo_warping_3D_with_mask(src_fea)")
    B, C, H, W = src_fea.shape
    D = depth_values.shape[1]
    dev = src_fea.device
    depth_values = _f32c(depth_values.to(dev))
    if depth_values.dim() == 2:  # warping.py:73-74
        depth_values = depth_values.view(B, D, 1, 1).expand(B, D, H, W).contiguous()
    sp, rp = _f32c(src_proj.to(dev)), _f32c(ref_proj.to(dev))
    homs = torch.empty((B, 12), device=dev, dtype=torch.float32)
    _lib.call("mvsf_homography_from_proj", sp, rp, B, homs)
    src = to_nhwc(src_fea)
    warped = torch.empty((B, C, D, H, W), device=dev, dtype=torch.float32)
    mask = torch.empty((B, D, H, W), device=dev, dtype=torch.uint8)
    for b in range(B):
        _lib.call("mvsf_homo_warp", src[b], homs[b], depth_values[b], warped[b], mask[b], C, D, H, W)
    return warped, mask.bool()


class _PackedMixin:
    """Packs the module's parameters for the CUDA library on first use / after load_state_dict.  A module implements
    _build_pack(device), which returns the dict of packed blobs; _pack(device) caches it per device."""

    def _pack(self, device):
        if self._packed is None or self._packed["device"] != device:
            self._packed = dict(self._build_pack(device), device=device)
        return self._packed

    def _invalidate(self, *a, **k):
        self._packed = None

    def repack(self):
        """Drop the packed (BN-folded, fp16-split) weight blobs; they are rebuilt on the next forward.  The cache is
        invalidated automatically by load_state_dict() and .to()/.cuda(); call this after in-place parameter edits
        (param.data.copy_, optimiser steps)."""
        self._packed = None

    def _init_packing(self):
        self._packed = None
        self.register_load_state_dict_post_hook(lambda m, k: m._invalidate())

    def _apply(self, fn, *a, **k):  # .to()/.cuda() move parameters: repack lazily
        self._packed = None
        return super()._apply(fn, *a, **k)


# =====================================================================================================
class StageNet(_PackedMixin, nn.Module):
    """Drop-in for the reference StageNet (models/cost_volume.py:21-133): same constructor arguments, parameter
    names, forward signature and output dict; eval-mode arithmetic (BatchNorm folded, depth_type 'ce')."""

    def __init__(self, args, ndepth, stage_idx):
        super().__init__()
        self.args = args
        self.fusion_type = args.get("fusion_type", "cnn")
        if self.fusion_type != "cnn":
            raise NotImplementedError(f"Not implemented fusion type: {self.fusion_type}.")
        self.ndepth = ndepth
        self.stage_idx = stage_idx
        self.cost_reg_type = args.get("cost_reg_type", ["Normal"] * 4)[stage_idx]
        self.depth_type = stage_list(args["depth_type"], stage_idx)
        bag = build_stage(args, ndepth, stage_idx)
        self.vis = bag.vis
        self.cost_reg = bag.cost_reg
        # per-view group correlations spilled between the two cost-volume passes; above this many bytes the stage
        # recomputes the gather in pass B instead (no spill buffer), so large inputs degrade instead of running out of memory
        self.corr_spill_budget_bytes = int(args.get("corr_spill_budget_bytes", 8 << 30))
        self._init_packing()

    # ---- packing
    def _build_pack(self, device):
        sd = {k: v for k, v in self.state_dict().items()}
        pk = {"vis": packing.pack_vis(sd, "vis.").to(device)}
        if self.cost_reg_type == "PureTransformerCostReg":
            cfg = self.args["transformer_config"][self.stage_idx]
            if (tuple(cfg["down_rate"]) != (2, 4, 4) or cfg["mid_channel"] != 64 or cfg["num_heads"] != 4
                    or cfg["mlp_ratio"] != 4):
                raise NotImplementedError("transformer regulariser: only the shipped geometry (down_rate (2,4,4), "
                                          "mid 64, 4 heads, mlp_ratio 4) is implemented")
            gemm, small = packing.pack_costreg_tr(sd, "cost_reg.", cfg["layer_num"])
            pk.update(kind="tr", layers=cfg["layer_num"], tc=split_weights_f16(gemm.to(device)))
        else:
            kind, conv, small = packing.pack_costreg_unet(sd, "cost_reg.")
            pk.update(kind=kind, tc=pack_unet_tc(kind, conv.to(device)))
        pk["w"] = small.to(device)
        return pk

    def _softmax_scale(self, n_tokens):
        tc = self.args["transformer_config"][self.stage_idx]
        scale = (tc["mid_channel"] // tc["num_heads"]) ** -0.5
        if tc.get("softmax_scale", None) is not None:  # attention.py:158-161
            scale *= math.log(n_tokens, tc["train_avg_length"])
        return scale

    # ---- one sample
    def _forward_one(self, feat_nhwc, proj, depth_values, tmp, position3d, pk, keep=False):
        V, H, W, C = feat_nhwc.shape
        D = depth_values.shape[0]
        dev = feat_nhwc.device
        G = stage_list(self.args["base_ch"], self.stage_idx)
        if G > C:
            raise AssertionError("G must <= C!")
        f32 = dict(device=dev, dtype=torch.float32)
        homs = torch.empty((V - 1) * 12, **f32)
        kinv = torch.empty(9, **f32)
        _lib.call("mvsf_compose_geometry", proj, V, homs, kinv)
        entropy = torch.empty((V - 1, H, W), **f32)
        vis = torch.empty((V - 1, H, W), **f32)
        volume = torch.empty((D, H, W, G), **f32)
        # spill plan (pass A stores the per-view group correlations, the aggregation streams them) unless the buffer would
        # exceed the budget: then both passes gather (TMA-staged window kernels at C = 8 / 16), no intermediate buffer
        two_gathers = _lib.lib().mvsf_warp_corr_plan(C, G, D, H, W, V, self.corr_spill_budget_bytes) == 1
        if not two_gathers:
            # pass A also stores the per-view group correlations; the view aggregation then streams them (no second gather)
            corr = torch.empty((V - 1, D, H, W, G), **f32)
            _lib.call("mvsf_warp_corr_entropy_store", feat_nhwc, homs, depth_values, entropy, corr, V, C, G, D, H, W)
            _lib.call("mvsf_vis_cnn", entropy, pk["vis"], vis, V - 1, H, W)
            _lib.call("mvsf_corr_aggregate", corr, vis, volume, V, G, D, H, W)
            del corr
        else:
            _lib.call("mvsf_warp_corr_entropy", feat_nhwc, homs, depth_values, entropy, V, C, G, D, H, W)
            _lib.call("mvsf_vis_cnn", entropy, pk["vis"], vis, V - 1, H, W)
            _lib.call("mvsf_warp_corr_aggregate", feat_nhwc, homs, depth_values, vis, volume, V, C, G, D, H, W)
        kept = dict(entropy=entropy, vis_weight=vis, volume_mean=volume.clone() if keep else None) if keep else None
        logits = torch.empty((D, H, W), **f32)
        if pk["kind"] == "tr":
            ws = _lib.workspace("mvsf_costreg_tr_workspace_bytes", G, D, H, W, device=dev)
            n_tok = (D // 2) * (H // 4) * (W // 4)
            _lib.call("mvsf_costreg_tr_forward", volume, position3d, pk["w"], pk["tc"], pk["tc"].numel() // 2, logits,
                      ws, ws.numel() * 4, G, D, H, W, pk["layers"], float(self._softmax_scale(n_tok)))
        else:
            ws = _lib.workspace("mvsf_costreg_unet_workspace_bytes", pk["kind"], G, D, H, W, device=dev)
            _lib.call("mvsf_costreg_unet_forward", pk["kind"], volume, pk["w"], pk["tc"], logits, ws, ws.numel() * 4,
                      G, D, H, W)
        prob = torch.empty((D, H, W), **f32)
        depth = torch.empty((H, W), **f32)
        conf = torch.empty((H, W), **f32)
        _lib.call("mvsf_softargmax", logits, depth_values, float(tmp), prob, depth, conf, D, H, W)
        return depth, prob, conf, logits, kept

    @torch.no_grad()
    def forward(self, features, proj_matrices, depth_values, tmp, position3d=None, keep_intermediates=False):
        if self.training:
            raise NotImplementedError("the hot path implements the eval-mode forward (test.py); call .eval()")
        if self.depth_type != "ce":
            raise NotImplementedError("depth_type must be 'ce'")
        _require_cuda(features, "StageNet.forward(features)")
        B, V, C, H, W = features.shape
        if V != proj_matrices.shape[1]:
            raise AssertionError("Different number of images and projection matrices")
        pk = self._pack(features.device)
        proj_matrices = _f32c(proj_matrices)
        depth_values = _f32c(depth_values)
        if depth_values.dim() == 2:  # [B,D] -> per-pixel hypotheses (warping.py:73 accepts both)
            depth_values = depth_values.view(B, -1, 1, 1).expand(B, depth_values.shape[1], H, W).contiguous()
        if position3d is not None:
            position3d = _f32c(position3d)
        outs = []
        for b in range(B):
            feat = to_nhwc(features[b])
            p3 = position3d[b] if position3d is not None else None
            outs.append(self._forward_one(feat, proj_matrices[b], depth_values[b], tmp, p3, pk, keep_intermediates))
        stack = (lambda i: torch.stack([o[i] for o in outs], 0)) if B > 1 else (lambda i: outs[0][i].unsqueeze(0))
        out = {"depth": stack(0), "prob_volume": stack(1), "photometric_confidence": stack(2),
               "depth_values": depth_values, "prob_volume_pre": stack(3)}
        if keep_intermediates:
            for k in ("entropy", "vis_weight", "volume_mean"):
                out[k] = torch.stack([o[4][k] for o in outs], 0)
        return out


# =====================================================================================================
class FMT_with_pathway(_PackedMixin, nn.Module):
    """Drop-in for the reference FMT_with_pathway (models/FMT.py:140-206)."""

    def __init__(self, base_channel=8, **kwargs):
        super().__init__()
        cfg = dict(kwargs)
        cfg["base_channel"] = base_channel
        if cfg.get("d_model", 64) != 64 or cfg.get("nhead", 4) != 4 or base_channel != 8:
            raise NotImplementedError("FMT: only the shipped geometry (d_model 64, 4 heads, base_channel 8)")
        if cfg.get("attention_type", "Linear") != "Linear":
            raise NotImplementedError("Unkown attention type", cfg.get("attention_type"))
        self.cfg = cfg
        bag = build_fmt(cfg)
        self.FMT = bag.FMT
        for k in (1, 2, 3):
            setattr(self, f"dim_reduction_{k}", getattr(bag, f"dim_reduction_{k}"))
            setattr(self, f"smooth_{k}", getattr(bag, f"smooth_{k}"))
        self.pe_dict = {}
        self._init_packing()

    def _build_pack(self, device):
        sd = {"FMT_module." + k: v for k, v in self.state_dict().items()}
        gemm, small = packing.pack_fmt(sd)
        tc = split_weights_f16(gemm.to(device))
        return {"w": small.to(device), "tc": tc}

    def _pe(self, H, W, device):
        """PositionEncodingSineNorm table (position_encoding.py:61-74) as [H*W, 64], cached per shape like the
        reference's pe_dict (constant per resolution; built with the same torch ops as the reference)."""
        key = (H, W, str(device))
        if key not in self.pe_dict:
            d_model, max_shape = 64, (128, 128)
            pe = torch.zeros((d_model, H, W))
            ypos = torch.ones((H, W)).cumsum(0).float().unsqueeze(0) * max_shape[0] / H
            xpos = torch.ones((H, W)).cumsum(1).float().unsqueeze(0) * max_shape[1] / W
            div = torch.exp(torch.arange(0, d_model // 2, 2).float() * (-math.log(10000.0) / (d_model // 2)))[:, None, None]
            pe[0::4] = torch.sin(xpos * div)
            pe[1::4] = torch.cos(xpos * div)
            pe[2::4] = torch.sin(ypos * div)
            pe[3::4] = torch.cos(ypos * div)
            self.pe_dict[key] = pe.permute(1, 2, 0).reshape(H * W, d_model).contiguous().to(device)
        return self.pe_dict[key]

    @torch.no_grad()
    def forward(self, features):
        f1 = features["stage1"]
        _require_cuda(f1, "FMT_with_pathway.forward(features)")
        B, V, C, H1, W1 = f1.shape
        assert C == 64, "FMT d_model must equal the stage-1 channel count"
        pk = self._pack(f1.device)
        pe = self._pe(H1, W1, f1.device)
        f32 = dict(device=f1.device, dtype=torch.float32)
        ws = _lib.workspace("mvsf_fmt_workspace_bytes", V, H1, W1, device=f1.device)
        outs = {k: [] for k in ("stage1", "stage2", "stage3", "stage4")}
        for b in range(B):
            ins = [_f32c(features[f"stage{k}"][b]) for k in (1, 2, 3, 4)]
            for k, (c, sc) in enumerate(((64, 1), (32, 2), (16, 4), (8, 8))):
                if tuple(ins[k].shape) != (V, c, H1 * sc, W1 * sc):
                    raise AssertionError(f"stage{k + 1} features must be [V,{c},{H1 * sc},{W1 * sc}], got {tuple(ins[k].shape)}")
            o = [torch.empty((V, H1 * sc, W1 * sc, c), **f32) for c, sc in ((64, 1), (32, 2), (16, 4), (8, 8))]
            _lib.call("mvsf_fmt_forward", *ins, pe, pk["w"], pk["tc"], pk["tc"].numel() // 2, *o, ws, ws.numel() * 4,
                      V, H1, W1)
            for k in range(4):
                outs[f"stage{k + 1}"].append(o[k])
        # logical [B,V,C,H,W]; channels-last in memory (StageNet consumes it without a copy)
        return {k: (v[0].unsqueeze(0) if B == 1 else torch.stack(v, 0)).permute(0, 1, 4, 2, 3) for k, v in outs.items()}


# =====================================================================================================
class HotPathNet(nn.Module):
    """FMT + 4-stage cascade from the FPN feature pyramid to the output dict: the part of
    DINOv2MVSNet.forward after feature extraction (DINOv2_mvsformer_model.py:117-179).  Sub-module names
    (FMT_module, fusions) and parameter names equal the reference's, so the hot-path subset of a reference
    checkpoint loads with load_state_dict(strict=True)."""

    def __init__(self, args):
        super().__init__()
        self.args = validate_args(load_args(args))
        a = self.args
        self.ndepths = a["ndepths"]
        self.depth_interals_ratio = a["depth_interals_ratio"]
        self.cost_reg_type = a.get("cost_reg_type", ["Normal"] * 4)
        self.use_pe3d = a.get("use_pe3d", False)
        self.FMT_module = FMT_with_pathway(**a["FMT_config"])
        self.fusions = nn.ModuleList([StageNet(a, self.ndepths[i], i) for i in range(len(self.ndepths))])

    @torch.no_grad()
    def forward_features(self, features, proj_matrices, depth_values, tmp=(5.0, 5.0, 5.0, 1.0), run_fmt=True,
                         keep_intermediates=False):
        return cascade_forward(self.FMT_module if run_fmt else None, self.fusions, self.args, features, proj_matrices,
                               depth_values, tmp, keep_intermediates)

    forward = forward_features


def cascade_forward(fmt_module, fusions, args, features, proj_matrices, depth_values, tmp, keep_intermediates=False):
    """DINOv2_mvsformer_model.py:117-179 with the element-wise glue (hypothesis scheduling, 3-D positions, confidence
    averaging) as CUDA kernels.  `fusions[i]` must be this package's StageNet."""
    ndepths, ratios = args["ndepths"], args["depth_interals_ratio"]
    if fmt_module is not None:
        features = fmt_module.forward(features)
    last = features[f"stage{len(ndepths)}"]
    _require_cuda(last, "features")
    B, Hf, Wf = last.shape[0], last.shape[3], last.shape[4]
    dev = last.device
    f32 = dict(device=dev, dtype=torch.float32)
    depth_values = _f32c(depth_values.to(dev))
    Dn = depth_values.shape[1]
    prob_maps = torch.empty((B, Hf, Wf), **f32)
    stats = torch.zeros(8, **f32)   # x/y extents of the 3-D positions + depth range, shared by the whole batch
    have_extents = False            # the reference computes them on the first stage that builds the PE and reuses them
    outputs, so = {}, None
    for s in range(len(ndepths)):
        pm = _f32c(proj_matrices[f"stage{s + 1}"].to(dev))
        f = features[f"stage{s + 1}"]
        _, V, C, H, W = f.shape
        D = ndepths[s]
        ds = torch.empty((B, D, H, W), **f32)
        for b in range(B):
            if s == 0:
                _lib.call("mvsf_init_inverse_range", depth_values[b], Dn, ds[b], D, H, W)
            else:
                _lib.call("mvsf_schedule_inverse_range", so["depth"][b], so["depth_values"][b], so["depth_values"].shape[1],
                          float(ratios[s]), ds[b], D, H, W)
        p3d = None
        if args["cost_reg_type"][s] != "Normal" and args.get("use_pe3d", False):
            # position_encoding.py:138-161: extents (first PE stage only) and depth_values.min()/max() are reductions
            # over the WHOLE batch (DINOv2_mvsformer_model.py:152-160)
            p3d = torch.empty((B, 3, D, H, W), **f32)
            kinvs = torch.empty((B, 9), **f32)
            homs = torch.empty((V - 1) * 12, **f32)
            for b in range(B):
                _lib.call("mvsf_compose_geometry", pm[b], V, homs, kinvs[b])
                if not have_extents:
                    _lib.call("mvsf_position3d", kinvs[b], ds[b], None, 0, stats, 2 if b == 0 else 3, None, D, H, W)
            if not have_extents:
                _lib.call("mvsf_position3d", None, None, depth_values, B * Dn, stats, 4, None, D, H, W)
                have_extents = True
            for b in range(B):
                _lib.call("mvsf_position3d", kinvs[b], ds[b], None, 0, stats, 5, p3d[b], D, H, W)
        so = fusions[s].forward(f, pm, ds, tmp=tmp[s], position3d=p3d, keep_intermediates=keep_intermediates)
        outputs[f"stage{s + 1}"] = so
        conf = so["photometric_confidence"]
        for b in range(B):
            _lib.call("mvsf_conf_accumulate", conf[b], H, W, prob_maps[b], Hf, Wf, 1.0 / len(ndepths), 1 if s == 0 else 0)
        outputs.update(so)
    outputs["refined_depth"] = so["depth"]
    outputs["photometric_confidence"] = prob_maps
    outputs["features"] = features
    return outputs


# =====================================================================================================
def _check_fpn_config(feat_chs, norm_type="BN"):
    if list(feat_chs) != [8, 16, 32, 64]:
        raise NotImplementedError(f"FPN: only feat_chs [8, 16, 32, 64] is implemented, got {list(feat_chs)}")
    if norm_type != "BN":
        raise NotImplementedError(f"FPN: only norm_type 'BN' is implemented, got {norm_type!r}")


def _check_fpn_size(H, W):
    if H % 8 or W % 8 or H < 8 or W < 8:
        raise ValueError(f"FPN: image height and width must be positive multiples of 8 (the decoder adds exact 2x "
                         f"upsamplings), got {H}x{W}")


class FPNEncoder(_PackedMixin, nn.Module):
    """Drop-in for the reference FPNEncoder (models/module.py:208-239), eval mode: returns [conv01, conv11, conv21, conv31]
    as fp32 [N,C,h,w] views of channels-last buffers.  Any float dtype and strides are accepted."""

    def __init__(self, feat_chs, norm_type="BN"):
        super().__init__()
        _check_fpn_config(feat_chs, norm_type)
        build_fpn_encoder(self)
        self._init_packing()

    def _build_pack(self, device):
        conv, small = packing.pack_fpn_encoder(self.state_dict(), "")
        tc = _pack_f16("fpn_pack_tc", conv.to(device), 0, query=("fpn_tc_bytes", 0))
        return {"w": small.to(device), "tc": tc}

    @torch.no_grad()
    def forward(self, x, vit_feat=None):
        """vit_feat [V,64,H/8,W/8] (DINOv2MVSNet): conv31 is returned as conv31 + vit_feat[n % V], added in the last
        layer's epilogue"""
        if self.training:
            raise NotImplementedError("the FPN hot path implements the eval-mode forward; call .eval()")
        N, C, H, W = x.shape
        if C != 3:
            raise AssertionError(f"FPNEncoder expects [N,3,H,W] images, got {tuple(x.shape)}")
        _check_fpn_size(H, W)
        _require_cuda(x, "FPNEncoder.forward(x)")
        pk = self._pack(x.device)
        x = _f32c(x)
        f32 = dict(device=x.device, dtype=torch.float32)
        outs = [torch.empty((N, H // s, W // s, c), **f32) for c, s in ((8, 1), (16, 2), (32, 4), (64, 8))]
        ws = _lib.workspace("mvsf_fpn_encoder_workspace_bytes", N, H, W, device=x.device)
        if vit_feat is None:
            _lib.call("mvsf_fpn_encoder_forward", x, pk["w"], pk["tc"], *outs, ws, ws.numel() * 4, N, H, W)
        else:
            V = vit_feat.shape[0]
            if tuple(vit_feat.shape) != (V, 64, H // 8, W // 8):
                raise AssertionError(f"FPNEncoder: vit_feat must be [V,64,{H // 8},{W // 8}], got {tuple(vit_feat.shape)}")
            _require_cuda(vit_feat, "FPNEncoder.forward(vit_feat)")
            vit = to_nhwc(vit_feat)
            _lib.call("mvsf_fpn_encoder_vit_forward", x, vit, V, pk["w"], pk["tc"], *outs, ws, ws.numel() * 4, N, H, W)
        return [o.permute(0, 3, 1, 2) for o in outs]


class FPNDecoder(_PackedMixin, nn.Module):
    """Drop-in for the reference FPNDecoder (models/module.py:242-270), eval mode: returns [out0, out1, out2, out3] as
    NCHW-contiguous fp32.  Inputs may be any float dtype and strides (bf16 appears under autocast after conv31 + vit_feat)."""

    def __init__(self, feat_chs):
        super().__init__()
        _check_fpn_config(feat_chs)
        build_fpn_decoder(self)
        self._init_packing()

    def _build_pack(self, device):
        conv, small = packing.pack_fpn_decoder(self.state_dict(), "")
        tc = _pack_f16("fpn_pack_tc", conv.to(device), 1, query=("fpn_tc_bytes", 1))
        return {"w": small.to(device), "tc": tc}

    @torch.no_grad()
    def forward(self, conv01, conv11, conv21, conv31):
        if self.training:
            raise NotImplementedError("the FPN hot path implements the eval-mode forward; call .eval()")
        N, _, H, W = conv01.shape
        _check_fpn_size(H, W)
        ins = (conv01, conv11, conv21, conv31)
        for t, c, s in zip(ins, (8, 16, 32, 64), (1, 2, 4, 8)):
            if tuple(t.shape) != (N, c, H // s, W // s):
                raise AssertionError(f"FPNDecoder: expected a [{N},{c},{H // s},{W // s}] map, got {tuple(t.shape)}")
            _require_cuda(t, "FPNDecoder.forward")
        pk = self._pack(conv01.device)
        ins = [to_nhwc(t) for t in ins]
        f32 = dict(device=conv01.device, dtype=torch.float32)
        outs = [torch.empty((N, c, H // s, W // s), **f32) for c, s in ((64, 8), (32, 4), (16, 2), (8, 1))]
        ws = _lib.workspace("mvsf_fpn_decoder_workspace_bytes", N, H, W, device=conv01.device)
        _lib.call("mvsf_fpn_decoder_forward", *ins, pk["w"], pk["tc"], *outs, ws, ws.numel() * 4, N, H, W)
        return outs


# =====================================================================================================
# the shipped decoder_cfg (config/mvsformer++.json); the last five default to these values in the reference
# (module.py:280-298, block.py:332-333)
_VIT_DECODER_CFG = dict(d_model=768, nhead=12, attention_type="Linear", ffn_type="ffn", self_cross_types=None,
                        post_norm=False, pre_norm_query=True, no_combine_norm=False)
_VIT_DECODER_OPTIONAL = ("ffn_type", "self_cross_types", "post_norm", "pre_norm_query", "no_combine_norm")


def _check_vit_decoder_config(args):
    dino = args["dino_cfg"]
    cfg = dino["decoder_cfg"]
    for k, want in _VIT_DECODER_CFG.items():
        got = cfg.get(k, want) if k in _VIT_DECODER_OPTIONAL else cfg[k]
        if got != want:
            raise NotImplementedError(f"CrossVITDecoder: only the shipped decoder_cfg is implemented ({k} = {want!r}), "
                                      f"got {k} = {got!r}")
    if cfg.get("init_values") is None:
        raise NotImplementedError("CrossVITDecoder: decoder_cfg init_values must be set (LayerScale)")
    if dino.get("cross_interval_layers") != 3:
        raise NotImplementedError(f"CrossVITDecoder: only cross_interval_layers = 3 is implemented, got "
                                  f"{dino.get('cross_interval_layers')!r}")
    for k, want in (("vit_ch", 768), ("out_ch", 64)):
        if args.get(k) != want:
            raise NotImplementedError(f"CrossVITDecoder: only {k} = {want} is implemented, got {args.get(k)!r}")


class CrossVITDecoder(_PackedMixin, nn.Module):
    """Drop-in for the reference CrossVITDecoder (models/module.py:273-364), eval mode, shipped decoder_cfg: same
    constructor argument (arch.args), parameter names and forward signature.  x = [x0, x1, x2], each [B,V,h*w,768] in any
    float dtype and strides (bf16 under autocast, non-contiguous [:, 1:] slices); vit_shape = (B, V, h, w, 768).  Returns
    fp32 [B*V,64,4h,4w] as a view of a channels-last buffer.  Fmats is accepted and ignored, as in the reference."""

    def __init__(self, args):
        super().__init__()
        _check_vit_decoder_config(args)
        cfg = args["dino_cfg"]["decoder_cfg"]
        build_vit_decoder(self, init_values=cfg["init_values"], prev_values=cfg.get("prev_values", 0.5))
        self._init_packing()

    def _build_pack(self, device):
        gemm, small = packing.pack_vit_decoder(self.state_dict())
        tc = split_weights_f16(gemm.to(device))
        return {"w": small.to(device), "tc": tc}

    @torch.no_grad()
    def forward(self, x, Fmats=None, vit_shape=None):
        if self.training:
            raise NotImplementedError("the ViT decoder implements the eval-mode forward; call .eval()")
        B, V, h, w, C = vit_shape
        if len(x) != 3:
            raise AssertionError(f"CrossVITDecoder expects the three interval feature maps, got {len(x)}")
        for t in x:
            if tuple(t.shape) != (B, V, h * w, C) or C != 768:
                raise AssertionError(f"CrossVITDecoder: expected [{B},{V},{h * w},768] tokens, got {tuple(t.shape)}")
            _require_cuda(t, "CrossVITDecoder.forward(x)")
        xs = []
        for t in x:
            t = _f32c(t)
            xs.append(t if t.data_ptr() % 16 == 0 else t.clone())
        dev = xs[0].device
        pk = self._pack(dev)
        f32 = dict(device=dev, dtype=torch.float32)
        out = torch.empty((B * V, 4 * h, 4 * w, 64), **f32)
        ws = _lib.workspace("mvsf_vit_decoder_workspace_bytes", B, V, h, w, device=dev)
        _lib.call("mvsf_vit_decoder_forward", *xs, pk["w"], pk["tc"], out, ws, ws.numel() * 4, B, V, h, w)
        return out.permute(0, 3, 1, 2)


# =====================================================================================================
def _check_vit_config(img_size, patch_size, in_chans, embed_dim, depth, num_heads, mlp_ratio, qkv_bias, ffn_bias,
                      proj_bias, init_values, act_layer, ffn_layer, block_chunks, kwargs):
    shipped = dict(img_size=(img_size, 518), patch_size=(patch_size, 14), in_chans=(in_chans, 3),
                   embed_dim=(embed_dim, 768), depth=(depth, 12), num_heads=(num_heads, 12), mlp_ratio=(mlp_ratio, 4),
                   qkv_bias=(qkv_bias, True), ffn_bias=(ffn_bias, True), proj_bias=(proj_bias, True),
                   act_layer=(act_layer, nn.GELU), ffn_layer=(ffn_layer, "mlp"), block_chunks=(block_chunks, 0),
                   cross_interval_layers=(kwargs.get("cross_interval_layers"), 3),
                   softmax_scale=(kwargs.get("softmax_scale"), None), dino_layer_idxs=(kwargs.get("dino_layer_idxs"), None))
    for k, (got, want) in shipped.items():
        if got != want:
            raise NotImplementedError(f"DinoVisionTransformer: only the shipped ViT-B/14 is implemented ({k} = {want!r}), "
                                      f"got {k} = {got!r}")
    if not init_values:
        raise NotImplementedError(f"DinoVisionTransformer: init_values must be set (LayerScale), got {init_values!r}")


class DinoVisionTransformer(_PackedMixin, nn.Module):
    """Drop-in for the reference DinoVisionTransformer (models/dino/dinov2.py:43-266) as DINOv2_mvsformer_model.py:40-41
    builds it (vit_base, img_size 518, patch 14, LayerScale, block_chunks 0, mlp ffn, cross_interval_layers 3), eval mode:
    same parameter names (load_state_dict(strict=True) of the reference's vit.* keys), embed_dim, patch_size and
    forward_interval_features(x, masks=None).  x [n,3,14 gh,14 gw] in any float dtype and strides; returns the outputs of
    blocks 3 and 7 and norm(x) after block 11 without the cls token, each fp32 [n, gh gw, 768], contiguous.
    use_flash2_dino selects the same math in the reference and is accepted either way."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0,
                 qkv_bias=True, ffn_bias=True, proj_bias=True, drop_path_rate=0.0, drop_path_uniform=False,
                 init_values=None, act_layer=nn.GELU, ffn_layer="mlp", block_chunks=1, **kwargs):
        super().__init__()
        _check_vit_config(img_size, patch_size, in_chans, embed_dim, depth, num_heads, mlp_ratio, qkv_bias, ffn_bias,
                          proj_bias, init_values, act_layer, ffn_layer, block_chunks, kwargs)
        self.num_features = self.embed_dim = embed_dim
        self.num_tokens = 1
        self.n_blocks = depth
        self.num_heads = num_heads
        self.patch_size = patch_size
        self.cross_interval_layers = kwargs["cross_interval_layers"]
        self.dino_layer_idxs = None
        build_vit(self, init_values=float(init_values))
        for prm in self.parameters():   # frozen, as in the reference (dinov2.py:164-165)
            prm.requires_grad = False
        self._init_packing()

    def _build_pack(self, device):
        gemm, small = packing.pack_vit(self.state_dict())
        tc = split_weights_f16(gemm.to(device))
        return {"w": small.to(device), "tc": tc, "pos": {}}

    def _pos(self, pk, gh, gw):
        """interpolated pos_embed of the grid (a weight transform), cached with the packed weights"""
        if (gh, gw) not in pk["pos"]:
            pk["pos"][(gh, gw)] = packing.vit_pos_embed(self.pos_embed, gh, gw).to(pk["device"])
        return pk["pos"][(gh, gw)]

    @torch.no_grad()
    def forward_interval_features(self, x, masks=None):
        if isinstance(x, list):
            raise NotImplementedError("DinoVisionTransformer: list inputs (forward_features_list) are not implemented")
        if masks is not None:
            raise NotImplementedError("DinoVisionTransformer: masks are not implemented")
        H, W = x.shape[-2:]
        ps = self.patch_size
        assert H % ps == 0, f"Input image height {H} is not a multiple of patch height {ps}"
        assert W % ps == 0, f"Input image width {W} is not a multiple of patch width: {ps}"
        return self._interval_features(x, H // ps, W // ps, resize=False)

    @torch.no_grad()
    def forward_interval_features_resized(self, x, size):
        """forward_interval_features(F.interpolate(x, size, mode="bicubic", align_corners=False)) with the resize done
        inside the patch embedding (DINOv2_mvsformer_model.py:76-78): the resized images are never stored.  size =
        (vit_h, vit_w), multiples of the patch size."""
        vh, vw = size
        ps = self.patch_size
        if vh % ps or vw % ps or vh < ps or vw < ps:
            raise ValueError(f"DinoVisionTransformer: the resized size must be positive multiples of {ps}, got {vh}x{vw}")
        return self._interval_features(x, vh // ps, vw // ps, resize=True)

    def _interval_features(self, x, gh, gw, resize):
        if self.training:
            raise NotImplementedError("the ViT implements the eval-mode forward; call .eval()")
        n, c, H, W = x.shape
        if c != 3:
            raise AssertionError(f"DinoVisionTransformer expects [n,3,H,W] images, got {tuple(x.shape)}")
        _require_cuda(x, "DinoVisionTransformer.forward_interval_features(x)")
        x = _f32c(x)
        if x.data_ptr() % 16:
            x = x.clone()
        pk = self._pack(x.device)
        pos = self._pos(pk, gh, gw)
        f32 = dict(device=x.device, dtype=torch.float32)
        P = gh * gw
        # out0 / out1 also carry the residual stream: the n cls rows follow the n * P patch rows
        outs = [torch.empty((n * (P + 1), 768), **f32), torch.empty((n * (P + 1), 768), **f32),
                torch.empty((n * P, 768), **f32)]
        ws = _lib.workspace("mvsf_vit_workspace_bytes", n, gh, gw, device=x.device)
        if resize:
            _lib.call("mvsf_vit_forward_image", x, H, W, pos, pk["w"], pk["tc"], *outs, ws, ws.numel() * 4, n, gh, gw)
        else:
            _lib.call("mvsf_vit_forward", x, pos, pk["w"], pk["tc"], *outs, ws, ws.numel() * 4, n, gh, gw)
        return [o[:n * P].view(n, P, 768) for o in outs]


def vit_base(patch_size=16, **kwargs):
    """models/dino/dinov2.py:388-398: the ViT-B DinoVisionTransformer (embed 768, depth 12, 12 heads, mlp_ratio 4)."""
    return DinoVisionTransformer(patch_size=patch_size, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, **kwargs)


# =====================================================================================================
class DINOv2MVSNet(nn.Module):
    """Drop-in for the reference DINOv2MVSNet (models/networks/DINOv2_mvsformer_model.py:22-179), eval mode: same
    constructor argument (config["arch"]["args"]), sub-module and parameter names (a reference checkpoint loads with
    load_state_dict(strict=True)) and forward(imgs, proj_matrices, depth_values, tmp) -> the reference's output dict.
    The whole forward, images to depth maps, runs on this package's kernels on the current stream:
      ViT on the full-resolution images with the bicubic resize fused into its patch embedding -> ViT decoder ->
      FPN encoder over all B V images with + vit_feat in conv31's epilogue -> FPN decoder over all B V images, whose NCHW
      outputs are the [B,V,C,h,w] stage features as views -> FMT + cascade (cascade_forward).
    As in the reference's eval forward (:88), image (b, v) receives batch item 0's vit_feat[v]: the ViT and its decoder run
    on batch item 0's V images only.  vit_path is not read (a checkpoint carries the vit.* keys).  Images may be any float
    dtype and strides; bf16 autocast does not change the arithmetic."""

    def __init__(self, args):
        super().__init__()
        self.args = validate_args(load_args(args))
        a = self.args
        self.ndepths = a["ndepths"]
        self.depth_interals_ratio = a["depth_interals_ratio"]
        self.inverse_depth = a.get("inverse_depth", False)
        self.use_pe3d = a.get("use_pe3d", False)
        self.cost_reg_type = a.get("cost_reg_type", ["Normal"] * 4)
        self.encoder = FPNEncoder(feat_chs=a["feat_chs"])
        self.decoder = FPNDecoder(feat_chs=a["feat_chs"])
        self.vit_args = a
        self.freeze_vit = a.get("freeze_vit", True)
        self.vit = vit_base(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp",
                            **a.get("dino_cfg", {}))
        self.decoder_vit = CrossVITDecoder(a)
        self.FMT_module = FMT_with_pathway(**a["FMT_config"])
        self.fusions = nn.ModuleList([StageNet(a, self.ndepths[i], i) for i in range(len(self.ndepths))])

    def vit_grid(self, H, W):
        """the ViT's patch grid for H x W images: vit_h = int(H * rescale // 14 * 14) (DINOv2_mvsformer_model.py:72)"""
        rescale = self.vit_args["rescale"]
        return int(H * rescale // 14 * 14) // 14, int(W * rescale // 14 * 14) // 14

    @torch.no_grad()
    def extract_features(self, imgs):
        """DINOv2_mvsformer_model.py:70-98: imgs [B,V,3,H,W] -> the FPN pyramid {stage1..4: [B,V,C,h,w]} (NCHW views)"""
        if self.training:
            raise NotImplementedError("DINOv2MVSNet implements the eval-mode forward (test.py); call .eval()")
        B, V, C, H, W = imgs.shape
        if C != 3:
            raise AssertionError(f"DINOv2MVSNet expects [B,V,3,H,W] images, got {tuple(imgs.shape)}")
        if H % 32 or W % 32 or H < 32 or W < 32:
            raise ValueError(f"DINOv2MVSNet: image height and width must be positive multiples of 32 (the stage-1 "
                             f"regulariser downsamples H/8 x W/8 by 4), got {H}x{W}")
        gh, gw = self.vit_grid(H, W)
        if 4 * gh != H // 8 or 4 * gw != W // 8:
            raise NotImplementedError(f"DINOv2MVSNet: the ViT grid {gh}x{gw} (rescale {self.vit_args['rescale']}) must give "
                                      f"vit_feat at H/8 x W/8 = {H // 8}x{W // 8}; the bilinear vit_feat resize of "
                                      "DINOv2_mvsformer_model.py:80-82 is not implemented")
        _require_cuda(imgs, "DINOv2MVSNet.forward(imgs)")
        imgs = _f32c(imgs)
        if imgs.data_ptr() % 16:
            imgs = imgs.clone()
        vit_out = self.vit.forward_interval_features_resized(imgs[0], (14 * gh, 14 * gw))
        vit_feat = self.decoder_vit.forward([o.view(1, V, gh * gw, 768) for o in vit_out], vit_shape=(1, V, gh, gw, 768))
        conv = self.encoder.forward(imgs.view(B * V, 3, H, W), vit_feat=vit_feat)
        outs = self.decoder.forward(*conv)
        return {f"stage{k + 1}": o.view(B, V, *o.shape[1:]) for k, o in enumerate(outs)}

    @torch.no_grad()
    def forward(self, imgs, proj_matrices, depth_values, tmp=(5.0, 5.0, 5.0, 1.0)):
        features = self.extract_features(imgs)
        return cascade_forward(self.FMT_module, self.fusions, self.args, features, proj_matrices, depth_values, tmp)


# =====================================================================================================
def install(model, args=None, feature_pyramid=False, vit_decoder=False, vit=False):
    """Rebinds the hot-path seams of a reference-constructed DINOv2MVSNet (models/networks/DINOv2_mvsformer_model.py)
    to the CUDA path: model.FMT_module and model.fusions[i] are replaced by this package's modules carrying the
    same weights (state_dict round trip, strict).  With feature_pyramid=True model.encoder and model.decoder (the FPN,
    DINOv2_mvsformer_model.py:34-35,87-89) are replaced as well, with vit_decoder=True model.decoder_vit
    (CrossVITDecoder, DINOv2_mvsformer_model.py:43,64), and with vit=True model.vit (the DINOv2 ViT-B backbone,
    DINOv2_mvsformer_model.py:40-41,55-59).  The bicubic image resize in front of the ViT stays PyTorch.  Returns model."""
    if vit:
        dino_cfg = (getattr(model, "vit_args", model.args) if args is None else load_args(args)).get("dino_cfg", {})
        v = vit_base(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp", **dino_cfg)
        v.load_state_dict(model.vit.state_dict(), strict=True)
        model.vit = v.to(next(model.vit.parameters()).device).eval()
    if vit_decoder:
        dec = CrossVITDecoder(getattr(model, "vit_args", model.args) if args is None else load_args(args))
        dec.load_state_dict(model.decoder_vit.state_dict(), strict=True)
        model.decoder_vit = dec.to(next(model.decoder_vit.parameters()).device).eval()
    if feature_pyramid:
        feat_chs = (model.args if args is None else load_args(args)).get("feat_chs", [8, 16, 32, 64])
        if any(isinstance(m, nn.InstanceNorm2d) for m in model.encoder.modules()):
            raise NotImplementedError("FPN: only norm_type 'BN' is implemented")
        dev = next(model.encoder.parameters()).device
        enc, dec = FPNEncoder(feat_chs), FPNDecoder(feat_chs)
        enc.load_state_dict(model.encoder.state_dict(), strict=True)
        dec.load_state_dict(model.decoder.state_dict(), strict=True)
        model.encoder = enc.to(dev).eval()
        model.decoder = dec.to(dev).eval()
    args = validate_args(load_args(args if args is not None else model.args))
    dev = next(model.parameters()).device
    fmt = FMT_with_pathway(**args["FMT_config"])
    fmt.load_state_dict(model.FMT_module.state_dict(), strict=True)
    model.FMT_module = fmt.to(dev).eval()
    new = []
    for i, old in enumerate(model.fusions):
        st = StageNet(args, args["ndepths"][i], i)
        st.load_state_dict(old.state_dict(), strict=True)
        new.append(st.to(dev).eval())
    model.fusions = nn.ModuleList(new)
    return model
