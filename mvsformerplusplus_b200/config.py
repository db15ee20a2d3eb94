"""Config schema of the depth-inference hot path.

The schema is the reference's ``arch.args`` block (reference: config/mvsformer++.json:10-115,
consumed at models/networks/DINOv2_mvsformer_model.py:25-53 and models/cost_volume.py:22-49).
Only the keys the hot path reads are interpreted; every other key is carried through untouched so a
reference JSON file can be passed in as-is.
"""
import copy
import json

# Defaults equal to the shipped DTU configuration (values restated from config/mvsformer++.json).
_FMT = dict(attention_type="Linear", base_channel=8, d_model=64, nhead=4, init_values=1.0,
            layer_names=["self", "cross", "self", "cross"], ffn_type="ffn",
            softmax_scale="entropy_invariance", train_avg_length=12185, attn_backend="FLASH2",
            self_cross_types=None, post_norm=False, pre_norm_query=False)
_TR = dict(base_channel=8, mid_channel=64, num_heads=4, down_rate=[2, 4, 4], mlp_ratio=4, layer_num=6,
           drop=0.0, attn_drop=0.0, position_encoding=True, attention_type="FLASH2",
           softmax_scale="entropy_invariance", train_avg_length=12185, use_pe_proj=True)

DEFAULT_ARGS = dict(
    model_type="DINOv2-base", depth_type=["ce", "ce", "ce", "ce"], fusion_type="cnn", inverse_depth=True,
    base_ch=[8, 8, 8, 8], ndepths=[32, 16, 8, 4], feat_chs=[8, 16, 32, 64],
    depth_interals_ratio=[4.0, 2.67, 1.5, 1.0], FMT_config=_FMT,
    cost_reg_type=["PureTransformerCostReg", "Normal", "Normal", "Normal"], use_pe3d=True,
    transformer_config=[_TR], model_th=8)


def default_args():
    return copy.deepcopy(DEFAULT_ARGS)


def load_args(path_or_dict):
    """Accepts a reference config JSON path, the parsed JSON, or an ``arch.args`` dict."""
    if isinstance(path_or_dict, str):
        with open(path_or_dict) as f:
            path_or_dict = json.load(f)
    d = path_or_dict
    if "arch" in d:
        d = d["arch"]["args"]
    out = default_args()
    out.update(copy.deepcopy(dict(d)))
    return out


def stage_list(value, stage_idx):
    return value[stage_idx] if isinstance(value, (list, tuple)) else value


def validate_args(args):
    """Raise exactly where the reference raises (models/cost_volume.py:39,87,95; FMT.py:45-51)."""
    if args.get("fusion_type", "cnn") != "cnn":
        raise NotImplementedError(f"Not implemented fusion type: {args.get('fusion_type')}.")
    if not args.get("inverse_depth", False):
        raise NotImplementedError("the hot path implements the shipped inverse_depth=True scheduling only")
    fm = args["FMT_config"]
    if fm.get("attention_type") != "Linear":
        raise NotImplementedError("Unkown attention type", fm.get("attention_type"))
    if fm.get("ffn_type", "ffn") != "ffn":
        raise NotImplementedError(f"Unknown FFN...{fm.get('ffn_type')}")
    if fm.get("post_norm", False) or fm.get("pre_norm_query", True):
        raise NotImplementedError("FMT blocks: only pre-norm with pre_norm_query=False (shipped config)")
    if list(fm.get("layer_names")) != ["self", "cross", "self", "cross"]:
        raise NotImplementedError("FMT layer_names must be [self,cross,self,cross] (shipped config)")
    for s, t in enumerate(args["cost_reg_type"]):
        dt = stage_list(args["depth_type"], s)
        if dt != "ce":
            raise NotImplementedError("depth_type must be 'ce' (shipped config)")
        if t == "PureTransformerCostReg":
            tc = args["transformer_config"][s]
            if tc.get("attention_type", "FLASH2") not in ("FLASH2", "FLASH1"):
                raise NotImplementedError(f"Unkown Attention Type {tc.get('attention_type')}")
            if not (tc.get("position_encoding", True) and tc.get("use_pe_proj", True)):
                raise NotImplementedError("transformer regulariser: pe_proj path only (shipped config)")
            # options the CUDA path hard-codes (FlashAttnBlock kwargs, models/module.py:536-582): a non-default value
            # would load with strict=True and silently compute different arithmetic, so reject it at construction
            if not tc.get("post_norm", True):
                raise NotImplementedError("transformer regulariser: post_norm=False is not implemented (shipped: post-norm)")
            if tc.get("qkv_bias", False):
                raise NotImplementedError("transformer regulariser: qkv_bias=True is not implemented (shipped: no qkv bias)")
            if not tc.get("proj_bias", True) or not tc.get("ffn_bias", True):
                raise NotImplementedError("transformer regulariser: proj_bias / ffn_bias must be True (shipped config)")
            if tuple(tc.get("down_rate", (2, 4, 4))) != (2, 4, 4) or tc.get("mid_channel", 64) != 64 or \
                    tc.get("num_heads", 4) != 4 or tc.get("mlp_ratio", 4) != 4:
                raise NotImplementedError("transformer regulariser: only the shipped geometry (down_rate (2,4,4), "
                                          "mid_channel 64, 4 heads, mlp_ratio 4) is implemented")
            if stage_list(args["base_ch"], s) != 8 or tc.get("base_channel", 8) != 8:
                raise NotImplementedError("transformer regulariser: base channel must be 8 (shipped config)")
        elif t != "Normal":
            raise NotImplementedError(f"cost_reg_type {t}")
    return args
