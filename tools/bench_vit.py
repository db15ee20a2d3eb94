"""DINOv2 ViT-B/14 backbone (forward_interval_features) for all views of one depth map on cuda:0: the CUDA path
(hotpath.DinoVisionTransformer) against the same layers in torch on the GPU (oracle/vit.py), in fp32 (TF32 off) and
under bf16 autocast as the reference's test.py:250 runs them; plus the softmax attention alone (mvsf_vit_attention_forward,
12 launches per depth map in the backbone).  Device events, warm-up, >= 20 timed repetitions (median reported).  Prints
one JSON line.

  python tools/bench_vit.py [--reps 20] [--warmup 3] [--workloads dtu,tt]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import vit as OVT  # noqa: E402
from tools.bench_fpn import card, timed  # noqa: E402

# ViT inputs at the shipped rescale 0.4375 and patch 14: DTU 1152x1536 -> 504x672 (36x48 patches),
# T&T 1088x1920 -> 476x840 (34x60)
WORKLOADS = {"dtu": (5, 36, 48), "tt": (10, 34, 60)}
KW = dict(img_size=518, patch_size=14, init_values=1.0, block_chunks=0, ffn_layer="mlp", cross_interval_layers=3)


def vit_gflop(n, gh, gw):
    """Algorithmic GFLOP (2 x multiply-adds from the layer shapes): (linears incl. the patch conv, softmax attention)."""
    d, hid, P = 768, 3072, gh * gw
    N = P + 1
    lin = 2 * n * P * 588 * d + 12 * 2 * n * N * d * (3 * d + d + 2 * hid)
    att = 12 * 2 * 2 * n * N * N * d     # Q K^T and P V over 12 heads of 64
    return lin / 1e9, att / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="dtu,tt")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit: no CUDA device (timings are only taken on the GPU)")
    from mvsformerplusplus_b200 import _lib, vit_base
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = torch.nn.Module()
    m.vit = vit_base(**KW)
    sd = synth.randomize_state_dict(m, seed=82)
    vit = m.vit.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    name, power = card()
    res = {"bench": "vit", "device": name, "power_limit": power, "reps": a.reps, "warmup": a.warmup, "workloads": {}}
    for wl in a.workloads.split(","):
        n, gh, gw = WORKLOADS[wl]
        img = synth.make_images(n, 14 * gh, 14 * gw, seed=1).to(dev)

        def run_cuda():
            return vit.forward_interval_features(img)

        def run_torch():
            with torch.no_grad():
                return OVT.vit_interval_features(img, sd_dev)

        def run_bf16():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return OVT.vit_interval_features(img, sd_dev)

        got, want, lo = run_cuda(), run_torch(), run_bf16()
        diff = [float((g - w).abs().max()) for g, w in zip(got, want)]
        diff_bf16 = [float((x.float() - w).abs().max()) for x, w in zip(lo, want)]
        scale = [float(w.abs().max()) for w in want]
        del got, want, lo
        lin, att = vit_gflop(n, gh, gw)
        arms = {}
        for arm, fn in (("cuda", run_cuda), ("torch_fp32", run_torch), ("torch_bf16_autocast", run_bf16)):
            ms = timed(fn, a.warmup, a.reps)
            torch.cuda.empty_cache()
            arms[arm] = {"ms_per_depth_map": round(ms, 3), "tflops": round((lin + att) / ms, 2)}
        # the attention launch alone (tile kernel + attention kernel), 12 of them per depth map
        N = gh * gw + 1
        qkv = torch.randn(n * N, 2304, device=dev)
        out = torch.empty(n * N, 768, device=dev)
        ws = torch.empty(n * 12 * ((N + 127) // 128) * 100352 // 4 + 64, device=dev)
        att_ms = timed(lambda: _lib.call("mvsf_vit_attention_forward", qkv, 2304, out, 768, ws, ws.numel() * 4, n, N),
                       a.warmup, a.reps)
        del qkv, out, ws
        res["workloads"][wl] = {
            "images": n, "patches": [gh, gw], "gflop_per_depth_map": {"linears": round(lin, 1), "attention": round(att, 1)},
            "arms": arms, "attention_one_block": {"ms": round(att_ms, 3), "tflops": round(att / 12 / att_ms, 2)},
            "max_abs_cuda_vs_torch_fp32": diff, "max_abs_bf16_vs_torch_fp32": diff_bf16, "max_abs_output": scale}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
