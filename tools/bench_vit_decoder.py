"""ViT feature decoder (CrossVITDecoder, models/module.py:273-364) per depth map on cuda:0: the CUDA path
(hotpath.CrossVITDecoder) against the same layers in torch on the GPU (oracle/vit_decoder.py), in fp32 (TF32 off) and
under bf16 autocast as the reference's test.py:250 runs them.  Device events, warm-up, >= 20 timed repetitions (median
reported).  Prints one JSON line.

  python tools/bench_vit_decoder.py [--reps 20] [--warmup 3] [--workloads dtu,tt]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import vit_decoder as OV  # noqa: E402
from tools.bench_fpn import card, timed  # noqa: E402

# token grids of the ViT at the shipped rescale 0.4375 and patch 14: DTU 1152x1536 -> 504x672 -> 36x48,
# T&T 1088x1920 -> 476x840 -> 34x60
WORKLOADS = {"dtu": (5, 36, 48), "tt": (10, 34, 60)}
SHIPPED = dict(vit_ch=768, out_ch=64, dino_cfg=dict(cross_interval_layers=3, decoder_cfg=dict(
    init_values=1.0, prev_values=0.5, d_model=768, nhead=12, attention_type="Linear", ffn_type="ffn",
    self_cross_types=None, post_norm=False, pre_norm_query=True, no_combine_norm=False)))


def vit_decoder_gflop(V, h, w):
    """Algorithmic GFLOP of one depth map (2 x multiply-adds from the layer shapes; attention summaries included)."""
    d, hid, L = 768, 3072, h * w
    block = lambda M, qkv_rows: 2 * M * d * (qkv_rows + d + 2 * hid) + 2 * 2 * M * d * 64   # linears + KV / apply
    f = 2 * block(L, 3 * d)                                   # two self blocks on the reference view
    f += 3 * (2 * L * d * 2 * d + 2 * L * d * 64)             # K / V summaries of the three cross layers
    f += 3 * block((V - 1) * L, d)                            # three cross blocks on the source views
    f += V * (2 * L * 9 * d * 256 + 2 * 4 * L * 4 * 256 * 128 + 2 * 16 * L * 4 * 128 * 64)   # conv head
    return f / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="dtu,tt")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit_decoder: no CUDA device (timings are only taken on the GPU)")
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = torch.nn.Module()
    m.decoder_vit = CrossVITDecoder(SHIPPED)
    sd = synth.randomize_state_dict(m, seed=52)
    dec = m.decoder_vit.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    name, power = card()
    res = {"bench": "vit_decoder", "device": name, "power_limit": power, "reps": a.reps, "warmup": a.warmup,
           "workloads": {}}
    for wl in a.workloads.split(","):
        V, h, w = WORKLOADS[wl]
        g = torch.Generator(device=dev).manual_seed(1)
        x = [torch.randn(1, V, h * w, 768, device=dev, generator=g) for _ in range(3)]
        shape = (1, V, h, w, 768)

        def run_cuda():
            return dec(x, vit_shape=shape)

        def run_torch():
            with torch.no_grad():
                return OV.vit_decoder(x, sd_dev, shape)

        def run_bf16():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return OV.vit_decoder(x, sd_dev, shape)

        got, want, lo = run_cuda(), run_torch(), run_bf16()
        diff = float((got - want).abs().max())
        diff_bf16 = float((lo.float() - want).abs().max())
        scale = float(want.abs().max())
        del got, want, lo
        gflop = vit_decoder_gflop(V, h, w)
        arms = {}
        for arm, fn in (("cuda", run_cuda), ("torch_fp32", run_torch), ("torch_bf16_autocast", run_bf16)):
            ms = timed(fn, a.warmup, a.reps)
            torch.cuda.empty_cache()
            arms[arm] = {"ms_per_depth_map": round(ms, 3), "tflops": round(gflop / ms, 2)}
        res["workloads"][wl] = {"views": V, "tokens": [h, w], "gflop_per_depth_map": round(gflop, 1), "arms": arms,
                                "max_abs_cuda_vs_torch_fp32": diff, "max_abs_bf16_vs_torch_fp32": diff_bf16,
                                "max_abs_output": scale}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
