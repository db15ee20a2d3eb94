"""FPN feature pyramid (models/module.py:208-270, encoder -> conv31 + vit_feat -> decoder) per depth map on cuda:0:
the CUDA path (hotpath.FPNEncoder / FPNDecoder) against the same layers in torch on the GPU (oracle/fpn.py), in fp32
(TF32 off) and under bf16 autocast as the reference's test.py:250 runs them.  Device events, warm-up, >= 20 timed
repetitions (median reported).  Prints one JSON line.

  python tools/bench_fpn.py [--reps 20] [--warmup 3] [--workloads dtu,tt]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import synth  # noqa: E402
from mvsformerplusplus_b200.params import FPN_ENCODER_LAYERS  # noqa: E402
from oracle import fpn as OF  # noqa: E402

WORKLOADS = {"dtu": (5, 1152, 1536), "tt": (10, 1088, 1920)}


def fpn_gflop(H, W):
    """Algorithmic GFLOP of one image (2 x multiply-adds from the layer shapes)."""
    f, h, w = 0, H, W
    for _, ci, co, k, s in FPN_ENCODER_LAYERS:
        h, w = h // s, w // s
        f += 2 * k * k * ci * co * h * w
    h8, w8 = H // 8, W // 8
    f += 2 * 64 * 64 * h8 * w8
    for k, (cl, co) in enumerate(((32, 32), (16, 16), (8, 8)), start=1):
        hk, wk = h8 << k, w8 << k
        f += 2 * cl * 64 * hk * wk + 2 * 9 * 64 * co * hk * wk
    return f / 1e9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="dtu,tt")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fpn: no CUDA device (timings are only taken on the GPU)")
    from mvsformerplusplus_b200.hotpath import FPNDecoder, FPNEncoder
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    m = torch.nn.Module()
    m.encoder, m.decoder = FPNEncoder([8, 16, 32, 64]), FPNDecoder([8, 16, 32, 64])
    sd = synth.randomize_state_dict(m, seed=33)
    m = m.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    name, power = card()
    res = {"bench": "fpn", "device": name, "power_limit": power, "reps": a.reps, "warmup": a.warmup, "workloads": {}}
    for wl in a.workloads.split(","):
        V, H, W = WORKLOADS[wl]
        x = synth.make_images(V, H, W, seed=1).to(dev)
        vit = torch.randn(V, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(2)).to(dev)

        def run_cuda():
            c = m.encoder(x)
            return list(c) + m.decoder(c[0], c[1], c[2], c[3] + vit)

        def run_torch():
            with torch.no_grad():
                c = OF.fpn_encoder(x, sd_dev)
                return c + OF.fpn_decoder(c[0], c[1], c[2], c[3] + vit, sd_dev)

        def run_bf16():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                c = OF.fpn_encoder(x, sd_dev)
                return c + OF.fpn_decoder(c[0], c[1], c[2], c[3] + vit, sd_dev)

        got, want, lo = run_cuda(), run_torch(), run_bf16()
        diff = max(float((g - w).abs().max()) for g, w in zip(got, want))
        scale = max(float(w.abs().max()) for w in want)
        diff_bf16 = max(float((g.float() - w).abs().max()) for g, w in zip(lo, want))
        del got, want, lo
        gflop = fpn_gflop(H, W) * V
        arms = {}
        for arm, fn in (("cuda", run_cuda), ("torch_fp32", run_torch), ("torch_bf16_autocast", run_bf16)):
            ms = timed(fn, a.warmup, a.reps)
            torch.cuda.empty_cache()
            arms[arm] = {"ms_per_depth_map": round(ms, 3), "tflops": round(gflop / ms, 2)}
        res["workloads"][wl] = {"views": V, "H": H, "W": W, "gflop_per_depth_map": round(gflop, 1), "arms": arms,
                                "max_abs_cuda_vs_torch_fp32": diff, "max_abs_bf16_vs_torch_fp32": diff_bf16,
                                "max_abs_output": scale}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
