"""Times forward + backward of the four cost volumes of one MVSFormer++ training step (models/cost_volume.py:64-101 under
autograd) and reports the peak memory above the inputs, for two arms on the same GPU:

  cuda       mvsformerplusplus_b200.training.cost_volume (the CUDA forward and mvsf_warp_corr_aggregate_backward)
  reference  the reference's arithmetic in torch: oracle/train.py with oracle.hotpath.USE_ATEN_KERNELS (F.grid_sample)

Both use the same train-mode visibility CNN (the reference's layers and parameter names).  Workloads: the DTU training
scales of config/mvsformer++.json, 512 x 640 with batch 4 and 1024 x 1280 with batch 2, V = 5, stages 1-4 (C 64/32/16/8,
ndepths 32/16/8/4 at 1/8 .. 1/1 resolution).  Arms alternate after warm-up; times are CUDA events over the whole step.
Prints one JSON line with the card name and power limit read in the same run.

  python tools/bench_train_cost_volume.py [--reps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import synth  # noqa: E402
from mvsformerplusplus_b200.training import cost_volume  # noqa: E402
from oracle import hotpath as O  # noqa: E402
from oracle import train as OT  # noqa: E402
from tests.train_common import make_vis  # noqa: E402

STAGES = ((64, 32, 8), (32, 16, 4), (16, 8, 2), (8, 4, 1))   # C, ndepth, downscale
WORKLOADS = {"dtu_512x640_b4": (4, 512, 640), "dtu_1024x1280_b2": (2, 1024, 1280)}
V = 5


def power_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:   # the number is still reported, without its power limit
        return torch.cuda.get_device_name(0), f"unavailable ({type(e).__name__})"


def make_inputs(B, H, W, dev):
    """per stage: features [B,V,C,h,w] (leaf, requires grad), proj [B,V,2,4,4], hypotheses [B,D,h,w], upstream gradient"""
    g = torch.Generator().manual_seed(1)
    pm = synth.make_proj_matrices(V, H, W, batch=B, theta_step=0.12)
    dv = synth.make_depth_values(192, batch=B)
    out = []
    for s, (C, D, sc) in enumerate(STAGES):
        h, w = H // sc, W // sc
        f = torch.randn(B, V, C, h, w, generator=g).to(dev).requires_grad_(True)
        hyp = O.init_inverse_range(dv, D, h, w).to(dev)
        out.append((f, pm[f"stage{s + 1}"].to(dev), hyp, torch.randn(B, 8, D, h, w, generator=g).to(dev)))
    return out


def step(arm, inputs, vis):
    for f, pm, hyp, grad in inputs:
        if arm == "cuda":
            vol = cost_volume(f, pm, hyp, vis[0])
        else:
            with torch.device(f.device):
                vol = OT.cost_volume(f, pm, hyp, vis[1], G=8)
        vol.backward(grad)
        del vol


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_cost_volume: needs a CUDA device")
    dev = torch.device("cuda:0")
    O.USE_ATEN_KERNELS = True
    torch.backends.cudnn.benchmark = True
    name, limit = power_info()
    torch.manual_seed(0)
    vis_c = make_vis().to(dev).train()
    vis_r = make_vis().to(dev).train()
    vis_r.load_state_dict(vis_c.state_dict())
    res = {}
    for wname, (B, H, W) in WORKLOADS.items():
        inputs = make_inputs(B, H, W, dev)
        arms = ("cuda", "reference")
        for _ in range(a.warmup):
            for arm in arms:
                step(arm, inputs, (vis_c, vis_r))
        times = {arm: [] for arm in arms}
        peak = {}
        for r in range(a.reps):
            for arm in arms if r % 2 == 0 else arms[::-1]:
                for f, *_ in inputs:
                    f.grad = None
                vis_c.zero_grad(set_to_none=True)
                vis_r.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                step(arm, inputs, (vis_c, vis_r))
                e.record()
                torch.cuda.synchronize()
                times[arm].append(s.elapsed_time(e))
                peak[arm] = max(peak.get(arm, 0), torch.cuda.max_memory_allocated() - base)
        res[wname] = {"B": B, "H": H, "W": W, "V": V}
        for arm in arms:
            t = sorted(times[arm])
            res[wname][arm] = {"ms_median": round(t[len(t) // 2], 3), "ms_min": round(t[0], 3), "ms_max": round(t[-1], 3),
                               "peak_gb_above_inputs": round(peak[arm] / 2**30, 3)}
        res[wname]["speedup"] = round(res[wname]["reference"]["ms_median"] / res[wname]["cuda"]["ms_median"], 2)
        del inputs
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "train_cost_volume", "device": name, "power_limit": limit, "reps": a.reps,
                      "warmup": a.warmup, "what": "forward + backward of the 4 stage cost volumes of one training step",
                      "workloads": res}))


if __name__ == "__main__":
    main()
