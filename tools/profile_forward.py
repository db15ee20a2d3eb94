"""Runs a few hot-path forwards at a named workload for timing breakdowns.
  python tools/profile_forward.py [--workload dtu] [--iters 2] [--breakdown]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from mvsformerplusplus_b200 import _lib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="dtu")
ap.add_argument("--iters", type=int, default=2)
ap.add_argument("--breakdown", action="store_true")
a = ap.parse_args()
wl = bench.WORKLOADS[a.workload]
dev = torch.device("cuda:0")
net, _ = bench.make_net()
net = net.to(dev)
feats, proj, dv = bench.make_inputs(wl, 1234)
f = {k: v.to(dev) for k, v in feats.items()}
p = {k: v.to(dev) for k, v in proj.items()}
d = dv.to(dev)
for _ in range(a.iters):
    net.forward_features(f, p, d, bench.TMP)
torch.cuda.synchronize()
import ctypes  # noqa: E402
used, miss = ctypes.c_int(-1), ctypes.c_int(-1)
if _lib.lib().mvsf_warp_corr_last_selection(ctypes.byref(used), ctypes.byref(miss)) == 0:
    print(f"finest stage, pass A: pipeline kernel chosen = {used.value}, sampled window misses = {miss.value} per mille")
if a.breakdown:
    with _lib.profile_calls() as prof:
        for _ in range(3):
            net.forward_features(f, p, d, bench.TMP)
    summ = prof.summary()
    tot = sum(v["ms"] for v in summ.values()) / 3
    print(json.dumps({k: {"ms_per_map": round(v["ms"] / 3, 4), "calls_per_map": v["calls"] // 3} for k, v in sorted(summ.items())}, indent=1))
    print("total ms per depth map (sum of bracketed calls):", round(tot, 3))
    torch.cuda.synchronize()
    per_call = [(n, round(s.elapsed_time(e), 4)) for n, s, e in prof.records[-len(prof.records) // 3:]]
    print("per call, last forward:", json.dumps([c for c in per_call if "warp_corr" in c[0] or "corr_aggregate" in c[0] or "vis_cnn" in c[0]]))
