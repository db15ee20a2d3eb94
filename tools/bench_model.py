"""Whole model, images to depth maps (DINOv2MVSNet.forward as the reference's test.py runs it), on cuda:0.  Arms,
alternated in one process, `--repeats` times each (median reported):
  (a) hotpath.DINOv2MVSNet.forward on device-resident images;
  (b) the reference-shaped model with the reference's eval glue (bicubic resize, per-view FPN calls, conv31 + vit_feat,
      torch.stack) around install(model, feature_pyramid=True, vit_decoder=True, vit=True): the path before (a);
  (c) the reference's own DINOv2MVSNet from oracle/_ref in torch on the GPU under bf16 autocast, as test.py:250-251 runs
      it (skipped when oracle/_ref is absent);
  (d) arm (a) from pinned host images through streaming.PrefetchingRunner (upload of the next batch overlapped).
Workloads: DTU (V=5, 1152x1536, numdepth 192) and Tanks & Temples (V=10, 1088x1920, numdepth 256); seeded images,
synth's look-at cameras, the same seeded weights in every arm.  Device events around `--steps` forwards after `--warmup`.
Prints one JSON line: ms per depth map and depth maps/s per arm, bytes uploaded per step (d), peak allocated memory per
arm, max |refined_depth (a) - (b)| and (a) - (c), card, power limit and SM clock read in the same call.

  python tools/bench_model.py [--workloads dtu,tt] [--steps 3] [--warmup 1] [--repeats 3] [--arms abcd]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.model_common import cuda_model, installed_glue_model, make_inputs, model_state_dict  # noqa: E402

WORKLOADS = {"dtu": dict(B=1, V=5, H=1152, W=1536, numdepth=192, iseed=401, wseed=402),
             "tt": dict(B=1, V=10, H=1088, W=1920, numdepth=256, iseed=403, wseed=404)}
TMP = [5.0, 5.0, 5.0, 1.0]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


def reference_model(sd, dev):
    """the reference's own DINOv2MVSNet (oracle/_ref) with the weights sd, or None"""
    from oracle import reference
    from oracle.gen_golden_model import reference_model as ref_cls
    if reference.root("models", reference.CONFIG) is None:
        return None
    cls, cfg = ref_cls()
    m = cls(cfg)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def timed(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def bench(name, wl, a, dev):
    sd = model_state_dict(wl["wseed"])
    host = make_inputs(wl)
    imgs, proj, dv = host[0].to(dev), {k: v.to(dev) for k, v in host[1].items()}, host[2].to(dev)
    arms, outs = {}, {}
    if "a" in a.arms:
        net = cuda_model(sd, dev)
        arms["a"] = lambda: net(imgs, proj, dv, TMP)
    if "b" in a.arms:
        glue = installed_glue_model(sd, dev)
        arms["b"] = lambda: glue(imgs, proj, dv, TMP)
    if "c" in a.arms:
        ref = reference_model(sd, dev)
        if ref is not None:
            def run_c():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                    return ref.forward(imgs, proj, dv, tmp=TMP)
            arms["c"] = run_c
    if "d" in a.arms:
        from mvsformerplusplus_b200.streaming import PrefetchingRunner
        net_d = net if "a" in a.arms else cuda_model(sd, dev)
        runner = PrefetchingRunner(net_d, dev)
        pinned = [(x.pin_memory(), {k: v.pin_memory() for k, v in p.items()}, d.pin_memory())
                  for x, p, d in (host, make_inputs(dict(wl, iseed=wl["iseed"] + 1)))]
        step = [0]

        def run_d():
            i = step[0]
            step[0] += 1
            return runner.run(pinned[i % 2], next_batch=pinned[(i + 1) % 2], tmp=TMP)
        arms["d"] = run_d
    for k, fn in arms.items():   # outputs (and a warm-up) of every arm before the timed rounds
        outs[k] = fn()["refined_depth"].float().clone()
    ms = {k: [] for k in arms}
    mem = {k: 0 for k in arms}
    for _ in range(a.repeats):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            ms[k].append(timed(fn, a.warmup, a.steps) / wl["B"])
            mem[k] = max(mem[k], torch.cuda.max_memory_allocated(dev))
    res = {"workload": name, **{k: v for k, v in wl.items() if k in ("B", "V", "H", "W", "numdepth")}}
    for k in arms:
        med = sorted(ms[k])[len(ms[k]) // 2]
        res[f"arm_{k}"] = dict(ms_per_depth_map=round(med, 2), depth_maps_per_s=round(1000.0 / med, 2),
                               ms_all=[round(x, 2) for x in ms[k]], max_memory_allocated_gb=round(mem[k] / 2**30, 2))
    if "d" in arms:
        res["arm_d"]["bytes_uploaded_per_step"] = runner.bytes_per_batch(pinned[0])
    for k in ("b", "c", "d"):
        if "a" in outs and k in outs:
            res[f"max_abs_refined_depth_a_vs_{k}"] = float((outs["a"] - outs[k]).abs().max())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="dtu,tt")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--arms", default="abcd")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_model.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from mvsformerplusplus_b200.build import build
    build()
    results = [bench(w, WORKLOADS[w], a, dev) for w in a.workloads.split(",")]
    print(json.dumps(dict(**card(), results=results)))


if __name__ == "__main__":
    main()
