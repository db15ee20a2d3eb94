"""Depth-map fusion (test.py:387-517 over misc/fusion.py:79-165) per reference view on cuda:0: this package's kernels
(fusion.fuse_scene) against the reference's own misc/fusion.py on the GPU (`kind: "reference"`, from oracle/_ref where
build() copied it; its glue is oracle/gen_golden_fusion.reference_filter plus the boolean-mask extraction of test.py:419-424
done on the device), or against oracle/fusion.py on the device (`kind: "port"`) where oracle/_ref is absent.

Workloads: DTU (49 views, 4 sources, 1152x1536) and T&T (50 views, 10 sources, 1088x1920), methods pcd and dpcd.  A scene
has n_src + 1 distinct synthetic views (synth.make_fusion_scene), repeated cyclically to the workload's view count on the
device, so every reference view reads n_src maps of other cameras.  Per reference view: the two arms alternate, warm-up,
median of --reps CUDA-event timings of one reference view each (for the kernel arm that is a fuse_scene call on a
one-view pair list: camera inverses, filter, the count read-back, extraction); `scene_ms_per_view` is a whole-scene
fuse_scene call over all views divided by the view count.  Algorithmic bytes: every map the method needs read once, the
image, and the points written.  Fails without a GPU.  Prints one JSON line.

  python tools/bench_fusion.py [--reps 20] [--warmup 3] [--workloads dtu,tt] [--methods pcd,dpcd]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fusion as OF  # noqa: E402
from oracle import gen_golden_fusion as GG  # noqa: E402

WORKLOADS = {"dtu": (49, 4, 1152, 1536), "tt": (50, 10, 1088, 1920)}
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def view_bytes(method, V, H, W, points):
    maps = (2 * (1 + V)) if method == "pcd" else (1 + V) + 1   # dpcd reads no source confidence
    return 4 * H * W * (maps + 3) + 15 * points


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="dtu,tt")
    ap.add_argument("--methods", default="pcd,dpcd")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fusion: no CUDA device (timings are only taken on the GPU)")
    from mvsformerplusplus_b200 import fusion as FU
    dev = torch.device("cuda:0")
    ref_mod = GG.reference_fusion_module()
    kind = "reference" if ref_mod is not None else "port"
    name, power = card()
    res = {"bench": "fusion", "device": name, "power_limit": power, "reps": a.reps, "warmup": a.warmup, "baseline_kind": kind,
           "workloads": {}}
    for wl in a.workloads.split(","):
        views, V, H, W = WORKLOADS[wl]
        sc = synth.make_fusion_scene(V + 1, H, W, seed=7, n_src=V)
        rep = [i % (V + 1) for i in range(views)]
        depths, confs, cams, images = (sc[k][rep].contiguous().to(dev) for k in ("depths", "confs", "cams", "images"))
        K = V + 1   # view i shows camera i % K: its sources are the other cameras of its block of K views
        pairs = [(i, [s if s < views else s - K for s in (i - i % K + (i % K + j) % K for j in range(1, K))]) for i in range(views)]
        for method in a.methods.split(","):

            def ours(i):
                return FU.fuse_scene(depths, confs, cams, images, [pairs[i]], method)

            def baseline(i):
                r, srcs = pairs[i]
                with torch.no_grad():
                    if ref_mod is not None:
                        mask, _, pts = GG.reference_filter(ref_mod, method, r, srcs, depths, confs, cams)
                        pts = pts.permute(1, 2, 0)
                    else:
                        mask, avg, _ = OF.filter_view(r, srcs, depths, confs, cams, method)
                        pts = OF.view_points(r, avg, cams)
                    return pts[mask], (images[r] * 255).permute(1, 2, 0)[mask].to(torch.uint8)

            t_ours, t_base, n_ours, n_base = [], [], 0, 0
            for k in range(a.warmup + a.reps):
                i = k % views
                ms_o, (xyz, _) = event_ms(lambda: ours(i))
                ms_b, (pts, _) = event_ms(lambda: baseline(i))
                if k >= a.warmup:
                    t_ours.append(ms_o)
                    t_base.append(ms_b)
                    n_ours += xyz.shape[0]
                    n_base += pts.shape[0]
                del xyz, pts
            scene_ms, (xyz, _) = event_ms(lambda: FU.fuse_scene(depths, confs, cams, images, pairs, method))
            scene_ms, (xyz, _) = event_ms(lambda: FU.fuse_scene(depths, confs, cams, images, pairs, method))
            total = xyz.shape[0]
            del xyz
            mo, mb = median(t_ours), median(t_base)
            per_view_pts = n_ours / a.reps
            nbytes = view_bytes(method, V, H, W, per_view_pts)
            res["workloads"][f"{wl}_{method}"] = {
                "views": views, "n_src": V, "H": H, "W": W, "algorithmic_mb_per_view": round(nbytes / 1e6, 1),
                "cuda": {"ms_per_view": round(mo, 3), "scene_ms_per_view": round(scene_ms / views, 3),
                         "gb_per_s": round(nbytes / mo / 1e6, 1), "share_of_hbm_peak": round(nbytes / (mo * 1e-3) / HBM_BYTES_PER_S, 4),
                         "scene_share_of_hbm_peak": round(nbytes / (scene_ms / views * 1e-3) / HBM_BYTES_PER_S, 4),
                         "points_per_s": round(per_view_pts / (mo * 1e-3)), "peak_mb": round(peak_bytes(lambda: ours(0)) / 1e6, 1),
                         "scene_peak_mb": round(peak_bytes(lambda: FU.fuse_scene(depths, confs, cams, images, pairs, method)) / 1e6, 1)},
                kind: {"ms_per_view": round(mb, 3), "gb_per_s": round(nbytes / mb / 1e6, 1),
                       "points_per_s": round(n_base / a.reps / (mb * 1e-3)), "peak_mb": round(peak_bytes(lambda: baseline(0)) / 1e6, 1)},
                "points_cuda": n_ours, "points_baseline": n_base, "scene_points": total,
                "speedup_per_view": round(mb / mo, 1)}
            torch.cuda.empty_cache()
        del depths, confs, cams, images
    print(json.dumps(res))


if __name__ == "__main__":
    main()
