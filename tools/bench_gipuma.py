"""Gipuma fusion (fusion.fuse_scene_gipuma: probability filter, then fusibile's cross-view voting and point averaging, every
view a reference view and every other view its source) per scene on cuda:0.

Workloads (N distinct synthetic views each):
  dtu   49 views, 1152x1536, disp_threshold 0.1, num_consistent 2    (scripts/test.sh of the reference)
  tt   150 views, 1088x1920, disp_threshold 0.4, num_consistent 5    (Family in scripts/test_tt_inter.sh, T&T-like size)

The views are made on the device: the look-at ring cameras of synth.make_fusion_scene (synth.lookat_camera, the same view
order and 1.6x focal length for the last view) ray-cast against its analytic surface (a tilted plane with a sphere in front),
then seeded smooth relative depth noise, gross-outlier blobs, low-confidence regions and holes from bicubically upsampled
low-resolution noise.  Building 150 T&T-size views with the host generator would take minutes.

Timing: CUDA events around whole fuse_scene_gipuma calls (prepare, N vote / count read / emit steps, the concatenation),
--warmup calls first, median of --reps.  Reported per workload: ms per scene and per reference view, source probes per
second (N (N-1) H W probes per scene over the scene time), point count and peak device memory, with the card name and power
limit read in the same run.  There is no baseline arm: fusibile, the external program the reference runs, is not part of
this project, so any comparison with it is not measured.  Fails without a GPU.  Prints one JSON line.

  python tools/bench_gipuma.py [--reps 3] [--warmup 1] [--workloads dtu,tt]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import fusion as FU, synth  # noqa: E402

WORKLOADS = {"dtu": dict(N=49, H=1152, W=1536, disp=0.1, nc=2), "tt": dict(N=150, H=1088, W=1920, disp=0.4, nc=5)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def _field(g, H, W, cells, dev):
    """seeded smooth [H,W] field of zero mean and unit variance: cells x cells-ish noise upsampled bicubically"""
    h, w = max(2, H // cells), max(2, W // cells)
    x = torch.randn(1, 1, h, w, generator=g, device=dev)
    x = F.interpolate(x, size=(H, W), mode="bicubic", align_corners=False)[0, 0]
    x = x - x.mean()
    return x / x.std().clamp_min(1e-12)


def device_scene(N, H, W, seed, dev, theta_step=0.12, radius=650.0):
    """-> depths, confs, cams, images on dev (float32), N distinct views of synth.make_fusion_scene's surface"""
    g = torch.Generator(device=dev).manual_seed(seed)
    order = [synth.VIEW_ORDER[i % len(synth.VIEW_ORDER)] + (i // len(synth.VIEW_ORDER)) * 0.37 for i in range(N)]
    cams = torch.zeros(N, 2, 4, 4, dtype=torch.float64)
    normal = torch.tensor([0.25, 0.12, -1.0], dtype=torch.float64, device=dev)
    normal = normal / normal.norm()
    on_plane = torch.tensor([0.0, 0.0, radius + 30.0], dtype=torch.float64, device=dev)
    centre = torch.tensor([25.0, -15.0, radius], dtype=torch.float64, device=dev)
    rad = 0.18 * radius * W / 1536.0 * 1536.0 / 2776.6
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev) + 0.5,
                            torch.arange(W, dtype=torch.float64, device=dev) + 0.5, indexing="ij")
    pix = torch.stack([xs, ys, torch.ones_like(xs)], -1)
    depths = torch.empty(N, H, W, device=dev)
    confs = torch.empty(N, H, W, device=dev)
    images = torch.empty(N, 3, H, W, device=dev)
    for i in range(N):
        E, K = synth.lookat_camera(order[i], H, W, radius=radius, theta_step=theta_step,
                                   focal_full=2776.6 * (1.6 if i == N - 1 and N > 2 else 1.0))
        cams[i, 0], cams[i, 1, :3, :3], cams[i, 1, 3, 3] = E, K, 1.0
        R, t = E[:3, :3].to(dev), E[:3, 3].to(dev)
        C = -R.T @ t
        d = (pix @ torch.linalg.inv(K.to(dev)).T) @ R
        plane = ((on_plane - C) @ normal) / (d @ normal)
        oc = C - centre
        a, b, c = (d * d).sum(-1), 2.0 * (d @ oc), oc @ oc - rad * rad
        disc = b * b - 4.0 * a * c
        sphere = torch.where(disc > 0, (-b - disc.clamp_min(0).sqrt()) / (2.0 * a), torch.full_like(a, float("inf")))
        sphere = torch.where(sphere > 0, sphere, torch.full_like(a, float("inf")))
        z = torch.minimum(plane, sphere).float()
        amp = (0.006 * (_field(g, H, W, 96, dev) + 0.6)).clamp_min(0.0)
        z = z * (1.0 + amp * _field(g, H, W, 24, dev))
        z = torch.where(_field(g, H, W, 64, dev) > 1.5, z * (1.0 + 0.08 * _field(g, H, W, 32, dev)), z)
        depths[i] = torch.where(_field(g, H, W, 48, dev) > 1.9, torch.zeros_like(z), z)
        confs[i] = (0.72 + 0.3 * _field(g, H, W, 48, dev)).clamp(0.0, 1.0)
        images[i] = torch.round((0.5 + 0.25 * _field(g, H, W, 32, dev)).clamp(0.0, 1.0) * 255.0) / 255.0
    return depths, confs, cams.float().to(dev), images


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="dtu,tt")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gipuma: no CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    res = {"bench": "gipuma", "device": name, "power_limit": power, "reps": a.reps, "warmup": a.warmup,
           "baseline": "none: fusibile is not measured", "workloads": {}}
    for wl in a.workloads.split(","):
        w = WORKLOADS[wl]
        N, H, W = w["N"], w["H"], w["W"]
        scene = device_scene(N, H, W, seed=7, dev=dev)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()

        def run():
            return FU.fuse_scene_gipuma(*scene, disp_threshold=w["disp"], num_consistent=w["nc"])

        for _ in range(a.warmup):
            run()
        times, points = [], None
        for _ in range(a.reps):
            ms, (xyz, _) = event_ms(run)
            times.append(ms)
            points = int(xyz.shape[0])
            del xyz
        ms = statistics.median(times)
        probes = N * (N - 1) * H * W
        res["workloads"][wl] = {"views": N, "H": H, "W": W, "disp_threshold": w["disp"], "num_consistent": w["nc"],
                                "ms_per_scene": round(ms, 3), "ms_per_ref_view": round(ms / N, 4),
                                "ms_all": [round(t, 3) for t in times], "probes": probes,
                                "probes_per_s": float(f"{probes / (ms * 1e-3):.4g}"), "points": points,
                                "valid_pixels": int((scene[0] > 0).sum()),
                                "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2)}
        del scene
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
