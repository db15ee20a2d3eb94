"""A whole scene, image folder to point cloud, on cuda:0.  Two arms, alternated, each run `--repeats` times after one
untimed run (median reported):
  (a) load_scene + reconstruct_scene (pcd fusion): each image decoded once, uploaded once as uint8, resized once on the
      device; each view set normalised on the device; depth maps and confidences stay on the device until fusion;
  (b) the reference flow: oracle/_ref's general_eval.MVSDataset in a DataLoader with 4 workers (test.py:202), the same
      DINOv2MVSNet, test.py's per-view file writes (save_pfm, the uint8 confidence .npy, write_cam, the colour JPEG), the
      read-back as test.py's filter_depth reads (read_pfm, np.load / 255, the cam text, read_img), then fuse_scene.
      Each view's files are read back once (test.py reads a source view's files again for every reference view naming
      it), so this arm's read-back is a lower bound.
Workloads, written from seeds to a temporary directory: DTU-like (49 views of 1600x1200 JPEGs, 10 sources per view,
nviews 5, 1152x1536, 192 depths) and T&T-like (`--tt-views` views of 1920x1080, nviews 20 as scripts/test_tt_inter.sh,
1088x1920 after the 4-row pad, 192 depths).  The weights are seeded and random, so depth maps are random and fusion point
counts are not those of a real scene.
Also: the load-and-prepare time alone (load_scene + every item's normalize) against the loader alone (every sample
collated and moved to the device); the resize and normalize kernels' CUDA-event time and their GB/s from the bytes the
shapes imply, against 3.35 TB/s; bytes uploaded per scene from shapes; peak allocated memory; card and power limit read in
the same call.  Prints one JSON line.

  python tools/bench_scene.py [--workloads dtu,tt] [--repeats 2] [--tt-views 30]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mvsformerplusplus_b200 import scene as S  # noqa: E402
from mvsformerplusplus_b200 import synth  # noqa: E402
from mvsformerplusplus_b200.fusion import fuse_scene, read_pair_file  # noqa: E402

TMP = [5.0, 5.0, 5.0, 1.0]
HBM = 3.35e12
PCD = dict(conf=0.5, thres_view=2, thres_disp=1.0)


def workloads(tt_views):
    return {"dtu": dict(dataset="dtu", scan="scan1", views=49, src=(1200, 1600), nviews=5, max_h=1152, max_w=1536,
                        ndepths=192, interval_scale=1.06, n_pair=10, line11="425.0 2.65", seed=601),
            "tt": dict(dataset="tt", scan="Family", views=tt_views, src=(1080, 1920), nviews=20, max_h=1088, max_w=1920,
                       ndepths=192, interval_scale=1.06, n_pair=20, line11="480.5 1.7 256 915.7", seed=602)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in q.split(",")]
    return dict(card=name, power_limit=power)


def write_scene(w, root):
    """JPEGs of a smooth seeded field plus texture, look-at cameras, pair.txt with the n_pair nearest views"""
    from PIL import Image
    h, wd = w["src"]
    g = np.random.default_rng(w["seed"])
    base = os.path.join(root, w["scan"])
    for sub in ("images", "cams"):
        os.makedirs(os.path.join(base, sub))
    N = w["views"]
    for v in range(N):
        low = Image.fromarray(g.integers(0, 256, (h // 24, wd // 24, 3), dtype=np.uint8)).resize((wd, h), Image.BILINEAR)
        img = np.clip(np.asarray(low, np.int16) + g.integers(-12, 13, (h, wd, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(base, "images", f"{v:08d}.jpg"), "JPEG", quality=90)
        E, K = synth.lookat_camera(v - N // 2, h, wd, theta_step=0.02)
        rows = ["extrinsic"] + [" ".join(f"{x:.6f}" for x in E[i].tolist()) for i in range(4)] + ["", "intrinsic"]
        rows += [" ".join(f"{x:.6f}" for x in K[i].tolist()) for i in range(3)] + ["", w["line11"]]
        with open(os.path.join(base, "cams", f"{v:08d}_cam.txt"), "w") as f:
            f.write("\n".join(rows) + "\n")
        if w["dataset"] == "dtu":   # the loader opens the reference view's ground truth; 8x8 placeholders keep that cheap
            gt = os.path.join(os.path.dirname(root), "mvs_training", "Depths_raw", w["scan"])
            os.makedirs(gt, exist_ok=True)
            Image.fromarray(np.full((8, 8), 200, np.uint8)).save(os.path.join(gt, f"depth_visual_{v:04d}.png"))
            with open(os.path.join(gt, f"depth_map_{v:04d}.pfm"), "wb") as f:
                f.write(b"Pf\n8 8\n-1.000000\n" + np.ones(64, "<f4").tobytes())
    lines = [str(N)]
    for v in range(N):
        srcs = sorted((s for s in range(N) if s != v), key=lambda s: abs(s - v))[:w["n_pair"]]
        lines += [str(v), " ".join([str(len(srcs))] + [f"{s} {100.0 - k:.1f}" for k, s in enumerate(srcs)])]
    with open(os.path.join(base, "pair.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return root


def load_args(w):
    return dict(scan=w["scan"], dataset=w["dataset"], nviews=w["nviews"], ndepths=w["ndepths"],
                interval_scale=w["interval_scale"], max_h=w["max_h"], max_w=w["max_w"])


def arm_ours(model, datapath, w):
    sc = S.load_scene(datapath, **load_args(w))
    xyz, _ = S.reconstruct_scene(model, sc, "pcd", tmp=TMP, **PCD)
    torch.cuda.synchronize()
    return xyz.shape[0]


def _loader(ge, datapath, w):
    import contextlib
    from torch.utils.data import DataLoader
    with contextlib.redirect_stdout(sys.stderr):   # the loader prints its view sets
        ds = ge.MVSDataset(datapath, [w["scan"]], "test", w["nviews"], ndepths=w["ndepths"], interval_scale=w["interval_scale"],
                           max_h=w["max_h"], max_w=w["max_w"], dataset=w["dataset"], use_short_range=False)
    return DataLoader(ds, batch_size=1, shuffle=False, num_workers=4)


def _read_cam(path):
    with open(path) as f:
        lines = [line.rstrip() for line in f.readlines()]
    cam = np.zeros((2, 4, 4), dtype=np.float32)
    cam[0] = np.fromstring(" ".join(lines[1:5]), dtype=np.float32, sep=" ").reshape((4, 4))
    cam[1, :3, :3] = np.fromstring(" ".join(lines[7:10]), dtype=np.float32, sep=" ").reshape((3, 3))
    cam[1, 3, 3] = 1.0
    return cam


def arm_reference(model, ge, data_io, datapath, w, out):
    import cv2
    from PIL import Image
    dev = torch.device("cuda:0")
    std = torch.tensor([0.229, 0.224, 0.225], device=dev).reshape((3, 1, 1))
    mean = torch.tensor([0.485, 0.456, 0.406], device=dev).reshape((3, 1, 1))
    for sub in ("depth_est", "confidence", "cams", "images"):
        os.makedirs(os.path.join(out, sub), exist_ok=True)
    refs = []
    with torch.no_grad():
        for sample in _loader(ge, datapath, w):
            imgs = sample["imgs"].to(dev)
            proj = {k: v.to(dev) for k, v in sample["proj_matrices"].items()}
            o = model(imgs, proj, sample["depth_values"].to(dev), TMP)
            ref = int(sample["filename"][0].split("/")[-1][:8])
            refs.append(ref)
            name = f"{ref:08d}"
            data_io.save_pfm(os.path.join(out, "depth_est", name + ".pfm"), o["refined_depth"][0].cpu().numpy())
            np.save(os.path.join(out, "confidence", name + ".npy"),
                    (o["photometric_confidence"][0].cpu().numpy() * 255).astype(np.uint8))
            S.write_cam(os.path.join(out, "cams", name + "_cam.txt"), sample["proj_matrices"]["stage4"][0, 0].numpy())
            img = (imgs[0, 0] * std + mean).permute(1, 2, 0).cpu().numpy()
            cv2.imwrite(os.path.join(out, "images", name + ".jpg"),
                        cv2.cvtColor(np.clip(img * 255, 0, 255).astype(np.uint8), cv2.COLOR_RGB2BGR))
    depths, confs, cams, images = [], [], [], []
    for ref in refs:
        name = f"{ref:08d}"
        depths.append(np.array(data_io.read_pfm(os.path.join(out, "depth_est", name + ".pfm"))[0], dtype=np.float32))
        confs.append((np.load(os.path.join(out, "confidence", name + ".npy")) / 255).astype(np.float32))
        cams.append(_read_cam(os.path.join(out, "cams", name + "_cam.txt")))
        images.append((np.array(Image.open(os.path.join(out, "images", name + ".jpg")), dtype=np.float32) / 255.).transpose(2, 0, 1))
    t = lambda x: torch.from_numpy(np.ascontiguousarray(np.stack(x))).to(dev)  # noqa: E731
    item = {r: k for k, r in enumerate(refs)}
    pairs = [(item[r], [item[s] for s in srcs if s in item]) for r, srcs in read_pair_file(os.path.join(datapath, w["scan"], "pair.txt"))
             if r in item]
    xyz, _ = fuse_scene(t(depths), t(confs), t(cams), t(images), pairs, "pcd", **PCD)
    torch.cuda.synchronize()
    return xyz.shape[0]


def prep_ours(datapath, w):
    sc = S.load_scene(datapath, **load_args(w))
    for k in range(len(sc)):
        sc.item(k)
    torch.cuda.synchronize()


def prep_reference(ge, datapath, w):
    dev = torch.device("cuda:0")
    for sample in _loader(ge, datapath, w):
        sample["imgs"].to(dev)
        {k: v.to(dev) for k, v in sample["proj_matrices"].items()}
        sample["depth_values"].to(dev)
    torch.cuda.synchronize()


def kernel_rates(datapath, w, reps=5):
    """CUDA-event ms and GB/s of the resize over the scene's images and of normalize over every item"""
    plan = S.ScenePlan(datapath, w["scan"], w["dataset"], w["nviews"])
    srcs = [torch.from_numpy(S._decode(p)).cuda() for p in plan.img_paths]
    H, W = w["max_h"], w["max_w"]
    images = torch.empty(len(srcs), H, W, 3, dtype=torch.uint8, device="cuda")
    slot = {v: k for k, v in enumerate(plan.view_ids)}
    sets = [[slot[v] for v in [r] + s] for r, s in plan.view_sets]

    def resize():
        for k, s in enumerate(srcs):
            S.resize_u8(s[None], H, W, plan.pad, out=images[k:k + 1])

    def normalize():
        for views in sets:
            S.normalize(images, views)
    out = {}
    for name, fn, nbytes in (("resize", resize, sum(s.numel() for s in srcs) + images.numel()),
                             ("normalize", normalize, sum(len(v) * H * W * 3 * (1 + 4) for v in sets))):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / reps
        out[name] = dict(ms=round(ms, 3), bytes=int(nbytes), gb_per_s=round(nbytes / ms / 1e6, 1),
                         share_of_hbm=round(nbytes / ms * 1e3 / HBM, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="dtu,tt")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--tt-views", type=int, default=30)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_scene needs a CUDA device"
    from oracle.gen_golden_scene import reference_datasets
    from tests.model_common import cuda_model, model_state_dict
    mods = reference_datasets()
    if mods is None:
        raise SystemExit("oracle/_ref/datasets is missing: run __graft_entry__.build() where the reference sources are")
    ge, data_io = mods
    model = cuda_model(model_state_dict(402), torch.device("cuda:0"))
    res = dict(bench="scene", **card(), repeats=args.repeats, fusion="pcd " + json.dumps(PCD),
               note="random weights: depth maps and point counts are not those of a real scene", workloads={})
    for name in args.workloads.split(","):
        w = workloads(args.tt_views)[name]
        with tempfile.TemporaryDirectory() as d:
            datapath = write_scene(w, os.path.join(d, "in"))
            times = {"ours": [], "reference": [], "prep_ours": [], "prep_reference": []}
            points = {}
            for r in range(args.repeats + 1):
                for arm in ("ours", "reference"):
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    if arm == "ours":
                        points[arm] = arm_ours(model, datapath, w)
                    else:
                        points[arm] = arm_reference(model, ge, data_io, datapath, w, os.path.join(d, f"out{r}"))
                    dt = time.perf_counter() - t0
                    if r:
                        times[arm].append(dt)
                        res.setdefault("peak_mem_gb", {}).setdefault(name, {})[arm] = round(
                            torch.cuda.max_memory_allocated() / 1e9, 2)
                for arm, fn in (("prep_ours", lambda: prep_ours(datapath, w)), ("prep_reference", lambda: prep_reference(ge, datapath, w))):
                    t0 = time.perf_counter()
                    fn()
                    if r:
                        times[arm].append(time.perf_counter() - t0)
            plan = S.ScenePlan(datapath, w["scan"], w["dataset"], w["nviews"])
            items, uniq = len(plan.view_sets), len(plan.view_ids)
            med = {k: float(np.median(v)) for k, v in times.items()}
            res["workloads"][name] = dict(
                views=uniq, items=items, nviews=w["nviews"], src=w["src"], size=[w["max_h"], w["max_w"]],
                scene_s={k: round(med[k], 3) for k in ("ours", "reference")},
                ms_per_view={k: round(1e3 * med[k] / items, 2) for k in ("ours", "reference")},
                load_prep_s={"ours": round(med["prep_ours"], 3), "reference_loader": round(med["prep_reference"], 3)},
                points=points,
                bytes_uploaded={"ours_u8_once": uniq * w["src"][0] * w["src"][1] * 3,
                                "reference_fp32_per_item": items * w["nviews"] * w["max_h"] * w["max_w"] * 3 * 4},
                kernels=kernel_rates(datapath, w))
            print(name, json.dumps(res["workloads"][name]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
