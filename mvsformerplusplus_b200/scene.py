"""A scene from its image folder to its point cloud on the GPU: the reference's eval loader (datasets/general_eval.py), the
model loop of test.py / test_tt.py and the fusion, without the per-item host work and the file round trip between them.

  load_scene(datapath, scan, dataset, nviews, ndepths, interval_scale, max_h, max_w, ...)  <- MVSDataset + DataLoader
  Scene.item(k)                         <- MVSDataset[k] after the default collate and tocuda (bit-identical)
  reconstruct_scene(model, scene, method, ...)   <- save_depth (test.py:187-295) + pcd_filter / gipuma_filter
  read_cam_file, build_view_sets, scale_intrinsics, stage_matrices, depth_values   <- the loader's camera and pair rules
  save_pfm, write_cam                   <- datasets/data_io.py:39-64, test.py:149-166 / test_tt.py:159-176

A scene folder has the MVSNet layout: {scan}/pair.txt, {scan}/images/%08d.jpg and {scan}/cams/%08d_cam.txt (dtu also
{scan}/cams_1/, T&T with use_short_range short_range_cameras/cams_{scan}/).  Each image the view sets name is decoded once
(PIL, as the loader does), uploaded once as uint8 and resized once on the device (csrc/image_prep.cu, bit-identical to
cv2.resize); the scene stays resident as uint8 [N,H,W,3], and each item normalises its view set from it on the device.
"""
import concurrent.futures
import ctypes
import os
import sys

import numpy as np
import torch

from . import _lib

MAX_VIEWS = 64        # views per normalize call (csrc/image_prep.cu)
TT_PAD_ROWS = 4       # general_eval.py:115-116
CONF_CHOICES = ("mean", "stage4")


# ---- the loader's camera and pair rules (numpy float32, as general_eval.py computes them)
def read_cam_file(filename, dataset, ndepths, interval_scale):
    """-> (intrinsics float32 [3,3], extrinsics float32 [4,4], depth_min, depth_interval): general_eval.py:80-110 (T&T's
    cy + 4, intrinsics / 4, dtu cams_1's interval 2.5, a third token's num_depth, eth3d's depth_max, interval_scale)."""
    with open(filename) as f:
        lines = [line.rstrip() for line in f.readlines()]
    extrinsics = np.fromstring(" ".join(lines[1:5]), dtype=np.float32, sep=" ").reshape((4, 4))
    intrinsics = np.fromstring(" ".join(lines[7:10]), dtype=np.float32, sep=" ").reshape((3, 3))
    if dataset == "tt":
        intrinsics[1, 2] += 4
    intrinsics[:2, :] /= 4.0
    tokens = lines[11].split()
    depth_min = float(tokens[0])
    depth_interval = 2.5 if "cams_1" in filename else float(tokens[1])
    if len(tokens) >= 3:
        depth_max = depth_min + int(float(tokens[2])) * depth_interval
        depth_interval = (depth_max - depth_min) / ndepths
    if dataset == "eth3d":
        depth_max = float(tokens[1])
        depth_interval = (depth_max - depth_min) / ndepths
    depth_interval *= interval_scale
    return intrinsics, extrinsics, depth_min, depth_interval


def build_view_sets(pair_path, nviews):
    """[(ref, [src, ...]), ...] of general_eval.py:56-71: views without sources are dropped, the sources are padded to
    nviews with the first one and cut to nviews - 1."""
    sets = []
    with open(pair_path) as f:
        for _ in range(int(f.readline())):
            ref = int(f.readline().rstrip())
            srcs = [int(x) for x in f.readline().rstrip().split()[1::2]]
            if srcs:
                if len(srcs) < nviews:
                    srcs += [srcs[0]] * (nviews - len(srcs))
                sets.append((ref, srcs[:nviews - 1]))
    return sets


def scale_intrinsics(intrinsics, h, w, max_h, max_w):
    """scale_mvs_input's camera half (general_eval.py:120-127) for an h x w (padded) image; in place, returns it"""
    intrinsics[0, :] *= 1.0 * max_w / w
    intrinsics[1, :] *= 1.0 * max_h / h
    return intrinsics


def stage_matrices(proj):
    """proj float32 [V,2,4,4] -> {stage1..4: [V,2,4,4]}, intrinsic rows 0-1 x 0.5, 1, 2, 4 (general_eval.py:229-242)"""
    out = {}
    for s, f in enumerate((0.5, None, 2, 4)):
        m = proj.copy()
        if f is not None:
            m[:, 1, :2, :] = proj[:, 1, :2, :] * f
        out[f"stage{s + 1}"] = m
    return out


def depth_values(depth_min, depth_interval, ndepths):
    """general_eval.py:223"""
    return np.arange(depth_min, depth_interval * (ndepths - 0.5) + depth_min, depth_interval, dtype=np.float32)


def cam_path(datapath, scan, vid, dataset, use_short_range=False):
    """general_eval.py:170-178"""
    if dataset == "tt":
        if use_short_range:
            return os.path.join(datapath, "short_range_cameras/cams_{}/{:0>8}_cam.txt".format(scan.lower(), vid))
        return os.path.join(datapath, "{}/cams/{:0>8}_cam.txt".format(scan, vid))
    p = os.path.join(datapath, "{}/cams_1/{:0>8}_cam.txt".format(scan, vid))
    return p if os.path.exists(p) else os.path.join(datapath, "{}/cams/{:0>8}_cam.txt".format(scan, vid))


# ---- the files test.py / test_tt.py write per reference view
def save_pfm(filename, image, scale=1):
    """datasets/data_io.py:39-64 for a float32 [H,W] map (greyscale, little-endian)"""
    image = np.asarray(image)
    if image.dtype != np.float32 or image.ndim != 2:
        raise ValueError(f"save_pfm: expected a float32 [H,W] map, got {image.dtype} {image.shape}")
    image = np.flipud(image)
    if image.dtype.byteorder == "<" or image.dtype.byteorder == "=" and sys.byteorder == "little":
        scale = -scale
    with open(filename, "wb") as f:
        f.write(b"Pf\n")
        f.write("{} {}\n".format(image.shape[1], image.shape[0]).encode("utf-8"))
        f.write(("%f\n" % scale).encode("utf-8"))
        image.tofile(f)


def write_cam(filename, cam, depth_range=None):
    """test.py:149-166 for a float32 [2,4,4] camera; with depth_range (two float32 scalars), test_tt.py:159-176"""
    rows = ["extrinsic\n"] + ["".join(str(cam[0][i][j]) + " " for j in range(4)) + "\n" for i in range(4)] + ["\n"]
    rows += ["intrinsic\n"] + ["".join(str(cam[1][i][j]) + " " for j in range(3)) + "\n" for i in range(3)]
    if depth_range is None:
        rows.append("\n" + " ".join(str(cam[1][3][j]) for j in range(4)) + "\n")
    else:
        rows.append("\n" + f"{depth_range[0]} {depth_range[1]}")
    with open(filename, "w") as f:
        f.write("".join(rows))


# ---- device kernels
def resize_u8(images, H, W, pad_rows=0, out=None):
    """uint8 [N,h,w,3] (CUDA, contiguous) -> uint8 [N,H,W,3]: edge pad of pad_rows rows top and bottom, then cv2.resize's
    INTER_LINEAR, bit for bit (csrc/image_prep.cu)."""
    if not isinstance(images, torch.Tensor) or not images.is_cuda:
        raise RuntimeError("resize_u8: expected a CUDA tensor (the hot path has no CPU fallback)")
    if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3 or not images.is_contiguous():
        raise ValueError(f"resize_u8: expected contiguous uint8 [N,h,w,3] images, got {images.dtype} {tuple(images.shape)}")
    N, h, w, _ = images.shape
    if out is None:
        out = torch.empty(N, H, W, 3, dtype=torch.uint8, device=images.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (N, H, W, 3) or not out.is_contiguous():
        raise ValueError(f"resize_u8: out must be contiguous uint8 {(N, H, W, 3)}, got {out.dtype} {tuple(out.shape)}")
    _lib.call("mvsf_image_resize_u8", images, N, h, w, int(pad_rows), out, int(H), int(W))
    return out


def normalize(scene_u8, views, norm=True, colour=False):
    """-> (norm [V,3,H,W] or None, colour [V,3,H,W] or None) of the images `views` of the uint8 [N,H,W,3] scene:
    ToTensor + Normalize (general_eval.py:29-32) and the saved-and-read-back fusion colour of test.py:287-292."""
    if scene_u8.dtype != torch.uint8 or scene_u8.dim() != 4 or scene_u8.shape[3] != 3 or not scene_u8.is_contiguous():
        raise ValueError(f"normalize: expected a contiguous uint8 [N,H,W,3] scene, got {scene_u8.dtype} {tuple(scene_u8.shape)}")
    views = [int(v) for v in views]
    N, H, W, _ = scene_u8.shape
    if not 1 <= len(views) <= MAX_VIEWS:
        raise ValueError(f"normalize: {len(views)} views, supported 1..{MAX_VIEWS}")
    outs = [torch.empty(len(views), 3, H, W, dtype=torch.float32, device=scene_u8.device) if want else None
            for want in (norm, colour)]
    idx = (ctypes.c_int * len(views))(*views)
    _lib.call("mvsf_image_normalize", scene_u8, N, idx, len(views), H, W, *outs)
    return tuple(outs)


class Scene:
    """A scene resident on the device: images uint8 [N,H,W,3] (the prepared images, in view-id order), view_ids [N],
    view_sets [(ref, [src, ...])] (the loader's items), pairs (pair.txt as test.py reads it), and per item the stage
    matrices and depth values the loader computes."""

    def __init__(self, images, view_ids, view_sets, pairs, projs, dvals, dataset):
        self.images, self.view_ids, self.view_sets, self.pairs = images, view_ids, view_sets, pairs
        self.projs, self.dvals, self.dataset = projs, dvals, dataset
        self.slot = {v: k for k, v in enumerate(view_ids)}

    def __len__(self):
        return len(self.view_sets)

    def item(self, k):
        """-> (imgs [1,V,3,H,W], {stage1..4: [1,V,2,4,4]}, depth_values [1,D]) on the device: MVSDataset[k] after the
        default collate and tocuda, bit for bit."""
        ref, srcs = self.view_sets[k]
        imgs, _ = normalize(self.images, [self.slot[v] for v in [ref] + srcs])
        dev = self.images.device
        proj = {s: torch.from_numpy(m)[None].to(dev) for s, m in self.projs[k].items()}
        return imgs[None], proj, torch.from_numpy(self.dvals[k])[None].to(dev)


def _decode(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"))


class ScenePlan:
    """What a scene folder's pair file asks the loader for: view_sets (its items), pairs (as test.py reads them),
    view_ids (every view an item names, sorted) and their image and camera paths."""

    def __init__(self, datapath, scan, dataset, nviews, use_short_range=False):
        if isinstance(nviews, bool) or int(nviews) != nviews or nviews < 2:
            raise ValueError(f"load_scene: nviews = {nviews!r} must be a whole number >= 2")
        from .fusion import read_pair_file
        self.dataset = dataset
        pair_path = os.path.join(datapath, scan, "pair.txt")
        self.view_sets = build_view_sets(pair_path, int(nviews))
        if not self.view_sets:
            raise ValueError(f"load_scene: {pair_path} names no view with a source view")
        self.pairs = read_pair_file(pair_path)
        self.view_ids = sorted({v for ref, srcs in self.view_sets for v in [ref] + srcs})
        self.img_paths = [os.path.join(datapath, "{}/images/{:0>8}.jpg".format(scan, v)) for v in self.view_ids]
        self.cam_paths = [cam_path(datapath, scan, v, dataset, use_short_range) for v in self.view_ids]
        for p in self.img_paths + self.cam_paths:
            if not os.path.isfile(p):
                raise FileNotFoundError(f"load_scene: {p} is missing (a view set of {pair_path} names its view)")
        self.pad = TT_PAD_ROWS if dataset == "tt" else 0

    def cameras(self, sizes, ndepths, interval_scale, max_h, max_w):
        """-> (per item {stage1..4: [V,2,4,4]}, per item depth_values [D]) for the source image sizes [(h, w)] of
        view_ids, as general_eval.py:186-242 computes them"""
        cams = []
        for path, (h, w) in zip(self.cam_paths, sizes):
            intr, extr, dmin, dint = read_cam_file(path, self.dataset, ndepths, interval_scale)
            scale_intrinsics(intr, h + 2 * self.pad, w, max_h, max_w)
            proj = np.zeros((2, 4, 4), dtype=np.float32)
            proj[0, :4, :4] = extr
            proj[1, :3, :3] = intr
            cams.append((proj, dmin, dint))
        slot = {v: k for k, v in enumerate(self.view_ids)}
        projs, dvals = [], []
        for ref, srcs in self.view_sets:
            projs.append(stage_matrices(np.stack([cams[slot[v]][0] for v in [ref] + srcs])))
            dvals.append(depth_values(cams[slot[ref]][1], cams[slot[ref]][2], ndepths))
        return projs, dvals


def _check_size(name, v):
    if isinstance(v, bool) or int(v) != v or v < 32 or v % 32:
        raise ValueError(f"load_scene: {name} = {v!r} must be a positive multiple of 32 (what DINOv2MVSNet accepts)")
    return int(v)


def load_scene(datapath, scan, dataset, nviews, ndepths, interval_scale, max_h, max_w, use_short_range=False, device="cuda",
               workers=8):
    """-> Scene: the items of general_eval.MVSDataset(datapath, [scan], "test", nviews, ndepths, interval_scale,
    max_h=max_h, max_w=max_w, dataset=dataset, use_short_range=use_short_range), with every image decoded once (in a
    pool of `workers` threads), uploaded once from pinned memory on a side stream and resized once on the device."""
    max_h, max_w = _check_size("max_h", max_h), _check_size("max_w", max_w)
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"load_scene: device {device} is not a CUDA device (the hot path has no CPU fallback)")
    plan = ScenePlan(datapath, scan, dataset, nviews, use_short_range)

    N = len(plan.view_ids)
    main = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device)
    images = torch.empty(N, max_h, max_w, 3, dtype=torch.uint8, device=device)
    side.wait_stream(main)
    images.record_stream(side)
    sizes = []
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, int(workers))) as pool, torch.cuda.stream(side):
        for k, arr in enumerate(pool.map(_decode, plan.img_paths)):
            staged = torch.empty(arr.shape, dtype=torch.uint8, pin_memory=True)
            staged.numpy()[...] = arr
            resize_u8(staged.to(device, non_blocking=True)[None], max_h, max_w, plan.pad, out=images[k:k + 1])
            sizes.append(arr.shape[:2])
    main.wait_stream(side)
    projs, dvals = plan.cameras(sizes, int(ndepths), interval_scale, max_h, max_w)
    return Scene(images, plan.view_ids, plan.view_sets, plan.pairs, projs, dvals, dataset)


def _confidence(out, conf_choose, combine_reg_conf):
    conf = out["photometric_confidence"] if conf_choose == "mean" else out["stage4"]["photometric_confidence"]
    if combine_reg_conf:
        conf = (conf * 3 + out["stage4"]["photometric_confidence"]) / 4
    return (conf[0] * 255).to(torch.uint8)   # np.uint8 of a float32 in [0, 255]: truncation


def reconstruct_scene(model, scene, method, tmp=(5.0, 5.0, 5.0, 1.0), conf_choose="mean", combine_reg_conf=False,
                      out_dir=None, **fusion_args):
    """-> (xyz [M,3] float32, rgb [M,3] uint8) on the device: model(*scene.item(k), tmp) for every item, the confidence
    test.py / test_tt.py save (conf_choose "mean" or "stage4"; combine_reg_conf: (conf 3 + stage4) / 4; then uint8 of
    conf 255), and the fusion of the depth maps with the confidences u8 / 255, the reference cameras (stage4) and the
    colours test.py saves: fuse_scene(method "pcd" / "dpcd", the scene's pairs) or fuse_scene_gipuma (method "gipuma").
    Fusion view k is item k's reference view.  fusion_args go to the fusion call.

    With out_dir, also writes what the reference's drivers write per reference view, byte for byte: depth_est/%08d.pfm,
    confidence/%08d.npy (uint8) and cams/%08d_cam.txt (test_tt.py's layout for dataset "tt", else test.py's)."""
    from .fusion import fuse_scene, fuse_scene_gipuma
    if method not in ("pcd", "dpcd", "gipuma"):
        raise ValueError(f"reconstruct_scene: method {method!r} is not one of pcd, dpcd, gipuma")
    if conf_choose not in CONF_CHOICES:
        raise ValueError(f"reconstruct_scene: conf_choose {conf_choose!r} is not one of {CONF_CHOICES}")
    R = len(scene)
    H, W = scene.images.shape[1:3]
    dev = scene.images.device
    depths = torch.empty(R, H, W, dtype=torch.float32, device=dev)
    confs = torch.empty(R, H, W, dtype=torch.uint8, device=dev)
    cams = torch.empty(R, 2, 4, 4, dtype=torch.float32, device=dev)
    with torch.no_grad():
        for k in range(R):
            imgs, proj, dv = scene.item(k)
            out = model(imgs, proj, dv, list(tmp))
            depths[k] = out["refined_depth"][0]
            confs[k] = _confidence(out, conf_choose, combine_reg_conf)
            cams[k] = proj["stage4"][0, 0]
    if out_dir is not None:
        _write_outputs(out_dir, scene, depths, confs, cams)
    cams[:, 1, 3, 3] = 1.0   # as test.py's read_camera_parameters rebuilds the camera
    refs = [scene.slot[ref] for ref, _ in scene.view_sets]
    colours = torch.cat([normalize(scene.images, refs[i:i + MAX_VIEWS], norm=False, colour=True)[1]
                         for i in range(0, R, MAX_VIEWS)])
    conf = confs.float() / 255
    if method == "gipuma":
        return fuse_scene_gipuma(depths, conf, cams, colours, **fusion_args)
    item = {ref: k for k, (ref, _) in enumerate(scene.view_sets)}
    pairs = []
    for ref, srcs in scene.pairs:   # a source without a depth map is skipped, as test.py's TTDataset does
        srcs = [item[s] for s in srcs if s in item]
        if ref in item and srcs:
            pairs.append((item[ref], srcs))
    return fuse_scene(depths, conf, cams, colours, pairs, method, **fusion_args)


def _write_outputs(out_dir, scene, depths, confs, cams):
    for sub in ("depth_est", "confidence", "cams"):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    depths, confs, cams = depths.cpu().numpy(), confs.cpu().numpy(), cams.cpu().numpy()
    for k, (ref, _) in enumerate(scene.view_sets):
        save_pfm(os.path.join(out_dir, "depth_est/{:0>8}.pfm".format(ref)), depths[k])
        np.save(os.path.join(out_dir, "confidence/{:0>8}.npy".format(ref)), confs[k])
        dr = (scene.dvals[k][0], scene.dvals[k][-1]) if scene.dataset == "tt" else None
        write_cam(os.path.join(out_dir, "cams/{:0>8}_cam.txt".format(ref)), cams[k], dr)
