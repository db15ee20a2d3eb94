"""Depth-map fusion on the GPU: a scene's depth maps -> one coloured point cloud, the step the reference runs right after
the model (test.py:552-560).

  filter_view(ref_idx, src_idx, depths, confs, cams, method, ...)     <- one iteration of test.py:395-408 / :453-480
  fuse_scene(depths, confs, cams, images, pairs, method, ...)         <- filter_depth / dynamic_filter_depth, test.py:387-517
  fuse_scene_gipuma(depths, confs, cams, images, ...)                 <- gipuma_filter, misc/gipuma.py:208-228 (fusibile)
  gipuma_prepare(...) / gipuma_step(scene, ref, ...)                  <- one reference view of fuse_scene_gipuma
  write_ply(path, xyz, rgb)                                           <- test.py:431-441
  read_pair_file(path)                                                <- test.py:136-146

`method` is "pcd" or "dpcd" (test.py:61); the third method, "gipuma", has its own entry point.  A scene is depths [N,H,W], confs [N,H,W] (fp32 in [0,1], what the model
returns), cams [N,2,4,4] (slot 0 extrinsic, slot 1 [:3,:3] intrinsic) and images [N,3,H,W] (fp32 in [0,1]), all on the
device; the views a pair names are read in place through their indices.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

METHODS = {"pcd": 0, "dpcd": 1}
MAX_SRC_VIEWS = 16


def read_pair_file(path):
    """[(ref_view, [src_view, ...]), ...] of a pair.txt; views without sources are dropped (test.py:136-146)."""
    with open(path) as f:
        tokens = f.read().split("\n")
    pairs = []
    for k in range(int(tokens[0])):
        ref = int(tokens[1 + 2 * k].rstrip())
        srcs = [int(x) for x in tokens[2 + 2 * k].rstrip().split()[1::2]]
        if srcs:
            pairs.append((ref, srcs))
    return pairs


def write_ply(path, xyz, rgb):
    """Binary little-endian PLY with one `vertex` element of x y z (float) and red green blue (uchar), the layout
    test.py:431-441 writes."""
    xyz = np.asarray(xyz.detach().cpu() if isinstance(xyz, torch.Tensor) else xyz)
    rgb = np.asarray(rgb.detach().cpu() if isinstance(rgb, torch.Tensor) else rgb)
    if xyz.ndim != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape:
        raise ValueError(f"write_ply: xyz {xyz.shape} and rgb {rgb.shape} must both be [M,3]")
    vertex = np.empty(len(xyz), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    for k, name in enumerate(("x", "y", "z")):
        vertex[name] = xyz[:, k]
    for k, name in enumerate(("red", "green", "blue")):
        vertex[name] = rgb[:, k]
    header = ("ply\nformat binary_little_endian 1.0\n" + f"element vertex {len(vertex)}\n"
              + "property float x\nproperty float y\nproperty float z\n"
              + "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vertex.tobytes())


def _check_scene(depths, confs, cams, images=None):
    for name, t in (("depths", depths), ("confs", confs), ("cams", cams)) + ((("images", images),) if images is not None else ()):
        if not t.is_cuda:
            raise RuntimeError(f"fusion: {name}: expected a CUDA tensor (the hot path has no CPU fallback)")
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"fusion: {name} must be a contiguous float32 tensor, got {t.dtype}, strides {t.stride()}")
    if depths.dim() != 3 or depths.numel() == 0:
        raise ValueError(f"fusion: depths must be a non-empty [N,H,W], got {tuple(depths.shape)}")
    N, H, W = depths.shape
    if confs.shape != depths.shape or tuple(cams.shape) != (N, 2, 4, 4):
        raise ValueError(f"fusion: confs {tuple(confs.shape)} / cams {tuple(cams.shape)} do not match depths {tuple(depths.shape)}")
    if images is not None and tuple(images.shape) != (N, 3, H, W):
        raise ValueError(f"fusion: images {tuple(images.shape)} do not match depths {tuple(depths.shape)}")
    return N, H, W


def _check_views(ref, srcs, N):
    srcs = [int(s) for s in srcs]
    if not 1 <= len(srcs) <= MAX_SRC_VIEWS:
        raise ValueError(f"fusion: {len(srcs)} source views, supported 1..{MAX_SRC_VIEWS}")
    for v in [int(ref)] + srcs:
        if not 0 <= v < N:
            raise ValueError(f"fusion: view {v} outside the scene's {N} views")
    return int(ref), srcs


def _method(method):
    if method not in METHODS:
        raise ValueError(f"fusion: method {method!r} is not one of {sorted(METHODS)}")
    return METHODS[method]


def _workspace_ints(H, W):
    return _lib.size("mvsf_fusion_workspace_bytes", H, W) // 4


def _prepare_cameras(cams):
    inv = torch.empty_like(cams)
    _lib.call("mvsf_fusion_prepare_cameras", cams, cams.shape[0], inv)
    return inv


def _filter(method, ref, srcs, depths, confs, cams, cams_inv, thr, mask, avg, ws):
    N, H, W = depths.shape
    idx = (ctypes.c_int * len(srcs))(*srcs)
    _lib.call("mvsf_fusion_filter", method, depths, confs, cams, cams_inv, N, ref, idx, len(srcs), H, W, *thr, mask, avg, ws,
              ws.numel() * 4)


def filter_view(ref_idx, src_idx, depths, confs, cams, method, conf=0.5, thres_view=2, thres_disp=1.0, dist_base=4.0,
                rel_diff_base=1300.0):
    """-> (mask bool [H,W], depth_avg [H,W]) of reference view `ref_idx` against the source views `src_idx`; the defaults
    are those of test.py:61-85."""
    m = _method(method)
    N, H, W = _check_scene(depths, confs, cams)
    ref, srcs = _check_views(ref_idx, src_idx, N)
    mask = torch.empty(H, W, dtype=torch.uint8, device=depths.device)
    avg = torch.empty(H, W, dtype=torch.float32, device=depths.device)
    ws = torch.empty(_workspace_ints(H, W), dtype=torch.int32, device=depths.device)
    _filter(m, ref, srcs, depths, confs, cams, _prepare_cameras(cams), (conf, thres_view, thres_disp, dist_base, rel_diff_base),
            mask, avg, ws)
    return mask.bool(), avg


def fuse_scene(depths, confs, cams, images, pairs, method, n_src_views=10, conf=0.5, thres_view=2, thres_disp=1.0,
               dist_base=4.0, rel_diff_base=1300.0):
    """-> (xyz [M,3] float32, rgb [M,3] uint8) on the device: the reference views in the order of `pairs`
    ([(ref, [src, ...]), ...] as read_pair_file returns it, sources cut to `n_src_views` as test.py:337 does), the points
    of a view in row-major pixel order, as the reference emits them.

    Every view is filtered first; the per-view survivor counts then cross to the host in one read, which sizes the cloud
    exactly, and the views are extracted at their offsets.  Between the two passes a view keeps its mask and averaged
    depth (5 bytes per pixel)."""
    m = _method(method)
    N, H, W = _check_scene(depths, confs, cams, images)
    views = [_check_views(ref, list(srcs)[:n_src_views], N) for ref, srcs in pairs]
    if not views:
        raise ValueError("fusion: empty pair list")
    dev, R = depths.device, len(views)
    cams_inv = _prepare_cameras(cams)
    nws = _workspace_ints(H, W)
    masks = torch.empty(R, H, W, dtype=torch.uint8, device=dev)
    avgs = torch.empty(R, H, W, dtype=torch.float32, device=dev)
    ws = torch.empty(R, nws, dtype=torch.int32, device=dev)
    thr = (conf, thres_view, thres_disp, dist_base, rel_diff_base)
    for k, (ref, srcs) in enumerate(views):
        _filter(m, ref, srcs, depths, confs, cams, cams_inv, thr, masks[k], avgs[k], ws[k])
    counts = ws[:, -1].cpu().tolist()   # the one synchronisation of a scene
    total = sum(counts)
    xyz = torch.empty(total, 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(total, 3, dtype=torch.uint8, device=dev)
    base = 0
    for k, (ref, _) in enumerate(views):
        if counts[k]:
            _lib.call("mvsf_fusion_extract", masks[k], avgs[k], ws[k], nws * 4, cams_inv[ref], images[ref], xyz[base:],
                      rgb[base:], counts[k], H, W)
        base += counts[k]
    return xyz, rgb


GIPUMA_CAM = 32   # floats per view of the gipuma camera table (csrc/fusion.cu)


class GipumaScene:
    """The state of a gipuma fusion between reference views: depth [N,H,W] (filtered), cams [N,32] (the camera table:
    P = K E[:3] row-major, M^-1 of M = P[:, :3] row-major, f b, padding), used [N,H,W] uint8 (the source pixels earlier
    views consumed), images [N,3,H,W], and the per-view mask and workspace the steps reuse."""

    def __init__(self, depth, cams, used, images):
        self.depth, self.cams, self.used, self.images = depth, cams, used, images
        N, H, W = depth.shape
        self.mask = torch.empty(H, W, dtype=torch.uint8, device=depth.device)
        self.ws = torch.empty(_workspace_ints(H, W), dtype=torch.int32, device=depth.device)


def _finite(name, x):
    x = float(x)
    if not math.isfinite(x):
        raise ValueError(f"fusion: {name} = {x} is not finite")
    return x


def gipuma_prepare(depths, confs, cams, images, prob_threshold=0.5, depth_min=0.001, depth_max=100000.0):
    """-> GipumaScene with no used marks: probability_filter (misc/gipuma.py:160-177; depth 0 where conf is not
    > prob_threshold) and fusibile's depth range (depth 0 outside [depth_min, depth_max]), and the camera table."""
    prob, dmin, dmax = (_finite(n, x) for n, x in (("prob_threshold", prob_threshold), ("depth_min", depth_min),
                                                      ("depth_max", depth_max)))
    if dmin <= 0:
        raise ValueError(f"fusion: depth_min = {dmin} must be > 0")
    N, H, W = _check_scene(depths, confs, cams, images)
    depth = torch.empty_like(depths)
    table = torch.empty(N, GIPUMA_CAM, dtype=torch.float32, device=depths.device)
    _lib.call("mvsf_fusion_gipuma_prepare", depths, confs, cams, N, H, W, prob, dmin, dmax, depth, table)
    return GipumaScene(depth, table, torch.zeros(N, H, W, dtype=torch.uint8, device=depths.device), images)


def _num_consistent(n):
    if isinstance(n, bool) or float(n) != int(n) or int(n) < 0:
        raise ValueError(f"fusion: num_consistent = {n!r} must be a whole number >= 0")
    return int(n)


def gipuma_step(scene, ref, disp_threshold=0.2, num_consistent=3):
    """-> (xyz [M,3] float32, rgb [M,3] uint8) of reference view `ref` on the device, in row-major pixel order, and
    scene.used updated: a valid pixel not yet used emits a point when at least num_consistent other views are consistent
    with it (its world point lands on a valid source pixel whose disparity f b / depth is within disp_threshold); the
    point and colour are the means over the pixel and those source pixels, which become used.  The view's point count
    crosses to the host in one 4-byte read, which sizes the output."""
    N, H, W = scene.depth.shape
    if not 0 <= int(ref) < N:
        raise ValueError(f"fusion: view {ref} outside the scene's {N} views")
    disp, nc = _finite("disp_threshold", disp_threshold), _num_consistent(num_consistent)
    nbytes = scene.ws.numel() * 4
    _lib.call("mvsf_fusion_gipuma_vote", scene.depth, scene.used, scene.cams, N, int(ref), H, W, disp, nc, scene.mask, scene.ws,
              nbytes)
    M = int(scene.ws[-1])   # the one synchronisation of a view
    xyz = torch.empty(M, 3, dtype=torch.float32, device=scene.depth.device)
    rgb = torch.empty(M, 3, dtype=torch.uint8, device=scene.depth.device)
    if M:
        _lib.call("mvsf_fusion_gipuma_emit", scene.depth, scene.cams, scene.images, N, int(ref), H, W, disp, scene.mask, scene.ws,
                  nbytes, scene.used, xyz, rgb, M)
    return xyz, rgb


def fuse_scene_gipuma(depths, confs, cams, images, prob_threshold=0.5, disp_threshold=0.2, num_consistent=3, depth_min=0.001,
                      depth_max=100000.0):
    """-> (xyz [M,3] float32, rgb [M,3] uint8) on the device: the gipuma fusion of gipuma_filter (misc/gipuma.py:208-228,
    which runs the external fusibile at normal_thresh = 360), every view a reference view, in index order, and every other
    view its source.  The defaults are those of test.py:71-73 and misc/gipuma.py:187-188.  Points come out view by view
    and, within a view, in row-major pixel order, in world coordinates; rgb is the integer mean of round(255 image) over
    the fused pixels.  To threshold confidences saved as uint8 exactly as the reference does, pass conf_u8.float() / 255.

    The views are sequential (each consumes source pixels the next ones no longer fuse): one gipuma_step per view, each
    with one 4-byte read of its point count."""
    _finite("disp_threshold", disp_threshold)
    _num_consistent(num_consistent)
    scene = gipuma_prepare(depths, confs, cams, images, prob_threshold, depth_min, depth_max)
    parts = [gipuma_step(scene, r, disp_threshold, num_consistent) for r in range(depths.shape[0])]
    return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
