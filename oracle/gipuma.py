"""ORACLE - TEST INFRASTRUCTURE ONLY.  Torch restatement of the gipuma fusion (probability_filter and fusibile's
cross-view voting and point averaging at normal_thresh = 360, misc/gipuma.py:160-228), step by step, one reference view at
a time, in the operation order csrc/fusion.cu evaluates (each product, sum and quotient rounded on its own).  Runs in fp32
(parity) and fp64 (truth, and the margin of every decision).

A scene is depths [N,H,W], confs [N,H,W], cams [N,2,4,4] (slot 0 extrinsic E, slot 1 [:3,:3] intrinsic K), images
[N,3,H,W] in [0,1].  The camera table is [N,32] per view: P = K E[:3] (12, row-major), M^-1 of M = P[:, :3] (9,
row-major), f b with f = K[0,0] / K[2,2] and b = 0.54, zero padding; computed in fp64 and rounded once.

The rules (the contract of mvsf_fusion_gipuma_*):
  - D = depth where conf > prob_threshold and depth_min <= depth <= depth_max, else 0; valid iff D > 0.
  - Reference views in index order; a pixel p = (x, y) of view r with used_r(p) = 0 and D_r(p) > 0 has the world point
    X = M_r^-1 (d x - p4.x, d y - p4.y, d - p4.z) (integer pixel positions, no +0.5).
  - For every other view s: t = P_s [X; 1], x' = t.x / t.z, y' = t.y / t.z; if 0 <= x' < W and 0 <= y' < H the source
    pixel is q = (floor x', floor y'), consistent iff D_s(q) > 0 and |f_r b / t.z - f_r b / D_s(q)| < disp_threshold.
  - n consistent views >= num_consistent: one point, the mean of X and the consistent X_s = M_s^-1 (D_s(q) q.x - ...),
    rgb the integer mean of round(255 image) over the same pixels; every consistent q is marked used.
"""
import torch

BASELINE = 0.54
CAM = 32


def camera_table(cams, dtype=torch.float32):
    """[N,32] camera table (layout above), fp64 rounded once to dtype"""
    c = cams.double()
    E, K = c[:, 0], c[:, 1, :3, :3]
    P = K @ E[:, :3]
    t = torch.zeros(c.shape[0], CAM, dtype=torch.float64, device=cams.device)
    t[:, :12] = P.reshape(-1, 12)
    t[:, 12:21] = torch.linalg.inv(P[:, :, :3]).reshape(-1, 9)
    t[:, 21] = K[:, 0, 0] / K[:, 2, 2] * BASELINE
    return t.to(dtype)


def filter_depths(depths, confs, prob_threshold=0.5, depth_min=0.001, depth_max=100000.0):
    """-> D [N,H,W] fp32 (the comparisons in fp32 against fp32 thresholds, as the kernel takes them) and the depth-range
    margin [N,H,W] fp64 of every pixel that passes the confidence test (inf elsewhere)"""
    thr = torch.tensor([prob_threshold, depth_min, depth_max], dtype=torch.float32)
    p, lo, hi = (float(v) for v in thr)
    d = depths.float()
    keep = (confs.float() > p) & (d >= lo) & (d <= hi)
    dd = d.double()
    rng = torch.minimum((dd - lo).abs() / lo, (dd - hi).abs() / hi)
    rng = torch.where(confs.float() > p, _nan_to_big(rng), torch.full_like(rng, float("inf")))
    return torch.where(keep, d, torch.zeros_like(d)), rng


def _nan_to_big(m):
    return torch.where(torch.isnan(m), torch.full_like(m, float("inf")), m)


def unproject(cam, x, y, d):
    """X = M^-1 (d x - p4.x, d y - p4.y, d - p4.z) in the kernel's order -> [X0, X1, X2]"""
    a = [d * x - cam[3], d * y - cam[7], d - cam[11]]
    return [(cam[12 + 3 * i] * a[0] + cam[13 + 3 * i] * a[1]) + cam[14 + 3 * i] * a[2] for i in range(3)]


def _coord_margin(c, size):
    """relative distance of a projected coordinate from the nearest decision boundary: the nearest integer (the floor and
    the bounds 0 and size) inside the image, the nearer bound outside it"""
    inside = (c >= 0) & (c < size)
    dist = torch.where(inside, (c - torch.round(c)).abs(), torch.minimum(c.abs(), (c - size).abs()))
    return _nan_to_big(dist / c.abs().clamp_min(1.0))


def step(ref, D, table, images, used, disp_threshold=0.2, num_consistent=3, dtype=torch.float32, range_margin=None,
         footprint_below=None):
    """One reference view from the used state `used` [N,H,W] (not modified) -> dict(
         keep [H,W] bool      the pixels that emit, row-major = the order of the points,
         xyz [M,3], rgb [M,3] uint8, used [N,H,W] uint8 (after the step), n [H,W] (consistent views of every valid pixel),
         margin [H,W] fp64    the smallest relative distance of any decision of the pixel to its boundary (inf for a
                              pixel that takes none; meaningful in fp64),
         footprint [N,H,W]    (with footprint_below) the 3x3 neighbourhoods of the source pixels that the pixels of margin
                              < footprint_below land on: the used marks a near-boundary decision could move)"""
    N, H, W = D.shape
    dev = D.device
    D = D.to(dtype)
    tab = table.to(dtype)
    disp = float(torch.tensor(disp_threshold, dtype=torch.float32))
    cam_r = tab[ref]
    x = torch.arange(W, dtype=dtype, device=dev).expand(H, W)
    y = torch.arange(H, dtype=dtype, device=dev).unsqueeze(1).expand(H, W)
    d = D[ref]
    valid = (d > 0) & (used[ref] == 0)
    X = unproject(cam_r, x, y, d)
    fb = cam_r[21]
    n = torch.zeros(H, W, dtype=torch.int64, device=dev)
    margin = torch.full((H, W), float("inf"), dtype=torch.float64, device=dev)
    if range_margin is not None:
        margin = torch.minimum(margin, range_margin[ref].double().to(dev))
    probes = []
    for s in range(N):
        if s == ref:
            continue
        P = tab[s]
        t = [((P[4 * i] * X[0] + P[4 * i + 1] * X[1]) + P[4 * i + 2] * X[2]) + P[4 * i + 3] for i in range(3)]
        xs, ys = t[0] / t[2], t[1] / t[2]
        inb = (xs >= 0) & (xs < W) & (ys >= 0) & (ys < H)
        qx = torch.where(inb, torch.floor(xs), torch.zeros_like(xs)).long()
        qy = torch.where(inb, torch.floor(ys), torch.zeros_like(ys)).long()
        q = qy * W + qx
        ds = torch.where(inb, D[s].reshape(-1)[q], torch.zeros_like(xs))
        dd = (fb / t[2] - fb / ds).abs()
        cons = inb & (ds > 0) & (dd < disp)
        n += cons
        m = torch.minimum(_coord_margin(xs.double(), W), _coord_margin(ys.double(), H))
        m = torch.where(inb & (ds > 0), torch.minimum(m, _nan_to_big((dd.double() - disp).abs() / abs(disp))), m)
        if range_margin is not None:
            m = torch.where(inb, torch.minimum(m, range_margin[s].double().to(dev).reshape(-1)[q]), m)
        margin = torch.where(valid, torch.minimum(margin, m), margin)
        probes.append((s, cons, qx, qy, q, ds, xs, ys, inb))
    keep = valid & (n >= num_consistent)
    total = [X[k].clone() for k in range(3)]
    col = [torch.round(images[ref, k].to(torch.float32) * 255).long() for k in range(3)]
    new_used = used.clone()
    for s, cons, qx, qy, q, ds, _, _, _ in probes:
        Xs = unproject(tab[s], qx.to(dtype), qy.to(dtype), ds)
        hit = cons & keep
        for k in range(3):
            total[k] = torch.where(hit, total[k] + Xs[k], total[k])
            c = torch.round(images[s, k].to(torch.float32) * 255).long().reshape(-1)[q]
            col[k] = torch.where(hit, col[k] + c, col[k])
        new_used[s].view(-1)[q[hit]] = 1
    cnt = (n + 1).to(dtype)
    xyz = torch.stack([(total[k] / cnt)[keep] for k in range(3)], 1)
    rgb = torch.stack([torch.div(col[k], n + 1, rounding_mode="floor")[keep] for k in range(3)], 1).to(torch.uint8)
    out = dict(keep=keep, xyz=xyz, rgb=rgb, used=new_used, n=n, margin=margin)
    if footprint_below is not None:
        low = valid & (margin < footprint_below)
        fp = torch.zeros(N, H, W, dtype=torch.bool, device=dev)
        for s, _, _, _, _, _, xs, ys, _ in probes:
            fx, fy = torch.floor(xs[low]).long(), torch.floor(ys[low]).long()
            for oy in (-1, 0, 1):
                for ox in (-1, 0, 1):
                    cx, cy = fx + ox, fy + oy
                    ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
                    fp[s][cy[ok], cx[ok]] = True
        out["footprint"] = fp
    return out


def fuse_scene(depths, confs, cams, images, prob_threshold=0.5, disp_threshold=0.2, num_consistent=3, depth_min=0.001,
               depth_max=100000.0, dtype=torch.float32, table=None, order=None):
    """-> xyz [M,3], rgb [M,3] uint8, the flat index (view * H*W + pixel) of every point and the final used marks; views in
    `order` (index order by default, the contract), pixels row-major.  table: the camera table to use (the kernel's own)."""
    N, H, W = depths.shape
    D, _ = filter_depths(depths, confs, prob_threshold, depth_min, depth_max)
    table = camera_table(cams, dtype) if table is None else table
    used = torch.zeros(N, H, W, dtype=torch.uint8, device=depths.device)
    xyz, rgb, flat = [], [], []
    for r in (range(N) if order is None else order):
        o = step(r, D, table, images, used, disp_threshold, num_consistent, dtype)
        used = o["used"]
        xyz.append(o["xyz"])
        rgb.append(o["rgb"])
        flat.append(torch.nonzero(o["keep"].reshape(-1)).squeeze(1) + r * H * W)
    return torch.cat(xyz), torch.cat(rgb), torch.cat(flat), used
