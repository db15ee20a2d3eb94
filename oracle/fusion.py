"""ORACLE - TEST INFRASTRUCTURE ONLY.  Torch restatement of the reference's depth-map fusion (test.py:387-517 over
misc/fusion.py:79-165), written from the formulas as per-pixel chains of elementwise operations in a fixed order, which is
the order csrc/fusion.cu evaluates.  Runs on any device in fp32 (parity) and fp64 (truth, and the margins of every
threshold comparison).  Camera inverses are taken in fp64 and rounded once to the working type.

A scene is depths [N,H,W], confs [N,H,W], cams [N,2,4,4] (slot 0 extrinsic, slot 1 [:3,:3] intrinsic), images [N,3,H,W].
"""
import torch

EPS = 1e-9


def camera_inverses(cams, dtype):
    """[N,2,4,4]: slot 0 = E^-1, slot 1 = inverse of (K in the [:3,:3] of an identity)  (fusion.py:24,32 invert per call)"""
    c = cams.double()
    K = torch.eye(4, dtype=torch.float64, device=cams.device).repeat(c.shape[0], 1, 1)
    K[:, :3, :3] = c[:, 1, :3, :3]
    return torch.stack([torch.linalg.inv(c[:, 0]), torch.linalg.inv(K)], 1).to(dtype)


def pixel_centres(H, W, dtype, device):
    """fusion.py:8-13: x + 0.5, y + 0.5 as [H,W] each"""
    x = (torch.arange(W, dtype=dtype, device=device) + 0.5).expand(H, W)
    y = (torch.arange(H, dtype=dtype, device=device) + 0.5).unsqueeze(1).expand(H, W)
    return x, y


def _dot(row, vec):
    acc = row[0] * vec[0]
    for a, b in zip(row[1:], vec[1:]):
        acc = acc + (a * b if b is not None else a)
    return acc


def img2world(inv, u, v, d):
    """idx_img2cam + idx_cam2world (fusion.py:23-34) with the view's inverses [2,4,4] -> 4 homogeneous world coordinates"""
    Ei, Ki = inv[0], inv[1]
    c = [_dot(Ki[i, :3], [u, v, None]) for i in range(3)]
    dc = c[2] + EPS
    c = [ci / dc * d for ci in c]
    w = [_dot(Ei[i], [c[0], c[1], c[2], None]) for i in range(4)]
    dw = w[3] + EPS
    return [wi / dw for wi in w]


def reproject(inv_a, cam_b, u, v, d):
    """pixel (u, v) of view a at depth d -> (x, y) in view b's image and its depth z in b's camera: the chain above, then
    idx_world2cam + idx_cam2img (fusion.py:37-47)"""
    w = img2world(inv_a, u, v, d)
    E, K = cam_b[0], cam_b[1]
    q = [_dot(E[i], w) for i in range(4)]
    dq = q[3] + EPS
    q = [qi / dq for qi in q]
    dr = q[3] + EPS
    r = [q[i] / dr for i in range(3)]
    im = [_dot(K[i, :3], r) for i in range(3)]
    di = im[2] + EPS
    return im[0] / di, im[1] / di, q[2]


def bilinear(maps, gx, gy):
    """F.grid_sample(mode='bilinear', padding_mode='zeros', align_corners=True) of each [H,W] map at normalised (gx, gy):
    corners nw, ne, sw, se accumulated in that order, a corner outside the map contributes zero"""
    H, W = maps[0].shape
    ix = (gx + 1) / 2 * (W - 1)
    iy = (gy + 1) / 2 * (H - 1)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    wx = [(x0 + 1) - ix, ix - x0]
    wy = [(y0 + 1) - iy, iy - y0]
    out = [torch.zeros_like(ix) for _ in maps]
    for k in range(4):
        fx, fy = x0 + (k & 1), y0 + (k >> 1)
        inb = (fx >= 0) & (fx <= W - 1) & (fy >= 0) & (fy <= H - 1)
        q = torch.where(inb, fy * W + fx, torch.zeros_like(fx)).long()
        wgt = wx[k & 1] * wy[k >> 1]
        for j, m in enumerate(maps):
            out[j] = out[j] + torch.where(inb, m.reshape(-1)[q] * wgt, torch.zeros_like(wgt))
    return out


def _margin(a, b):
    """relative distance of the comparison a < b from flipping"""
    return (a - b).abs() / b.abs().clamp_min(1e-30)


def _nan_to_big(m):
    return torch.where(torch.isnan(m), torch.full_like(m, float("inf")), m)


def filter_pcd(ref, srcs, depths, confs, cams, conf=0.5, thres_view=2, thres_disp=1.0, dtype=torch.float32, inv=None):
    """filter_depth, test.py:395-412 -> mask [H,W] bool, averaged depth [H,W], margin [H,W]: the smallest relative
    distance to its threshold over the comparisons of the pixel (meaningful in fp64).  inv: camera inverses to use instead
    of camera_inverses(cams) (the kernels' own, so that a parity run shares every input of the per-pixel chain)."""
    depths, confs, cams_t = depths.to(dtype), confs.to(dtype), cams.to(dtype)
    inv = camera_inverses(cams, dtype) if inv is None else inv.to(dtype)
    H, W = depths.shape[-2:]
    u, v = pixel_centres(H, W, dtype, depths.device)
    d_ref = depths[ref]
    total, count = torch.zeros_like(d_ref), torch.zeros_like(d_ref)
    margin = _margin(confs[ref], torch.full_like(d_ref, conf))
    for s in srcs:
        d_src = depths[s] * (confs[s] > conf).to(dtype)                                   # test.py:397-400
        xyd = reproject(inv[s], cams_t[ref], u, v, d_src)                               # get_reproj, fusion.py:87-91
        wx, wy, _ = reproject(inv[ref], cams_t[s], u, v, d_ref)                         # project_img, fusion.py:53-57
        gx = (wx / W * 2 - 1).clamp(-1.1, 1.1)
        gy = (wy / H * 2 - 1).clamp(-1.1, 1.1)
        in_range = (-1 <= gx) & (gx <= 1) & (-1 <= gy) & (gy <= 1)
        bx, by, bd = bilinear(xyd, gx, gy)
        dist = ((bx - u) * (bx - u) + (by - v) * (by - v)).sqrt()                       # vis_filter, fusion.py:99-107
        diff, tol = (d_ref - bd).abs(), torch.maximum(d_ref, bd) * 0.01
        m = (in_range & (dist < thres_disp) & (diff < tol)).to(dtype)
        total, count = total + bd * m, count + m                                         # ave_fusion, fusion.py:110-112
        edge = torch.minimum(torch.minimum((gx.abs() - 1).abs(), (gy.abs() - 1).abs()),
                             torch.minimum(_margin(dist, torch.full_like(dist, thres_disp)), _margin(diff, tol)))
        margin = torch.minimum(margin, _nan_to_big(edge))
        # the confidence test of the source pixels the sample blends
        margin = torch.minimum(margin, _nan_to_big(corner_min(_margin(confs[s], torch.full_like(d_ref, conf)), gx, gy)))
    vis = count.double() >= thres_view - 1.1
    avg = (total + d_ref) / (count + 1)
    return vis & (confs[ref] > conf), avg, margin


def corner_min(m, gx, gy):
    """smallest value of map m over the in-map corners of the bilinear sample at (gx, gy) (inf where there is none)"""
    H, W = m.shape
    ix, iy = (gx + 1) / 2 * (W - 1), (gy + 1) / 2 * (H - 1)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    out = torch.full_like(ix, float("inf"))
    for k in range(4):
        fx, fy = x0 + (k & 1), y0 + (k >> 1)
        inb = (fx >= 0) & (fx <= W - 1) & (fy >= 0) & (fy <= H - 1)
        q = torch.where(inb, fy * W + fx, torch.zeros_like(fx)).long()
        out = torch.minimum(out, torch.where(inb, m.reshape(-1)[q], out))
    return out


def filter_dpcd(ref, srcs, depths, confs, cams, conf=0.5, dist_base=4.0, rel_diff_base=1300.0, dtype=torch.float32, inv=None):
    """dynamic_filter_depth, test.py:453-483 -> mask, averaged depth, margin as filter_pcd.  One source view leaves no
    threshold (the reference fails there): nothing is accepted, the averaged depth is the reference depth."""
    depths, confs, cams_t = depths.to(dtype), confs.to(dtype), cams.to(dtype)
    inv = camera_inverses(cams, dtype) if inv is None else inv.to(dtype)
    H, W = depths.shape[-2:]
    V = len(srcs)
    u, v = pixel_centres(H, W, dtype, depths.device)
    d_ref = depths[ref]
    steps = torch.arange(2, V + 1, device=depths.device).to(dtype)
    t_dist, t_rel = steps / dist_base, steps / rel_diff_base                             # fusion.py:160-161
    votes = torch.zeros(max(V - 1, 0), H, W, dtype=torch.int64, device=depths.device)
    total = torch.zeros_like(d_ref)
    margin = _margin(confs[ref], torch.full_like(d_ref, conf))
    for s in srcs:
        wx, wy, _ = reproject(inv[ref], cams_t[s], u, v, d_ref)                         # get_reproj_dynamic, fusion.py:122-127
        gx = wx / ((W - 1) / 2) - 1
        gy = wy / ((H - 1) / 2) - 1
        d = bilinear([depths[s]], gx, gy)[0]
        rx, ry, rz = reproject(inv[s], cams_t[ref], wx, wy, d)                          # fusion.py:140-148
        dist = ((rx - u) * (rx - u) + (ry - v) * (ry - v)).sqrt()                       # vis_filter_dynamic, fusion.py:157-162
        rel = (d_ref - rz).abs() / d_ref
        for j in range(V - 1):
            ok = (dist < t_dist[j]) & (rel < t_rel[j])
            votes[j] += ok
            margin = torch.minimum(margin, _nan_to_big(torch.minimum(_margin(dist, t_dist[j].expand_as(dist)),
                                                                      _margin(rel, t_rel[j].expand_as(rel)))))
            if j == V - 2:
                total = total + torch.where(ok, rz, torch.zeros_like(rz))               # test.py:471-475
    geo = torch.zeros(H, W, dtype=torch.bool, device=depths.device)
    for j in range(V - 1):
        geo = geo | (votes[j] >= j + 2)                                                  # test.py:477-478
    last = votes[V - 2] if V >= 2 else torch.zeros(H, W, dtype=torch.int64, device=depths.device)
    avg = (total + d_ref) / (last + 1).to(dtype)
    return geo & (confs[ref] > conf), avg, margin


def view_points(ref, avg, cams, dtype=torch.float32, inv=None):
    """test.py:410-412: world points [H,W,3] of the averaged depth"""
    inv = camera_inverses(cams, dtype) if inv is None else inv.to(dtype)
    H, W = avg.shape
    u, v = pixel_centres(H, W, dtype, avg.device)
    w = img2world(inv[ref], u, v, avg.to(dtype))
    return torch.stack(w[:3], -1)


def filter_view(ref, srcs, depths, confs, cams, method, conf=0.5, thres_view=2, thres_disp=1.0, dist_base=4.0,
                rel_diff_base=1300.0, dtype=torch.float32, inv=None):
    if method == "pcd":
        return filter_pcd(ref, srcs, depths, confs, cams, conf, thres_view, thres_disp, dtype, inv)
    if method == "dpcd":
        return filter_dpcd(ref, srcs, depths, confs, cams, conf, dist_base, rel_diff_base, dtype, inv)
    raise ValueError(method)


def fuse_scene(depths, confs, cams, images, pairs, method, n_src_views=10, dtype=torch.float32, **kw):
    """-> xyz [M,3], rgb [M,3] uint8, and the flat index (view position in `pairs` * H*W + pixel) of every point: views in
    pair order, pixels row-major (test.py:417-429)"""
    H, W = depths.shape[-2:]
    xyz, rgb, flat = [], [], []
    for k, (ref, srcs) in enumerate(pairs):
        mask, avg, _ = filter_view(ref, list(srcs)[:n_src_views], depths, confs, cams, method, dtype=dtype, **kw)
        pts = view_points(ref, avg, cams, dtype)
        xyz.append(pts[mask])
        rgb.append((images[ref].to(torch.float32) * 255).permute(1, 2, 0)[mask].to(torch.uint8))   # test.py:421-424
        flat.append(torch.nonzero(mask.reshape(-1)).squeeze(1) + k * H * W)
    return torch.cat(xyz), torch.cat(rgb), torch.cat(flat)
