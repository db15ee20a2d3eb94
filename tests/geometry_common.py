"""fp64 references of the cascade glue kernels of geometry.cu, evaluated on the kernels' own fp32 inputs, and the cases
of tests/test_gpu_geometry_fp64.py.

- W1 projection composition (`mvsf_compose_geometry`, `mvsf_homography_from_proj`): P = E; P[:3, :4] = K E[:3, :4],
  then P_src P_ref^-1, all in fp64 from the fp32 matrices.  The kernels also work in fp64 and round once.
- F5 / F6 hypothesis scheduling: the inverse hypotheses v (the planes are 1 / v) in fp64 from the fp32 depth values,
  previous depth map and previous planes.  The x2 upsample blends with the kernel's own fp32 source coordinates and
  weights (`blend_axis`): one fp32 rounding of a coordinate near 960 moves a weight by 6e-5, which would swamp the
  kernel's arithmetic on a map whose neighbours differ.
- F7 3-D positions: the rays are restated in torch fp32 op for op (`fmaf(k_r1, y, k_r0 x)` with the fma done in fp64
  and rounded once, then `+ k_r2`, then `x d`), so the extents, a min or max of fp32 values, compare bit for bit.  The
  normalised positions are fp64 from the kernel's kinv, hypotheses and decoded extents.
- S1 soft-argmax: softmax and confidence in fp64; the depth weights are the fp64 softmax of the fp32 product
  `z * tmp`, which is the reference's own fp32 input of that softmax (F.softmax(prob_volume_pre * tmp)).
- S2 confidence averaging: nearest upsampling restated as source indices, in the fp32 arithmetic ATen uses.

Every function runs on the device of its inputs."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import hotpath as O

H100_SMS = 132
POS3D_THREADS, POS3D_BLOCKS_PER_SM = 256, 8   # pos3d_minmax_kernel: blocks of 256, grid capped at 8 x SMs blocks

DTU, TT = (1152, 1536), (1088, 1920)          # full image sizes; stage s runs at 1 / 2^(4 - s)
NDEPTHS, RATIOS, TMP = (32, 16, 8, 4), (4.0, 2.67, 1.5, 1.0), (5.0, 5.0, 5.0, 1.0)   # config.default_args()
DTU_RANGE, TT_RANGE, WIDE_RANGE = (425.0, 931.0), (1.5, 9.0), (0.5, 50.0)


def stage_size(full, s):
    """(H, W) of stage s = 1..4"""
    return full[0] >> (4 - s), full[1] >> (4 - s)


def f32(x):
    """x rounded to fp32, as a Python float (the value a kernel receives for a float argument)"""
    return float(np.float32(x))


def depth_values(lo, hi, Dn=192):
    """[Dn] fp32 depth values evenly spaced from lo to hi (datasets/general_eval.py:223)"""
    return (lo + (hi - lo) * torch.arange(Dn, dtype=torch.float64) / (Dn - 1)).float()


# ------------------------------------------------------------------------------------------------ W1 cameras
def ring_cameras(V, H, W, kind, seed=0):
    """[V, 2, 4, 4] fp32 projection matrices in the reference's layout (slot 0 the extrinsics, slot 1[:3, :3] the
    intrinsics) of V cameras on an arc around a point in front of camera 0.  kind "dtu": 650 mm away, focal 2776.6 px
    at 1536 wide; "tt": 4 m away, focal 1170 px at 1920 wide, with a small skew so that every entry of K^-1 is used.
    Each camera gets its own seeded jitter of the pose, the focal length and the principal point."""
    g = torch.Generator().manual_seed(seed)
    u = lambda: float(torch.rand((), generator=g, dtype=torch.float64)) * 2 - 1   # noqa: E731
    radius, focal, width, skew = (650.0, 2776.6, 1536.0, 0.0) if kind == "dtu" else (4.0, 1170.0, 1920.0, 0.37)
    target = torch.tensor([0.0, 0.0, radius], dtype=torch.float64)
    P = torch.zeros(V, 2, 4, 4, dtype=torch.float64)
    for v in range(V):
        th = 1.2 * v / max(V - 1, 1) * (1 if v % 2 else -1) + (0.02 * u() if v else 0.0)
        C = radius * torch.tensor([math.sin(th), 0.03 * u() if v else 0.0, 1 - math.cos(th)], dtype=torch.float64)
        z = (target - C) / (target - C).norm()
        x = torch.linalg.cross(torch.tensor([0.02 * u(), 1.0, 0.0], dtype=torch.float64), z)
        x = x / x.norm()
        R = torch.stack([x, torch.linalg.cross(z, x), z])
        P[v, 0] = torch.eye(4, dtype=torch.float64)
        P[v, 0, :3, :3] = R
        P[v, 0, :3, 3] = -R @ C
        f = focal * W / width * (1 + 0.02 * u())
        P[v, 1, :3, :3] = torch.tensor([[f, skew, W / 2 + 3 * u()], [0.0, f * (1 + 1e-3 * u()), H / 2 + 3 * u()],
                                        [0.0, 0.0, 1.0]], dtype=torch.float64)
    return P.float()


def compose64(pm):
    """pm [V, 2, 4, 4] fp32 -> (homs [V-1, 12], kinv [9]) fp64: rotation (row-major) | translation of P_v P_0^-1 with
    P = E, P[:3, :4] = K E[:3, :4] (cost_volume.py:68-71, warping.py:80-82), and the inverse of camera 0's K"""
    p = pm.double()
    P = p[:, 0].clone()
    P[:, :3, :4] = p[:, 1, :3, :3] @ p[:, 0, :3, :4]
    M = P[1:] @ torch.inverse(P[0])
    return torch.cat([M[:, :3, :3].reshape(-1, 9), M[:, :3, 3]], 1), torch.inverse(p[0, 1, :3, :3]).reshape(9)


def homography64(src_proj, ref_proj):
    """src_proj, ref_proj [B, 4, 4] fp32 -> [B, 12] fp64 of src_proj @ inverse(ref_proj); NaN where ref_proj is singular"""
    out = torch.full((src_proj.shape[0], 12), float("nan"), dtype=torch.float64, device=src_proj.device)
    for b in range(src_proj.shape[0]):
        r = ref_proj[b].double()
        if torch.linalg.matrix_rank(r) == 4:
            M = src_proj[b].double() @ torch.inverse(r)
            out[b] = torch.cat([M[:3, :3].reshape(-1), M[:3, 3]])
    return out


def ulp_ratio(got, want, rows):
    """max over the entries of |got - want| / (one fp32 ulp of want + 1e-14 x the largest |want| of its row); rows is the
    number of entries per row.  <= 1 is the bar of a value computed in fp64 and rounded once to fp32."""
    want = want.double().reshape(-1, rows)
    got = got.double().reshape(-1, rows)
    m = want.abs().float()
    ulp = (torch.nextafter(m, torch.full_like(m, float("inf"))) - m).double()
    return float(((got - want).abs() / (ulp + 1e-14 * want.abs().amax(1, keepdim=True))).max())


# ------------------------------------------------------------------------------------------------ F5 / F6 scheduling
def init_inv64(dv, D):
    """dv [Dn] fp32 -> inverse hypotheses [D] fp64 of module.py:692-704: 1/dv[-1] + (1/dv[0] - 1/dv[-1]) k / (D - 1)"""
    d = dv.double()
    k = torch.arange(D, dtype=torch.float64, device=dv.device) / (D - 1)
    return 1 / d[-1] + (1 / d[0] - 1 / d[-1]) * k


def blend_axis(n_in, n_out, dtype=torch.float32, device="cpu"):
    """source indices i0, i1 and weights w0, w1 of the align_corners=True upsample n_in -> n_out along one axis.
    fp32: schedule_inverse_range_kernel's own (scale = __fdiv_rn(n_in - 1, n_out - 1), f = scale * i, i0 = (int)f,
    w1 = f - i0, w0 = 1 - w1, all fp32); fp64: the same in fp64 (oracle.hotpath.upsample2x_align_corners in fp64)."""
    if dtype == torch.float32:
        scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
        f = torch.arange(n_out, dtype=torch.float32, device=device) * torch.tensor(scale, device=device)
    else:
        f = torch.arange(n_out, dtype=dtype, device=device) * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    i0 = f.long().clamp(max=n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    w1 = f - i0.to(dtype)
    return i0, i1, (1 - w1).double(), w1.double()


def schedule_halfres64(depth, hypo, D, ratio):
    """depth [h, w], hypo [Dp, h, w] fp32 -> the half-resolution inverse hypotheses [D, h, w] fp64 of
    module.py:707-719 (split ratio rounded to fp32, the kernel's float argument)"""
    itv = 1 / hypo[2].double() - 1 / hypo[1].double()
    invd, s = 1 / depth.double(), f32(ratio) * itv
    k = torch.arange(D, dtype=torch.float64, device=depth.device).view(D, 1, 1) / (D - 1)
    return (invd - s)[None] + (2 * s)[None] * k


def schedule_inv64(depth, hypo, D, ratio, H, W, coords=torch.float32):
    """-> inverse hypotheses [D, H, W] fp64 of module.py:707-724: the half-resolution planes blended at the source
    coordinates of `blend_axis(coords)` (fp32: the kernel's; fp64: the oracle's in fp64)"""
    v = schedule_halfres64(depth, hypo, D, ratio)
    h, w = depth.shape
    y0, y1, wy0, wy1 = blend_axis(h, H, coords, depth.device)
    x0, x1, wx0, wx1 = blend_axis(w, W, coords, depth.device)
    top = v[:, y0][:, :, x0] * wx0 + v[:, y0][:, :, x1] * wx1
    bot = v[:, y1][:, :, x0] * wx0 + v[:, y1][:, :, x1] * wx1
    return top * wy0[:, None] + bot * wy1[:, None]


def inverse_error(out, want, tol):
    """out [D, H, W] fp32 planes, want [D, H, W] fp64 inverse hypotheses -> (max |1/out - want| / max|want|, the largest
    relative error of out itself where |want| >= 1e-2 max|want|, divided by its bound, and the count of such entries
    whose sign differs).  The bound on out is the inverse-space bar scaled by max|want| / |want|, plus one fp32
    rounding (tol is the inverse-space bar); near a zero crossing of want, 1/want is ill-conditioned and only the inverse-space bar applies."""
    scale = float(want.abs().max())
    e_inv = float((1 / out.double() - want).abs().max()) / scale
    far = want.abs() >= 1e-2 * scale
    o, v = out.double()[far], want[far]
    rel = (o * v - 1).abs()
    bound = tol * scale / v.abs() + 2.0 ** -23
    return e_inv, float((rel / bound).max()) if rel.numel() else 0.0, int((torch.sign(o) != torch.sign(v)).sum())


def cascade_inputs(full, wide, seed):
    """the inputs of a four-stage schedule on the depth range of `full` (or the wide range): (depth values [192] fp32, a
    function stage_depth(planes) -> the fp32 depth map that a stage with these planes hands the next one).  The depth map is one of
    the stage's own hypotheses per pixel, jittered by 1 %, as a soft-argmax of a peaked volume gives."""
    lo, hi = WIDE_RANGE if wide else (DTU_RANGE if full == DTU else TT_RANGE)
    g = torch.Generator().manual_seed(seed)

    def stage_depth(planes):
        D, h, w = planes.shape
        k = torch.randint(0, D, (1, h, w), generator=g).to(planes.device)
        j = (1 + 0.01 * (2 * torch.rand(h, w, generator=g) - 1)).to(planes.device)
        return (planes.gather(0, k)[0] * j).contiguous()

    return depth_values(lo, hi), stage_depth


def wide_planes(H, W, D=16, seed=0):
    """stage-2 planes [D, H, W] fp32 of the wide depth range 0.5 ... 50 (oracle, fp32): the stage-1 hypotheses are
    uniform in inverse depth with 1/dmin - 1/dmax = 1.98, so 1/depth - 2.67 x itv < 0 wherever the depth exceeds ~ 6"""
    dv, stage_depth = cascade_inputs(DTU, True, seed)
    prev = O.init_inverse_range(dv[None], NDEPTHS[0], H // 2, W // 2)[0]
    depth = stage_depth(prev)
    return O.schedule_inverse_range(depth[None], prev[None], D, RATIOS[1], H, W)[0].contiguous()


def narrow_planes(D, H, W, lo=DTU_RANGE[0], hi=DTU_RANGE[1], seed=0):
    """per-pixel planes [D, H, W] fp32 in [lo, hi] (oracle, fp32): scheduled from a stage at half size where H and W
    are even, else the first stage's planes jittered per pixel by 1 %"""
    g = torch.Generator().manual_seed(seed)
    dv = depth_values(lo, hi)
    if H % 2 or W % 2:
        return (O.init_inverse_range(dv[None], D, H, W)[0] * (1 + 0.01 * torch.rand(D, H, W, generator=g))).contiguous()
    prev = O.init_inverse_range(dv[None], NDEPTHS[0], H // 2, W // 2)[0]
    depth = prev.gather(0, torch.randint(0, NDEPTHS[0], (1, H // 2, W // 2), generator=g))[0]
    return O.schedule_inverse_range(depth[None], prev[None], D, 2.67, H, W)[0].contiguous()


# ------------------------------------------------------------------------------------------------ F7 3-D positions
def rays(kinv, H, W):
    """kinv [9] -> ax, ay, az [H*W] of the pixel rays K^-1 (x, y, 1).  fp32 kinv: pos3d_minmax_kernel's arithmetic,
    __fadd_rn(fmaf(k_r1, y, __fmul_rn(k_r0, x)), k_r2) with the fma in fp64 rounded once; fp64 kinv: plain fp64."""
    dt, dev = kinv.dtype, kinv.device
    y, x = torch.meshgrid(torch.arange(H, dtype=dt, device=dev), torch.arange(W, dtype=dt, device=dev), indexing="ij")
    x, y = x.reshape(-1), y.reshape(-1)
    out = []
    for r in range(3):
        k0, k1, k2 = kinv[3 * r], kinv[3 * r + 1], kinv[3 * r + 2]
        if dt == torch.float32:
            out.append((k1.double() * y.double() + (k0 * x).double()).float() + k2)
        else:
            out.append(k0 * x + k1 * y + k2)
    return out


def extents(kinvs, depths):
    """the x and y extents (wmin, wmax, hmin, hmax) of the 3-D positions over a batch: kinvs [B, 9], depths [B, D, H, W]
    (position_encoding.py:152-154).  fp32 inputs give the fp32 values pos3d_minmax_kernel reduces, so the result is
    what the kernel must decode bit for bit."""
    B, D, H, W = depths.shape
    px = torch.stack([rays(kinvs[b], H, W)[0] * depths[b].reshape(D, -1) for b in range(B)])
    py = torch.stack([rays(kinvs[b], H, W)[1] * depths[b].reshape(D, -1) for b in range(B)])
    return px.min(), px.max(), py.min(), py.max()


def extreme_owners(kinvs, depths, dvs):
    """{extent: (sample, flat sample index d * H * W + p)} of the smallest index holding each of the six extremes that
    mvsf_position3d reduces: x / y min and max of the positions and the depth-value min and max (dvs [B, Dn])"""
    B, D, H, W = depths.shape
    own = {}
    pxs = [rays(kinvs[b], H, W)[0] * depths[b].reshape(D, -1) for b in range(B)]
    pys = [rays(kinvs[b], H, W)[1] * depths[b].reshape(D, -1) for b in range(B)]
    for name, vals, pick in (("xmin", pxs, torch.min), ("xmax", pxs, torch.max), ("ymin", pys, torch.min),
                             ("ymax", pys, torch.max), ("dmin", list(dvs), torch.min), ("dmax", list(dvs), torch.max)):
        best = pick(torch.stack([pick(v) for v in vals]))
        b = next(i for i, v in enumerate(vals) if bool((v == best).any()))
        own[name] = (b, int((vals[b].reshape(-1) == best).nonzero()[0, 0]))
    return own


def minmax_trips(D, H, W, sms):
    """grid-stride trips of pos3d_minmax_kernel over D * H * W samples on `sms` SMs"""
    total = D * H * W
    grid = min(-(-total // POS3D_THREADS), POS3D_BLOCKS_PER_SM * sms)
    return -(-total // (grid * POS3D_THREADS)), grid * POS3D_THREADS


def positions64(kinv, depth, stats):
    """kinv [9] fp32, depth [D, H, W] fp32, stats = (wmin, wmax, hmin, hmax, dmin, dmax) -> normalised positions
    [3, D, H, W] fp64 of position_encoding.py:158-161"""
    D, H, W = depth.shape
    wmin, wmax, hmin, hmax, dmin, dmax = (float(s) for s in stats)
    ax, ay, az = rays(kinv.double(), H, W)
    d = depth.double().reshape(D, -1)
    px, py, pz = ax * d, ay * d, az * d
    return torch.stack([(px - wmin) / (wmax - wmin + 1e-5), (py - hmin) / (hmax - hmin + 1e-5),
                        (pz.clamp(dmin, dmax) - dmin) / (dmax - dmin + 1e-5)]).reshape(3, D, H, W)


def position_case(B, H, W, D, kind, wide, seed):
    """(projection matrices [B, V = 2, 2, 4, 4] fp32, hypotheses [B, D, H, W] fp32, depth values [B, 192] fp32, owners):
    each sample has its own cameras, depth range and hypotheses, and each of the six extremes comes from the sample
    `owners` names.  The x and y extremes are spikes of 3x the batch's largest |hypothesis| in the last plane (the last
    grid-stride trip at the shipped stage-1 sizes): x extremes at the left / right edge of a middle row, y extremes at
    the top / bottom of a middle column, where the other coordinate of the ray is near 0.  Every spike lies above the
    depth range, and 1 % of the hypotheses are halved, below it, so that the z clamp acts at both ends.  wide: the
    hypotheses are the wide-range stage-2 planes, with negative and huge entries."""
    g = torch.Generator().manual_seed(seed)
    owners = dict(xmin=B - 1, xmax=0, ymin=1 % B, ymax=B - 1, dmin=B - 1, dmax=1 % B)
    lo, hi = WIDE_RANGE if wide else (DTU_RANGE if kind == "dtu" else TT_RANGE)
    pm = torch.stack([ring_cameras(2, H * 8, W * 8, kind, seed=seed + b) for b in range(B)])
    pm[:, :, 1, :2] /= 8   # stage-1 intrinsics
    dvs, hyps = [], []
    for b in range(B):
        dvs.append(depth_values(lo * (0.9 if b == owners["dmin"] else 1.0), hi * (1.1 if b == owners["dmax"] else 1.0)))
        if wide:
            hyps.append(wide_planes(H, W, D, seed=seed + b))
        else:
            hyps.append(narrow_planes(D, H, W, float(dvs[b][0]), float(dvs[b][-1]), seed=seed + b))
    hyp = torch.stack(hyps)
    low = torch.rand(hyp.shape, generator=g) < 0.01
    hyp = torch.where(low, hyp * 0.5, hyp)
    big = 3 * float(hyp.abs().max())
    K = pm[:, 0, 1, :3, :3].double()
    cx, cy = [int(round(float(K[b, 0, 2]))) for b in range(B)], [int(round(float(K[b, 1, 2]))) for b in range(B)]
    for name, (x, y) in (("xmin", (0, None)), ("xmax", (W - 1, None)), ("ymin", (None, 0)), ("ymax", (None, H - 1))):
        b = owners[name]
        hyp[b, D - 1, cy[b] if y is None else y, cx[b] if x is None else x] = big
    return pm, hyp.contiguous(), torch.stack(dvs), owners


# ------------------------------------------------------------------------------------------------ S1 soft-argmax
def softargmax_logits(D, H, W, seed):
    """[D, H, W] fp32 logits, one kind per pixel p (p % 4): 0 = 10 randn; 1 = peaked (one logit 30 above the others);
    2 = flat (all equal, so prob and conf are exactly 1/D); 3 = ties (two logits share the maximum).  Returns the logits
    and the flat mask [H, W]."""
    g = torch.Generator().manual_seed(seed)
    z = 10 * torch.randn(D, H * W, generator=g)
    kind = torch.arange(H * W) % 4
    pk = torch.randint(0, D, (H * W,), generator=g)
    cols = torch.arange(H * W)
    peak = kind == 1
    z[pk[peak], cols[peak]] = z[:, peak].max(0).values + 30
    flat = kind == 2
    z[:, flat] = 10 * torch.randn(1, int(flat.sum()), generator=g)
    tie = kind == 3
    if D >= 2:
        p2 = (pk + 1 + torch.randint(0, D - 1, (H * W,), generator=g)) % D
        top = z[:, tie].max(0).values + 5
        z[pk[tie], cols[tie]] = top
        z[p2[tie], cols[tie]] = top
    return z.view(D, H, W).contiguous(), flat.view(H, W)


def softargmax64(logits, hypo, tmp):
    """-> prob [D, H, W], conf [H, W], depth [H, W] and the depth's scale sum_d w_d |hypo_d| [H, W], all fp64, of
    cost_volume.py:105-117 / module.py:649-655"""
    p = torch.softmax(logits.double(), 0)
    w = torch.softmax((logits * f32(tmp)).double(), 0)
    h = hypo.double()
    return p, p.max(0).values, (w * h).sum(0), (w * h.abs()).sum(0)


# ------------------------------------------------------------------------------------------------ S2 confidence
def nearest_index(n_in, n_out, device="cpu"):
    """source index of each output index of F.interpolate(mode="nearest"): min(floor(i * (float)(n_in / n_out)),
    n_in - 1) in fp32, as ATen's nearest_idx and conf_accumulate_kernel compute it"""
    scale = torch.tensor(np.float32(n_in) / np.float32(n_out), device=device)
    return (torch.arange(n_out, dtype=torch.float32, device=device) * scale).floor().long().clamp(max=n_in - 1)


def nearest_upsample(conf, H, W):
    """conf [h, w] -> [H, W] by the restated source indices"""
    h, w = conf.shape
    return conf[nearest_index(h, H, conf.device)][:, nearest_index(w, W, conf.device)]


def confidence_average(confs, H, W):
    """sum over the stages, in stage order, of F.interpolate(conf_s, (H, W), mode="nearest") x 0.25
    (DINOv2_mvsformer_model.py:167-177: prob_maps += conf, then / 4; scaling each term by 0.25 is exact)"""
    acc = None
    for c in confs:
        u = c if tuple(c.shape) == (H, W) else F.interpolate(c[None, None], (H, W), mode="nearest")[0, 0]
        acc = u * 0.25 if acc is None else acc + u * 0.25
    return acc


# ------------------------------------------------------------------------------------------------ bars
# Each about 3x the worst error measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit) over every case of
# tests/test_gpu_geometry_fp64.py.  The homographies and kinv are held to one fp32 ulp plus 1e-14 of their row instead:
# they are rounded once from fp64, and the worst measured is 0.4993 of that bound.
INIT_TOL = 4e-7       # the first stage's inverse hypotheses, |1/out - v| / max|v|; measured 1.3e-7
INV_TOL = 9e-7        # the schedule in inverse space; measured 3.0e-7 (T&T stage 3, wide range)
POS_TOL = 4e-7        # normalised positions, absolute; measured 1.3e-7


def prob_tol(D):
    """soft-argmax probability and confidence, absolute: measured 4.4e-7 up to D = 32, 6.9e-7 at D = 96"""
    return 1e-6 if D <= 32 else 2e-6


def depth_tol(D):
    """soft-argmax depth, relative to sum_d w_d |hypo_d|: measured 4.3e-7 up to D = 32, 6.3e-7 at D = 96"""
    return 1e-6 if D <= 32 else 2e-6
