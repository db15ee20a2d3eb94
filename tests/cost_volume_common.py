"""fp64 reference of the cost volume (W2-W4: homography warp, group correlation, entropy, visibility CNN, view
aggregation) at the library's own sample coordinates.

The homographies are the 12 floats per source view that mvsf_compose_geometry wrote (read back), so their rounding is
out of every comparison.  The sample coordinates restate warp_geom.cuh (ref_ray + warp_coord) in torch fp32, one torch op
per rounded device op, in the same order; everything after them (bilinear samples, correlations, softmax, entropy, vis
CNN, aggregation) runs in fp64.  What is left between a kernel and this reference is the kernel's own fp32 arithmetic.

Also here: the selection kernel's window-miss count (warp_tile.cu warp_stream_select_kernel) restated on the host, and
the launch constants the loop-coverage assertions depend on."""
import math

import torch

from oracle import hotpath as O

G = 8   # groups of the cost volume (the spill and window kernels exist for G == 8 only)

# ---- launch constants mirrored from the kernels
TW, PS_TROWS = 32, 8              # warp_tile.cu:32 (TW) and :426 (PsCfg::TROWS): the pipeline kernel's 8 x 32 pixel tile
PS_BLOCKS, PS_NBUF = 2, 3         # warp_tile.cu:38 kPsBlocks (CTAs per SM, grid = min(tiles, 2 * SMs)), kPsNbuf (ring)
PS_NSAMPLE = 96                   # warp_tile.cu:703 selection CTAs: min(tiles, 96) sample tiles
WX, WY = 64, 16                   # warp_tile.cu:45 Cfg::WX, Cfg::WY: the staged window (source texels)
STRIDED_CAP_PER_SM = 16           # warp_corr.cu:348 the strided L1 kernel's grid cap, 16 * SMs CTAs
L1_PIX_PER_CTA = 8 * 16           # warp_corr.cu:47,126: 8 warps x P = 32 / (C / 4) = 16 pixels per warp at C = 8
MAX_MISS_PERMILLE = 60            # warp_corr.cu:391 kMaxMissPermille


# ---- bars against this reference: |kernel - fp64| <= TOL * max(1, max|fp64|), entropy absolute.  Each is about 3x the
# worst error measured on an H100 SXM (132 SMs, 700 W) over every case of test_cost_volume_kernels, test_vis_cnn_tile_borders,
# test_identity_homography_property and tests/test_gpu_cost_volume_fp64.py.  Storing the spilled correlations in fp16
# costs >= 3.0e-4 on corr (pipeline and strided kernels, full size); a CTA of the pipeline kernel dropping its last
# partial tile, or the strided kernel skipping its last trip, leaves NaN in the outputs
ENT_TOL = 1e-5         # measured 3.4e-6: window kernel, generic D = 96 (96 expf / logf terms summed in fp32)
CORR_TOL = 5e-7        # measured 1.7e-7
VOL_TOL = 6e-7         # measured 2.1e-7
VIS_TOL = 2e-6         # vis CNN on the kernel's own entropy; measured 6.7e-7
VIS_CHAIN_TOL = 2e-6   # vis of the chain (entropy error included) against the vis CNN of the fp64 entropy; measured 6.6e-7
WARP_TOL = 4e-7        # mvsf_homo_warp samples; measured 1.2e-7


def pipeline_coverage(H, W, V, sms):
    """tiles per CTA (fewest, most) and ring turns per tile of warp_stream_entropy_store_kernel on `sms` SMs"""
    ntiles = -(-W // TW) * -(-H // PS_TROWS)
    grid = min(ntiles, PS_BLOCKS * sms)
    return ntiles // grid, -(-ntiles // grid), (V - 1) / PS_NBUF


def strided_trips(H, W, sms):
    """trips per CTA (fewest, most) of the strided L1 kernel warp_corr_entropy_kernel<8, false, 1, true>"""
    blocks = -(-H * W // L1_PIX_PER_CTA)
    grid = min(blocks, STRIDED_CAP_PER_SM * sms)
    return blocks // grid, -(-blocks // grid)


# ---- coordinates
def restated_coords(homs, depth):
    """homs [V-1, 12] fp32 (rotation row-major, translation); depth [D, H, W] fp32 -> ix, iy, Z [V-1, D, H*W] fp32, the
    values of warp_geom.cuh ref_ray + warp_coord.  Every divisor is a full tensor: torch turns a division by a scalar
    into a multiplication by its reciprocal, which is not the device's IEEE quotient."""
    dev = depth.device
    D, H, W = depth.shape
    h = homs.reshape(-1, 12).to(dev, torch.float32)
    y, x = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32),
                          indexing="ij")
    fx, fy = x.reshape(1, -1), y.reshape(1, -1)

    def ray(i):   # __fadd_rn(fmaf(r_i1, fy, __fmul_rn(r_i0, fx)), r_i2); the fma in fp64 (the product is exact), rounded once
        m = h[:, 3 * i, None] * fx
        f = (h[:, 3 * i + 1, None].double() * fy.double() + m.double()).float()
        return f + h[:, 3 * i + 2, None]

    d = depth.reshape(1, D, H * W)
    X = ray(0)[:, None] * d + h[:, 9, None, None]
    Y = ray(1)[:, None] * d + h[:, 10, None, None]
    Z = ray(2)[:, None] * d + h[:, 11, None, None]
    Zs = Z + torch.tensor(1e-6, dtype=torch.float32, device=dev)
    px, py = X / Zs, Y / Zs
    gx = px / torch.full_like(px, (W - 1) * 0.5) - 1.0
    gy = py / torch.full_like(py, (H - 1) * 0.5) - 1.0
    ix = ((gx + 1.0) * 0.5) * float(W - 1)
    iy = ((gy + 1.0) * 0.5) * float(H - 1)
    return ix, iy, Z


def in_bounds(ix, iy, H, W):
    """make_tap's rule: a sample inside (-1, W) x (-1, H) has at least one corner in the image (false for NaN / Inf)"""
    return (ix > -1) & (ix < W) & (iy > -1) & (iy < H)


def sample(src, ix, iy, H, W):
    """bilinear sample of src [H*W, C] (fp64) at fp32 (ix, iy) [N] -> [N, C] fp64, zero padding per corner"""
    inb = in_bounds(ix, iy, H, W)
    sx = torch.where(inb, ix, torch.zeros_like(ix)).double()
    sy = torch.where(inb, iy, torch.zeros_like(iy)).double()
    x0, y0 = torch.floor(sx), torch.floor(sy)
    wx1, wy1 = sx - x0, sy - y0
    out = torch.zeros(ix.shape[0], src.shape[1], dtype=torch.float64, device=src.device)
    for dx, dy, w in ((0, 0, (1 - wx1) * (1 - wy1)), (1, 0, wx1 * (1 - wy1)), (0, 1, (1 - wx1) * wy1), (1, 1, wx1 * wy1)):
        xi, yi = x0 + dx, y0 + dy
        ok = inb & (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        out += src[idx] * torch.where(ok, w, torch.zeros_like(w))[:, None]
    return out


class CostVolumeRef:
    """feat [V, H, W, C] fp32 channels-last (view 0 = reference), homs [V-1, 12] fp32, depth [D, H, W] fp32, all on the
    device the reference runs on.  Views are evaluated one at a time (hypothesis by hypothesis) so that full-size cases
    stay within a few GB."""

    def __init__(self, feat, homs, depth):
        self.V, self.H, self.W, self.C = feat.shape
        self.D = depth.shape[0]
        self.feat = feat.reshape(self.V, -1, self.C)
        self.ix, self.iy, self.Z = restated_coords(homs, depth)

    def view(self, v):
        """-> corr [D, H*W, 8] fp64 (mean over the C/8 channels of each group of ref * warped) and entropy [H*W] fp64 of
        source view v (0-based over the source views)"""
        ref = self.feat[0].double()
        src = self.feat[v + 1].double()
        corr = torch.empty(self.D, ref.shape[0], G, dtype=torch.float64, device=ref.device)
        for d in range(self.D):
            s = sample(src, self.ix[v, d], self.iy[v, d], self.H, self.W)
            corr[d] = (ref * s).view(-1, G, self.C // G).mean(-1)
        p = torch.softmax(corr.sum(-1), 0)
        return corr, -(p * torch.log(p + 1e-7)).sum(0)

    def pass_a(self):
        """-> corr [V-1, D, H*W, 8], entropy [V-1, H*W] (fp64)"""
        out = [self.view(v) for v in range(self.V - 1)]
        return torch.stack([c for c, _ in out]), torch.stack([e for _, e in out])


def vis_fp64(entropy, sd64, prefix):
    """oracle vis CNN on an fp64 state dict: entropy [N, H, W] -> [N, H, W] fp64"""
    e = entropy.double()
    return torch.cat([O.vis_cnn(e[None, i:i + 1], sd64, prefix) for i in range(e.shape[0])], 1)[0]


def aggregate(corr, vis):
    """volume [D, H*W, 8] = sum_v w_v corr_v / (sum_v w_v + 1e-6); corr [V-1, D, H*W, 8], vis [V-1, H*W] (fp64)"""
    w = vis.double().reshape(vis.shape[0], 1, -1, 1)
    return (corr * w).sum(0) / (w.sum(0) + 1e-6)


def state_dict_fp64(sd, device):
    return {k: v.to(device, torch.float64) for k, v in O.state_dict_to(sd, torch.float64).items()}


def compose_homs_fp64(pm):
    """pm [V, 2, 4, 4] -> [V-1, 12] fp32: P_src * P_ref^-1 composed in fp64 and rounded once (as mvsf_compose_geometry)"""
    P = [O.compose_projection(pm[None, v].double())[0].double() for v in range(pm.shape[0])]
    inv = torch.inverse(P[0])
    return torch.stack([torch.cat([(P[v] @ inv)[:3, :3].reshape(-1), (P[v] @ inv)[:3, 3]]) for v in range(1, len(P))]).float()



def seam_hom(src_proj, ref_proj):
    """12 floats of src_proj @ ref_proj^-1 for already composed 4 x 4 projections (the warp seam's arguments), fp64, rounded once"""
    M = src_proj.double() @ torch.inverse(ref_proj.double())
    return torch.cat([M[:3, :3].reshape(-1), M[:3, 3]]).float()

# ---- the selection kernel's count (warp_tile.cu:437-455, 174-186, 587-627)
def selector_restated(ref):
    """-> (miss per mille, decision, sampled in-bound taps, misses) that warp_stream_select_kernel computes for the call
    whose restated coordinates `ref` (a CostVolumeRef) holds"""
    H, W, D = ref.H, ref.W, ref.D
    dev = ref.ix.device
    tiles_x, ntiles = -(-W // TW), -(-W // TW) * -(-H // PS_TROWS)
    nsample = min(ntiles, PS_NSAMPLE)
    tile = torch.arange(nsample, device=dev) * ntiles // nsample                   # sample tile of CTA b
    lane = torch.arange(32, device=dev)
    sr, sc = (lane >> 3) * 2 + 1, (lane & 7) * 4 + 1                              # sample_pixel: 4 rows x 8 columns
    x = torch.clamp((tile % tiles_x)[:, None] * TW + sc, max=W - 1)
    y = torch.clamp((tile // tiles_x)[:, None] * PS_TROWS + sr, max=H - 1)
    p = (y * W + x).reshape(-1)
    tot = miss = 0
    big = 1 << 30
    for v in range(ref.V - 1):
        ix, iy = ref.ix[v][:, p].view(D, nsample, 32), ref.iy[v][:, p].view(D, nsample, 32)
        inb = in_bounds(ix, iy, H, W)
        x0 = torch.floor(torch.where(inb, ix, torch.zeros_like(ix))).long()
        y0 = torch.floor(torch.where(inb, iy, torch.zeros_like(iy))).long()
        e = torch.tensor([0, D - 1], device=dev)   # predict_window: first and last hypothesis
        bi, bx, by = inb[e], x0[e], y0[e]
        bx0 = torch.where(bi, bx, big).amin((0, 2))
        bx1 = torch.where(bi, bx, -big).amax((0, 2))
        by0 = torch.where(bi, by, big).amin((0, 2))
        by1 = torch.where(bi, by, -big).amax((0, 2))
        empty = bx0 > bx1
        slack_x, slack_y = WX - (bx1 + 2 - bx0), WY - (by1 + 2 - by0)
        ox = torch.where(empty, 0, bx0 - torch.where(slack_x > 0, slack_x // 2, 0))   # window_origin
        oy = torch.where(empty, 0, (by0 - torch.where(slack_y > 0, slack_y // 2, 0)) & ~1)
        lx, ly = x0 - ox[None, :, None], y0 - oy[None, :, None]
        inwin = (lx >= 0) & (lx <= WX - 2) & (ly >= 0) & (ly <= WY - 2)           # in_window
        tot += int(inb.sum())
        miss += int((inb & ~inwin).sum())
    permille = miss * 1000 // tot if tot else 0
    return permille, int(permille <= MAX_MISS_PERMILLE), tot, miss


# ---- geometry of the grazing case
def grazing_projections(H, W):
    """[3, 2, 4, 4] projection matrices (identity reference camera, unit intrinsics, so that mvsf_compose_geometry returns
    the source extrinsics exactly).  Source view 1: a camera turned ~70 degrees whose principal plane cuts through the
    hypothesis range, so that taps behind it (Z <= 0) land in the image.  Source view 2: its principal plane holds the
    reference rays of column W // 2 (Z = -1e-6 exactly there, so Z + 1e-6 = 0): those taps go to +-Inf, or NaN where the
    numerator is 0 too (row H // 2)."""
    pm = torch.zeros(3, 2, 4, 4, dtype=torch.float64)
    for v in range(3):
        pm[v, 0] = torch.eye(4, dtype=torch.float64)
        pm[v, 1, :3, :3] = torch.eye(3, dtype=torch.float64)
    th = 1.2
    c, s = math.cos(th), math.sin(th)
    pm[1, 0, :3, :4] = torch.tensor([[c, 0.0, -s, -20.0], [0.0, 1.0, 0.0, -10.0], [s, 0.0, c, -40.0]], dtype=torch.float64)
    c2, r2 = float(W // 2), float(H // 2)
    pm[2, 0, :3, :4] = torch.tensor([[0.0, 1.0, -r2, 0.0], [0.25, 0.5, 1.0, 2.0], [1.0, 0.0, -c2, float(torch.tensor(-1e-6).float())]],
                                    dtype=torch.float64)
    return pm.float()


def grazing_depth(D, H, W, seed):
    """per-pixel hypotheses spread over [0.5, 2.5] (in the reference camera's unit-focal coordinates)"""
    g = torch.Generator().manual_seed(seed)
    base = 0.5 + 2.0 * torch.arange(D, dtype=torch.float32).view(D, 1, 1) / max(D - 1, 1)
    return (base * (1.0 + 0.05 * torch.rand(D, H, W, generator=g))).contiguous()
