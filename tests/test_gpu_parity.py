"""GPU parity tests: every libmvsf_b200 entry point (called through the ctypes C ABI / the host seam mirrors) against
the CPU oracle on the same seeded inputs, and against the reference-executed golden fixtures.
Tolerances: north-star 1e-3 relative L-inf on depth, 1e-4 absolute on per-pixel probability; intermediates tighter.
A JSON report with every measured error is written to parity_report.json in tests.common.REPORT_DIR."""
import ctypes
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import _lib
from tests import conv3d_common as C3
from tests import cost_volume_common as R
from tests.common import ROOT, TMP, build_case, load_golden, max_abs, rec, rel_linf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def hp():
    from mvsformerplusplus_b200 import hotpath
    return hotpath


# ----------------------------------------------------------------------------------------------- boundary helpers
def test_layout_roundtrip(dev, hp):
    x = torch.randn(3, 24, 13, 37, device=dev)
    n = hp.to_nhwc(x)
    assert torch.equal(n, x.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(hp.to_nchw(n), x)
    assert hp.to_nhwc(n.permute(0, 3, 1, 2)).data_ptr() == n.data_ptr()  # channels-last view: zero copy


def test_compose_geometry(dev):
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    pm = synth.make_proj_matrices(5, 1152, 1536)["stage3"][0]
    homs = torch.empty(4 * 12, device=dev)
    kinv = torch.empty(9, device=dev)
    pmd = pm.to(dev)
    _lib.call("mvsf_compose_geometry", pmd, 5, homs, kinv)
    pm64 = pm.double()
    ref = O.compose_projection(pm64[None, 0])[0]
    want = []
    for v in range(1, 5):
        M = O.compose_projection(pm64[None, v])[0] @ torch.inverse(ref)
        want.append(torch.cat([M[:3, :3].reshape(-1), M[:3, 3]]))
    want = torch.stack(want).reshape(-1)
    err = float(((homs.cpu().double() - want).abs() / want.abs().clamp_min(1e-3)).max())
    kerr = max_abs(kinv.cpu(), torch.inverse(pm64[0, 1, :3, :3]).reshape(-1))
    rec("compose_geometry", rel=err, kinv_abs=kerr)
    assert err < 1e-6 and kerr < 1e-7


def test_homo_warp_seam_vs_reference(dev):
    g, _ = load_golden("warp_seam")
    from oracle import hotpath as O
    src = g["src"][0]
    C, H, W = src.shape
    D = g["depth_values"].shape[1]
    M = (g["src_proj"].double() @ torch.inverse(g["ref_proj"].double()))[0]
    hom = torch.cat([M[:3, :3].reshape(-1), M[:3, 3]]).float().to(dev)
    src_nhwc = src.permute(1, 2, 0).contiguous().to(dev)
    warped = torch.empty(C, D, H, W, device=dev)
    mask = torch.empty(D, H, W, dtype=torch.uint8, device=dev)
    dvd = g["depth_values"][0].contiguous().to(dev)
    _lib.call("mvsf_homo_warp", src_nhwc, hom, dvd, warped, mask, C, D, H, W)
    e = max_abs(warped.cpu(), g["warped"][0])
    mm = float((mask.cpu().bool() != g["mask"][0]).float().mean())
    rec("homo_warp_seam", abs=e, mask_mismatch=mm)
    assert e < 2e-4 and mm < 0.01


# ----------------------------------------------------------------------------------------------- scheduling
def test_init_and_schedule_inverse_range(dev):
    from oracle import hotpath as O
    dv = (425.0 + 2.65 * torch.arange(192)).float()
    D, H, W = 32, 12, 20
    out = torch.empty(D, H, W, device=dev)
    dvd = dv.to(dev)  # keep device inputs alive until the (asynchronous) kernels have consumed them
    _lib.call("mvsf_init_inverse_range", dvd, 192, out, D, H, W)
    want = O.init_inverse_range(dv[None], D, H, W)[0]
    e0 = rel_linf(out.cpu(), want)
    g = torch.Generator().manual_seed(1)
    depth = 500.0 + 300.0 * torch.rand(1, H, W, generator=g)
    hyp = want[None] * (1.0 + 0.01 * torch.rand(1, D, H, W, generator=g))
    D2, H2, W2 = 16, 2 * H, 2 * W
    out2 = torch.empty(D2, H2, W2, device=dev)
    depth_d, hyp_d = depth[0].contiguous().to(dev), hyp[0].contiguous().to(dev)
    _lib.call("mvsf_schedule_inverse_range", depth_d, hyp_d, D, 2.67, out2, D2, H2, W2)
    want2 = O.schedule_inverse_range(depth, hyp, D2, 2.67, H2, W2)[0]
    e1 = rel_linf(out2.cpu(), want2)
    rec("inverse_range", init_rel=e0, schedule_rel=e1)
    assert e0 < 1e-6 and e1 < 2e-6


def test_position3d(dev):
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    H, W, D = 12, 16, 8
    pm = synth.make_proj_matrices(3, H * 8, W * 8)["stage1"]
    dv = synth.make_depth_values(192)
    ds = O.init_inverse_range(dv, D, H, W)
    want, hmin, hmax, wmin, wmax = O.get_position_3d(1, H, W, pm[:, 0, 1, :3, :3], ds, dv.min(), dv.max(), None, None, None, None)
    homs = torch.empty(2 * 12, device=dev)
    kinv = torch.empty(9, device=dev)
    pmd, dsd, dvd = pm[0].to(dev), ds[0].contiguous().to(dev), dv[0].to(dev)
    _lib.call("mvsf_compose_geometry", pmd, 3, homs, kinv)
    stats = torch.zeros(8, device=dev)
    pos = torch.empty(3, D, H, W, device=dev)
    _lib.call("mvsf_position3d", kinv, dsd, dvd, 192, stats, 1, pos, D, H, W)
    e = max_abs(pos.cpu(), want[0])
    se = max_abs(stats[:4].cpu(), torch.stack([wmin, wmax, hmin, hmax]))
    rec("position3d", abs=e, stats_abs=se)
    assert e < 2e-6


# ----------------------------------------------------------------------------------------------- cost volume
def _rand_vis_sd(seed):
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    torch.manual_seed(0)
    params = build_hotpath_params(default_args()).eval()
    return synth.randomize_state_dict(params, seed=seed)


COST_CASES = [  # C, D, H, W, V, theta_step, depth jitter
    (8, 4, 37, 53, 3, 0.1, 0.02), (16, 8, 24, 40, 3, 0.1, 0.02), (32, 16, 16, 24, 4, 0.12, 0.02), (64, 32, 12, 16, 5, 0.1, 0.02),
    (8, 4, 31, 45, 3, 0.6, 0.02),   # wide baseline: many taps leave the image (zero padding per corner)
    (8, 48, 10, 14, 3, 0.1, 0.02),  # generic-D path (D-sweep configuration)
    (64, 8, 9, 11, 2, 0.1, 0.02),
    (32, 16, 20, 28, 4, 0.6, 0.3), (64, 32, 14, 18, 4, 0.6, 0.3),   # wide baseline and depth jitter at the coarse stages
    # shapes served by the TMA-staged window kernels (C = 8 / 16, even H): several tiles, ragged right / bottom edges,
    # taps leaving the image, depth outliers that leave the staged window (global fallback), D = 4 / 8 / chunked D
    (8, 4, 64, 96, 3, 0.1, 0.02), (8, 4, 30, 44, 5, 0.6, 0.02), (8, 4, 48, 80, 3, 0.15, 0.4), (8, 8, 16, 40, 3, 0.1, 0.02),
    (8, 7, 18, 34, 2, 0.1, 0.02), (16, 8, 32, 48, 4, 0.1, 0.02), (16, 8, 28, 68, 3, 0.5, 0.3), (16, 4, 12, 20, 3, 0.1, 0.02),
    (16, 24, 10, 36, 3, 0.1, 0.02), (8, 96, 12, 20, 3, 0.1, 0.0),
    # grazing geometry (cost_volume_common.grazing_projections): taps behind a source camera land in the image, taps on
    # its principal plane go to +-Inf / NaN
    (8, 4, 36, 52, 3, "grazing", 0.0), (16, 8, 36, 52, 3, "grazing", 0.0),
]


@pytest.mark.parametrize("C,D,H,W,V,th,jit", COST_CASES)
def test_cost_volume_kernels(dev, C, D, H, W, V, th, jit):
    """Pass A (entropy, spilled correlations), vis CNN and pass B (aggregation) of every organisation the library has
    (L1 gathers with recompute, L1 gathers with the correlation spill and, where they apply, the window kernels and the
    pipeline kernel, forced and chosen per call) against the fp64 reference at the library's own sample coordinates
    (tests/cost_volume_common.py), and against each other.  The fp32 oracle's errors are recorded only: they are sized by
    its own coordinate rounding."""
    from mvsformerplusplus_b200 import packing, synth
    from oracle import hotpath as O
    sd = _rand_vis_sd(5)
    g = torch.Generator().manual_seed(C * 1000 + D)
    feats = torch.randn(1, V, C, H, W, generator=g)
    if th == "grazing":
        pm = R.grazing_projections(H, W)[None]
        dvals = R.grazing_depth(D, H, W, seed=C + D)[None]
    else:
        sc = {8: 1, 16: 2, 32: 4, 64: 8}[C]
        pm = synth.make_proj_matrices(V, H * sc, W * sc, theta_step=th)[f"stage{ {1: 4, 2: 3, 4: 2, 8: 1}[sc] }"]
        dv = synth.make_depth_values(192)
        dvals = O.init_inverse_range(dv, D, H, W) * (1.0 + jit * torch.rand(1, D, H, W, generator=g))
    want = O.cost_volume(feats, pm, dvals, sd, "fusions.3.", 8)
    homs = torch.empty((V - 1) * 12, device=dev)
    kinv = torch.empty(9, device=dev)
    pmd = pm[0].to(dev)
    _lib.call("mvsf_compose_geometry", pmd, V, homs, kinv)
    f = feats[0].permute(0, 2, 3, 1).contiguous().to(dev)
    dd = dvals[0].contiguous().to(dev)
    wts = packing.pack_vis(sd, "fusions.3.vis.").to(dev)
    vol_scale = max(1.0, float(want["volume_mean"].abs().max()))

    # fp64 reference at the library's coordinates
    ref = R.CostVolumeRef(f, homs.view(V - 1, 12), dd)
    corr64, ent64 = ref.pass_a()
    sd64 = R.state_dict_fp64(sd, dev)
    vis64 = R.vis_fp64(ent64.view(V - 1, H, W), sd64, "fusions.3.")
    corr_scale = max(1.0, float(corr64.abs().max()))
    if th == "grazing":   # both kinds of tap the geometry is there for
        finite = torch.isfinite(ref.ix) & torch.isfinite(ref.iy)
        behind_in_image = R.in_bounds(ref.ix, ref.iy, H, W) & (ref.Z <= 0)
        assert bool((~finite).any()) and bool(behind_in_image.any())
    e64 = {}

    def check64(tag, ent_k, vis_k, vol_k, corr_k=None):
        """one organisation's outputs against the reference; pass B fed the organisation's own vis"""
        vis_k = vis_k.reshape(V - 1, H * W)
        own = R.vis_fp64(ent_k, sd64, "fusions.3.").reshape(V - 1, H * W)
        vol64 = R.aggregate(corr64, vis_k)
        e = {f"{tag}_entropy64": max_abs(ent_k.reshape(V - 1, -1), ent64),
             f"{tag}_vis64": max_abs(vis_k, own), f"{tag}_vis64_chain": max_abs(vis_k, vis64.reshape(V - 1, -1)),
             f"{tag}_volume64": max_abs(vol_k.reshape(D, H * W, 8), vol64) / max(1.0, float(vol64.abs().max()))}
        if corr_k is not None:
            e[f"{tag}_corr64"] = max_abs(corr_k.reshape(V - 1, D, H * W, 8), corr64) / corr_scale
        e64.update(e)

    def run_two_gathers():
        ent = torch.empty(V - 1, H, W, device=dev)
        _lib.call("mvsf_warp_corr_entropy", f, homs, dd, ent, V, C, 8, D, H, W)
        vis = torch.empty(V - 1, H, W, device=dev)
        _lib.call("mvsf_vis_cnn", ent, wts, vis, V - 1, H, W)
        vol = torch.empty(D, H, W, 8, device=dev)
        _lib.call("mvsf_warp_corr_aggregate", f, homs, dd, vis, vol, V, C, 8, D, H, W)
        return ent, vis, vol

    _lib.call("mvsf_warp_corr_set_tile_path", 0)
    try:
        ent, vis, vol = run_two_gathers()
        # spill plan: pass A stores the per-view group correlations, the aggregation streams them
        ent_s = torch.empty(V - 1, H, W, device=dev)
        corr = torch.empty(V - 1, D, H, W, 8, device=dev)
        vol_s = torch.empty(D, H, W, 8, device=dev)
        _lib.call("mvsf_warp_corr_entropy_store", f, homs, dd, ent_s, corr, V, C, 8, D, H, W)
        _lib.call("mvsf_corr_aggregate", corr, vis, vol_s, V, 8, D, H, W)
    finally:
        _lib.call("mvsf_warp_corr_set_tile_path", 1)
    check64("l1", ent, vis, vol)
    check64("l1_spill", ent_s, vis, vol_s, corr)
    assert torch.equal(ent_s, ent)
    e_paths = max_abs(vol_s.cpu(), vol.cpu())
    assert e_paths <= 2e-6 * vol_scale, e_paths   # identical up to the pair sum of 8-channel groups
    assert _lib.lib().mvsf_warp_corr_plan(C, 8, D, H, W, V, 1 << 40) == 0      # room for the spill buffer: spill plan
    assert _lib.lib().mvsf_warp_corr_plan(C, 8, D, H, W, V, 1024) == 1         # no room: two gathers
    tiled = C in (8, 16) and H % 2 == 0    # shapes the window kernels serve
    e_tile = {}
    if tiled:   # window kernels: the two-gather plan ...
        ent_t, vis_t, vol_t = run_two_gathers()
        check64("tile", ent_t, vis_t, vol_t)
        e_tile = dict(tile_vs_l1_entropy=max_abs(ent_t.cpu(), ent.cpu()), tile_vs_l1_volume=max_abs(vol_t.cpu(), vol_s.cpu()))
        assert e_tile["tile_vs_l1_entropy"] < 2e-5 and e_tile["tile_vs_l1_volume"] < 1e-5 * vol_scale, e_tile
        # ... and the spill plan: forced through the persistent TMA pipeline kernel where it exists (C = 8, D = 4; mode 2,
        # other shapes run the L1 kernel), then as hotpath.py runs it (mode 1: at C = 8, D = 4 the device picks pipeline or
        # L1 kernel per call)
        for mode in (2, 1):
            _lib.call("mvsf_warp_corr_set_tile_path", mode)
            try:
                ent_p = torch.empty(V - 1, H, W, device=dev)
                corr_p = torch.full((V - 1, D, H, W, 8), float("nan"), device=dev)
                vol_p = torch.empty(D, H, W, 8, device=dev)
                _lib.call("mvsf_warp_corr_entropy_store", f, homs, dd, ent_p, corr_p, V, C, 8, D, H, W)
            finally:
                _lib.call("mvsf_warp_corr_set_tile_path", 1)
            vis_p = torch.empty(V - 1, H, W, device=dev)
            _lib.call("mvsf_vis_cnn", ent_p, wts, vis_p, V - 1, H, W)
            _lib.call("mvsf_corr_aggregate", corr_p, vis_p, vol_p, V, 8, D, H, W)
            tag = "pipe" if mode == 2 else "adaptive"
            check64(tag, ent_p, vis_p, vol_p, corr_p)
            e_tile.update({f"{tag}_vs_l1_entropy": max_abs(ent_p.cpu(), ent.cpu()), f"{tag}_vs_l1_corr": max_abs(corr_p.cpu(), corr.cpu()),
                           f"{tag}_vs_l1_volume": max_abs(vol_p.cpu(), vol_s.cpu())})
            assert bool(torch.isfinite(corr_p).all())
            assert e_tile[f"{tag}_vs_l1_entropy"] < 2e-5 and e_tile[f"{tag}_vs_l1_corr"] < 1e-5 * vol_scale * 8 and e_tile[f"{tag}_vs_l1_volume"] < 1e-5 * vol_scale, e_tile
            if mode == 1 and C == 8 and D == 4:
                used, miss = ctypes.c_int(-1), ctypes.c_int(-1)
                _lib.call("mvsf_warp_corr_last_selection", ctypes.byref(used), ctypes.byref(miss))
                e_tile.update(adaptive_used_pipeline=used.value, adaptive_window_miss_permille=miss.value)
                assert used.value in (0, 1) and 0 <= miss.value <= 1000
                assert used.value == (1 if miss.value <= 60 else 0)   # wide baseline (theta 0.6): 193 per mille -> L1 kernel
        ent, vis, vol_s = ent_p, vis_p, vol_p
    vol = vol_s
    e_ent = max_abs(ent.cpu(), want["entropy"][0])
    e_vis = max_abs(vis.cpu(), want["vis_weight"][0])
    e_vol = max_abs(vol.cpu().permute(3, 0, 1, 2), want["volume_mean"][0])
    # vis CNN in isolation on the oracle's entropy
    vis2 = torch.empty(V - 1, H, W, device=dev)
    ent_o = want["entropy"][0].contiguous().to(dev)
    _lib.call("mvsf_vis_cnn", ent_o, wts, vis2, V - 1, H, W)
    e_vis2 = max_abs(vis2.cpu(), want["vis_weight"][0])
    rec(f"cost_volume_C{C}_D{D}_{H}x{W}_V{V}_th{th}_j{jit}", entropy=e_ent, vis=e_vis, vis_isolated=e_vis2, volume=e_vol,
        vol_scale=float(want["volume_mean"].abs().max()), corr64_scale=corr_scale, tiled=int(tiled), **e_tile, **e64)
    for k, e in e64.items():
        kind = k.rsplit("_", 1)[1] if not k.endswith("_chain") else "chain"
        lim = {"entropy64": R.ENT_TOL, "vis64": R.VIS_TOL, "chain": R.VIS_CHAIN_TOL, "volume64": R.VOL_TOL, "corr64": R.CORR_TOL}[kind]
        assert e < lim, f"{k}: {e:.3e} against fp64, limit {lim:.1e}"


def test_vis_cnn_tile_borders(dev):
    """the fused vis CNN (wgmma on fp16 hi|lo operands) against the vis CNN in fp64, at sizes that cut its 14 x 30 tiles"""
    from mvsformerplusplus_b200 import packing
    sd = _rand_vis_sd(9)
    sd64 = R.state_dict_fp64(sd, "cpu")
    g = torch.Generator().manual_seed(3)
    for (N, H, W) in [(1, 30, 30), (2, 61, 95), (3, 7, 5), (1, 1, 1), (2, 64, 128)]:
        ent = 3.0 * torch.rand(N, H, W, generator=g)
        want = R.vis_fp64(ent, sd64, "fusions.1.")
        vis = torch.empty(N, H, W, device=dev)
        ent_d, wts = ent.contiguous().to(dev), packing.pack_vis(sd, "fusions.1.vis.").to(dev)
        _lib.call("mvsf_vis_cnn", ent_d, wts, vis, N, H, W)
        e = max_abs(vis.cpu(), want)
        rec(f"vis_cnn_{N}x{H}x{W}", abs=e)
        assert e < R.VIS_TOL, f"{e:.3e} against fp64"


# ----------------------------------------------------------------------------------------------- regularisers
@pytest.mark.parametrize("mode,sd,cin,cout,ID,IH,IW", [
    (0, 1, 16, 16, 3, 16, 32), (0, 1, 32, 32, 2, 20, 44), (0, 1, 64, 64, 4, 9, 13), (0, 1, 16, 16, 5, 48, 160),
    (0, 1, 16, 16, 9, 64, 1200), (0, 2, 32, 32, 11, 40, 72), (1, 1, 8, 16, 6, 96, 1300), (0, 1, 16, 16, 1, 16, 16),
    (1, 1, 8, 16, 3, 32, 64), (1, 2, 8, 16, 8, 24, 40), (1, 1, 16, 32, 2, 18, 26), (1, 2, 32, 64, 4, 16, 16),
    (2, 1, 64, 32, 2, 9, 12), (2, 2, 32, 16, 3, 16, 24), (2, 1, 16, 8, 3, 20, 36), (2, 2, 16, 8, 2, 8, 8)])
@pytest.mark.parametrize("skip", [False, True])
def test_conv3d_tensor_core_layer(dev, mode, sd, cin, cout, ID, IH, IW, skip):
    """One 3x3x3 layer of the wgmma implicit-GEMM path against torch's fp64 convolution (conv / strided conv /
    transposed conv with output_padding = stride - 1, bias, ReLU, skip added after the ReLU)."""
    e, scale = C3.layer_vs_fp64(dev, mode, sd, cin, cout, ID, IH, IW, skip, seed=mode * 100 + cin + ID)
    rec(f"conv3d_tc_mode{mode}_sd{sd}_{cin}to{cout}_{ID}x{IH}x{IW}_skip{int(skip)}", abs=e, scale=scale)
    assert e < C3.LAYER_TOL * max(1.0, scale)


@pytest.mark.parametrize("stage,D,H,W", [(1, 16, 16, 24), (1, 8, 8, 40), (2, 8, 16, 24), (3, 4, 24, 40), (3, 3, 8, 8)])
def test_costreg_unet_two_part(dev, stage, D, H, W):
    """Both parts of a U-Net (conv weights packed for the tensor cores, fp32 biases and `prob` conv) against the fp64
    oracle; stage 1 is CostRegNet, stages 2 and 3 CostRegNet3D"""
    e, scale = C3.unet_vs_fp64(dev, _rand_vis_sd(13), f"fusions.{stage}.cost_reg.", 0 if stage == 1 else 1, D, H, W,
                               seed=stage * 7 + D)
    rec(f"costreg_unet_stage{stage}_{D}x{H}x{W}", abs=e, scale=scale)
    assert e < C3.UNET_TOL * max(1.0, scale)


# |logits - fp64| <= COSTREG_TR_TOL * max(1, max|fp64|).  The attention's P is fp16, so the error grows as the token count
# falls: measured on an H100, 1.3e-4 at 8 tokens, 1.5e-5 at 12288; the linear layers losing a lo part costs >= 8.2e-4
COSTREG_TR_TOL = 2e-4
# zero_q: with the query projection zeroed every score is exactly 0 and P exactly 2^14, so the fp16 P costs nothing and
# the whole regulariser is an fp32-class computation.  Measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power
# limit): worst 9.7e-6 (32 x 136 x 240, without position), against 6.7e-5 with the normal weights
COSTREG_TR_ZERO_Q_TOL = 3e-5


# tokens = (D/2)(H/4)(W/4), attention query tiles of 128: (8, 48, 68) = 816 tokens, 7 tiles, the last 48 rows;
# (16, 64, 96) = 3072, 24 full tiles; (32, 96, 128) = 12288
COSTREG_TR_SHAPES = [(8, 12, 16), (32, 16, 16), (4, 8, 8), (8, 48, 68), (16, 64, 96), (32, 96, 128)]
# DTU and T&T stage 1: 27 648 and 32 640 tokens, where the attention's split plan cuts the last wave's items into key
# ranges (on 132 SMs) and attention_merge_kernel writes the hi|lo rows the proj GEMM reads
COSTREG_TR_STAGE1 = [(32, 144, 192), (32, 136, 240)]
COSTREG_TR_CASES = ([pytest.param(D, H, W, False, id=f"{D}-{H}-{W}") for D, H, W in COSTREG_TR_SHAPES + COSTREG_TR_STAGE1] +
                    [pytest.param(D, H, W, True, id=f"{D}-{H}-{W}-zero_q") for D, H, W in COSTREG_TR_SHAPES + COSTREG_TR_STAGE1])


@pytest.mark.parametrize("D,H,W,zero_q", COSTREG_TR_CASES)
def test_costreg_transformer_two_part(dev, D, H, W, zero_q):
    _check_costreg_transformer(dev, D, H, W, with_pos=True, zero_q=zero_q)


@pytest.mark.parametrize("D,H,W,zero_q", COSTREG_TR_CASES)
def test_costreg_transformer_two_part_without_position(dev, D, H, W, zero_q):
    _check_costreg_transformer(dev, D, H, W, with_pos=False, zero_q=zero_q)


def _check_costreg_transformer(dev, D, H, W, with_pos, zero_q=False):
    """The regulariser against the fp64 oracle, computed by torch on the device.  zero_q zeroes rows 0:64 (the query
    projection) of every layer's attn.qkv.weight: uniform attention, so the attention output is the same for every token
    and a row permutation of the proj GEMM's input would not show; the normal weights and the exact-weight kernel tests
    (test_gpu_attention_exact.py) cover how tokens mix."""
    from mvsformerplusplus_b200 import packing
    from mvsformerplusplus_b200.config import default_args
    from oracle import hotpath as O
    sd = _rand_vis_sd(17)
    cfg = default_args()["transformer_config"][0]
    p = "fusions.0.cost_reg."
    if zero_q:
        sd = dict(sd)
        for i in range(cfg["layer_num"]):
            k = f"{p}attention_layers.{i}.attn.qkv.weight"
            sd[k] = sd[k].clone()
            sd[k][:64] = 0.0
    g = torch.Generator().manual_seed(D)
    vol = torch.randn(1, 8, D, H, W, generator=g) * 0.5
    pos = torch.rand(1, 3, D, H, W, generator=g)
    if not with_pos:
        pos = None
    with torch.no_grad():
        want = O.costreg_transformer(vol.double().to(dev), pos.double().to(dev) if with_pos else None,
                                     {k: v.to(dev) for k, v in O.state_dict_to(sd, torch.float64).items()}, p, cfg)[0, 0]
    gemm, small = packing.pack_costreg_tr(sd, p, cfg["layer_num"])
    ws = _lib.workspace("mvsf_costreg_tr_workspace_bytes", 8, D, H, W, device=dev)
    logits = torch.full((D, H, W), float("nan"), device=dev)
    v = vol[0].permute(1, 2, 3, 0).contiguous().to(dev)
    n_tok = (D // 2) * (H // 4) * (W // 4)
    scale = 16 ** -0.5 * math.log(n_tok, cfg["train_avg_length"])
    pos_d = pos[0].contiguous().to(dev) if with_pos else None
    from mvsformerplusplus_b200.hotpath import split_weights_f16
    tc = split_weights_f16(gemm.to(dev))
    _lib.call("mvsf_costreg_tr_forward", v, pos_d, small.to(dev), tc, gemm.numel(), logits, ws, ws.numel() * 4, 8, D, H,
              W, cfg["layer_num"], float(scale))
    e = max_abs(logits, want)
    lim = (COSTREG_TR_ZERO_Q_TOL if zero_q else COSTREG_TR_TOL) * max(1.0, float(want.abs().max()))
    rec(f"costreg_tr_{D}x{H}x{W}" + ("" if with_pos else "_nopos") + ("_zero_q" if zero_q else ""), abs=e,
        scale=float(want.abs().max()), tokens=n_tok)
    assert e < lim, f"max error {e:.3e} vs fp64, limit {lim:.3e}"


def test_softargmax(dev):
    g = torch.Generator().manual_seed(2)
    for D in (4, 8, 16, 32, 5):
        H, W = 9, 21
        z = 3.0 * torch.randn(D, H, W, generator=g)
        hyp = 425.0 + 500.0 * torch.rand(D, H, W, generator=g)
        prob = torch.empty(D, H, W, device=dev)
        depth = torch.empty(H, W, device=dev)
        conf = torch.empty(H, W, device=dev)
        zd, hd = z.to(dev), hyp.to(dev)
        _lib.call("mvsf_softargmax", zd, hd, 5.0, prob, depth, conf, D, H, W)
        wp = F.softmax(z, 0)
        wd = (F.softmax(z * 5.0, 0) * hyp).sum(0)
        e = (max_abs(prob.cpu(), wp), rel_linf(depth.cpu(), wd), max_abs(conf.cpu(), wp.max(0)[0]))
        rec(f"softargmax_D{D}", prob=e[0], depth_rel=e[1], conf=e[2])
        assert e[0] < 1e-6 and e[1] < 1e-6 and e[2] < 1e-6


# ----------------------------------------------------------------------------------------------- FMT
# per output: |out - fp64| <= FMT_TOL * max(1, max|fp64|).  Measured on an H100 (all cases below): at most 1.8e-6; one
# GEMM family losing a lo operand part or the lo half of its split output costs >= 1.9e-4
FMT_TOL = 1e-5


@pytest.fixture(scope="module")
def fmt_net(dev, hp):
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    from oracle import hotpath as O
    args = default_args()
    torch.manual_seed(0)
    net = hp.HotPathNet(args).eval()
    sd = synth.randomize_state_dict(net, seed=23)
    return net.to(dev), O.state_dict_to(sd, torch.float64), args["FMT_config"]


def _check_fmt(name, out, feats, sd64, cfg):
    from oracle import hotpath as O
    with torch.no_grad():
        want = O.fmt_with_pathway({k: v.double() for k, v in feats.items()}, sd64, cfg)
    errs = {k: max_abs(out[k].cpu(), want[k]) for k in want}
    scales = {k: max(1.0, float(want[k].abs().max())) for k in want}
    rec(name, **errs, **{k + "_scale": s for k, s in scales.items()})
    for k in want:
        assert errs[k] < FMT_TOL * scales[k], f"{k}: max error {errs[k]:.3e} vs fp64, limit {FMT_TOL * scales[k]:.3e}"


# L = H1 * W1 tokens per view.  (2, 7, 9): L = 63, partial 32-token PE block and K/V tile, one source view.
# (5, 24, 40): L = 960, 4 K/V chunks (the last partial), L % 128 != 0 -> one linattn_apply launch per source view.
# (5, 16, 48): L = 768, L % 128 == 0 -> one batched linattn_apply over 4 source views.  (10, 48, 48): L = 2304 (9
# K/V chunks) and 9 * 2304 tokens > SMs * 128, so the linear-layer CTAs run more than one tile.
@pytest.mark.parametrize("V,H1,W1", [(3, 8, 12), (2, 16, 16), (4, 6, 10), (2, 7, 9), (5, 24, 40), (5, 16, 48),
                                     (10, 48, 48)])
def test_fmt_with_pathway(dev, fmt_net, V, H1, W1):
    from mvsformerplusplus_b200 import synth
    net, sd64, cfg = fmt_net
    feats = synth.make_features(V, H1 * 8, W1 * 8, seed=V)
    out = net.FMT_module.forward({k: v.to(dev) for k, v in feats.items()})
    _check_fmt(f"fmt_V{V}_{H1}x{W1}", out, feats, sd64, cfg)


def test_fmt_with_pathway_batch(dev, fmt_net):
    """B = 2 through FMT_with_pathway.forward: the batch loop reuses one workspace"""
    from mvsformerplusplus_b200 import synth
    net, sd64, cfg = fmt_net
    V, H1, W1 = 3, 16, 24
    f = [synth.make_features(V, H1 * 8, W1 * 8, seed=s) for s in (31, 32)]
    feats = {k: torch.cat([f[0][k], f[1][k]], 0) for k in f[0]}
    out = net.FMT_module.forward({k: v.to(dev) for k, v in feats.items()})
    for b in range(2):
        _check_fmt(f"fmt_B2_b{b}_V{V}_{H1}x{W1}", {k: v[b:b + 1] for k, v in out.items()}, f[b], sd64, cfg)


# ----------------------------------------------------------------------------------------------- stage seam + cascade
@pytest.fixture(scope="module", params=["hotpath_v3_96x128", "hotpath_v4_64x96"])
def cascade(request, dev, hp):
    from oracle import hotpath as O
    gold, meta = load_golden(request.param)
    args, params, sd, feats, proj, dv = build_case(meta)
    net = hp.HotPathNet(args).eval()
    net.load_state_dict(sd, strict=True)
    net = net.to(dev)
    out = net.forward_features({k: v.to(dev) for k, v in feats.items()}, {k: v.to(dev) for k, v in proj.items()},
                               dv.to(dev), TMP, keep_intermediates=True)
    with torch.no_grad():
        ora = O.hotpath_forward(feats, proj, dv, sd, args, tmp=TMP, keep_intermediates=True)
    return request.param, gold, out, ora, net, args, sd, proj, dv


@pytest.mark.parametrize("s", [1, 2, 3, 4])
def test_stage_seam_teacher_forced(cascade, dev, s):
    """StageNet.forward on the ORACLE's stage inputs (features, hypotheses, 3-D positions): per-stage parity at the
    north-star tolerances without cascade error accumulation."""
    from oracle import hotpath as O
    name, gold, out, ora, net, args, sd, proj, dv = cascade
    f = ora["features"][f"stage{s}"]
    ds = ora[f"stage{s}"]["depth_values"]
    p3d = None
    if s == 1:
        B, _, _, H, W = f.shape
        p3d, *_ = O.get_position_3d(B, H, W, proj["stage1"][:, 0, 1, :3, :3], ds, dv.min(), dv.max(), None, None, None, None)
    so = net.fusions[s - 1].forward(f.to(dev), proj[f"stage{s}"].to(dev), ds.to(dev), TMP[s - 1],
                                    position3d=None if p3d is None else p3d.to(dev), keep_intermediates=True)
    want = ora[f"stage{s}"]
    e = dict(entropy=max_abs(so["entropy"].cpu(), want["entropy"]), vis=max_abs(so["vis_weight"].cpu(), want["vis_weight"]),
             volume=max_abs(so["volume_mean"].cpu().permute(0, 4, 1, 2, 3), want["volume_mean"]),
             logits=max_abs(so["prob_volume_pre"].cpu(), want["prob_volume_pre"]),
             prob=max_abs(so["prob_volume"].cpu(), want["prob_volume"]),
             conf=max_abs(so["photometric_confidence"].cpu(), want["photometric_confidence"]),
             depth_rel=rel_linf(so["depth"].cpu(), want["depth"]))
    rec(f"stage_seam_{name}_s{s}", **e)
    assert e["prob"] < 1e-4 and e["conf"] < 1e-4 and e["depth_rel"] < 1e-3


@pytest.mark.parametrize("s", [1, 2, 3, 4])
def test_cascade_vs_reference_golden(cascade, s):
    """Full FMT + cascade on the GPU against the reference-executed fixture (fp32 reference forward)."""
    name, gold, out, ora, *_ = cascade
    so = out[f"stage{s}"]
    gp = torch.softmax(gold[f"stage{s}.prob_volume_pre"], dim=0)
    e = dict(depth_values_rel=rel_linf(so["depth_values"][0].cpu(), gold[f"stage{s}.depth_values"]),
             entropy=max_abs(so["entropy"][0].cpu(), gold[f"stage{s}.entropy"]),
             vis=max_abs(so["vis_weight"][0].cpu(), gold[f"stage{s}.vis_weight"]),
             prob=max_abs(so["prob_volume"][0].cpu(), gp),
             conf=max_abs(so["photometric_confidence"][0].cpu(), gold[f"stage{s}.photometric_confidence"]),
             depth_rel=rel_linf(so["depth"][0].cpu(), gold[f"stage{s}.depth"]))
    rec(f"cascade_{name}_s{s}", **e)
    assert e["prob"] < 1e-4 and e["conf"] < 1e-4 and e["depth_rel"] < 1e-3


def test_cascade_final_outputs(cascade):
    name, gold, out, ora, *_ = cascade
    e = dict(refined_depth_rel=rel_linf(out["refined_depth"][0].cpu(), gold["refined_depth"]),
             confidence=max_abs(out["photometric_confidence"][0].cpu(), gold["photometric_confidence"]),
             fmt_stage1=max_abs(out["features"]["stage1"][0].cpu(), gold["fmt.stage1"]),
             fmt_stage4_view1=max_abs(out["features"]["stage4"][0, 1].cpu(), gold["fmt.stage4.view1"]))
    rec(f"cascade_{name}_final", **e)
    assert e["refined_depth_rel"] < 1e-3 and e["confidence"] < 1e-4 and e["fmt_stage1"] < 2e-4


# ----------------------------------------------------------------------------------------------- full-size properties
def test_full_size_properties(dev, hp):
    """BASELINE config 2 sizes (V=5, 1152x1536, ndepths 32/16/8/4): properties that do not need the CPU oracle."""
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    args = default_args()
    V, H, W = 5, 1152, 1536
    torch.manual_seed(0)
    net = hp.HotPathNet(args).eval()
    synth.randomize_state_dict(net, seed=7)
    net = net.to(dev)
    feats = {k: v.to(dev) for k, v in synth.make_features(V, H, W, seed=1234, smooth=False).items()}
    proj = {k: v.to(dev) for k, v in synth.make_proj_matrices(V, H, W).items()}
    dv = synth.make_depth_values(192).to(dev)
    out = net.forward_features(feats, proj, dv, TMP)
    out2 = net.forward_features(feats, proj, dv, TMP)
    torch.cuda.synchronize()
    facts = {}
    for s in range(1, 5):
        so = out[f"stage{s}"]
        pv = so["prob_volume"]
        facts[f"s{s}_finite"] = bool(torch.isfinite(pv).all() and torch.isfinite(so["depth"]).all())
        facts[f"s{s}_prob_sum_err"] = float((pv.sum(1) - 1).abs().max())
        facts[f"s{s}_conf_is_max"] = float((so["photometric_confidence"] - pv.max(1)[0]).abs().max())
        lo, hi = so["depth_values"].min(1)[0], so["depth_values"].max(1)[0]
        facts[f"s{s}_depth_in_range"] = bool(((so["depth"] >= lo * (1 - 1e-5)) & (so["depth"] <= hi * (1 + 1e-5))).all())
        facts[f"s{s}_deterministic"] = bool(torch.equal(so["depth"], out2[f"stage{s}"]["depth"]))
    facts["refined_shape"] = list(out["refined_depth"].shape)
    rec("full_size_properties", **{k: (v if not isinstance(v, bool) else int(v)) for k, v in facts.items()})
    for s in range(1, 5):
        assert facts[f"s{s}_finite"] and facts[f"s{s}_depth_in_range"] and facts[f"s{s}_deterministic"]
        assert facts[f"s{s}_prob_sum_err"] < 1e-5 and facts[f"s{s}_conf_is_max"] == 0.0
    assert facts["refined_shape"] == [1, H, W]


def test_identity_homography_property(dev):
    """src camera == ref camera at full DTU stage-4 size: pass B (window kernel) against the fp64 reference at the
    library's own coordinates, which sit within fp32 normalisation rounding of the pixel centres, so the volume is
    vol[g] = mean_{c in g} ref * src (all views weighted alike) up to that rounding"""
    from mvsformerplusplus_b200 import synth
    H, W, C, D, V = 1152, 1536, 8, 4, 2
    pm = synth.make_proj_matrices(1, H, W)["stage4"][0]
    pm = torch.cat([pm, pm], 0).to(dev)
    homs = torch.empty(12, device=dev)
    kinv = torch.empty(9, device=dev)
    _lib.call("mvsf_compose_geometry", pm, 2, homs, kinv)
    g = torch.Generator(device="cpu").manual_seed(0)
    f = torch.randn(V, H, W, C, generator=g).to(dev)
    dd = (425.0 + 100.0 * torch.arange(D, dtype=torch.float32)).view(D, 1, 1).expand(D, H, W).contiguous().to(dev)
    vis = torch.full((1, H, W), 0.7, device=dev)
    vol = torch.empty(D, H, W, C, device=dev)
    _lib.call("mvsf_warp_corr_aggregate", f, homs, dd, vis, vol, V, C, 8, D, H, W)
    corr64, _ = R.CostVolumeRef(f, homs.view(1, 12), dd).view(0)
    want = R.aggregate(corr64[None], vis.view(1, -1))
    scale = max(1.0, float(want.abs().max()))
    e = max_abs(vol.view(D, H * W, 8), want) / scale
    e_closed = float((vol - (f[0] * f[1])[None] * (0.7 / (0.7 + 1e-6))).abs().max())
    rec("identity_homography", abs64=e, scale=scale, closed_form_abs=e_closed)
    assert e < R.VOL_TOL, f"{e:.3e} against fp64"


# ----------------------------------------------------------------------------------------------- tensor-core attention
@pytest.mark.parametrize("N", [1, 64, 128, 129, 200, 385, 1000, 4000, 27648, 32640])
def test_attention_tensor_core_vs_fp64(dev, N):
    """Product attention kernel (wgmma, fp16 hi|lo split Q/K/V operands, fp16 softmax probabilities) against an fp64
    softmax(QK^T*scale)V evaluated with torch on the GPU (test-side ground truth, chunked over queries).
    Inputs are deliberately harsher than LayerNorm-ed tokens (std 1.5 -> |score| up to ~14 in log2 units).
    N = 32640 is the Tanks&Temples token count (odd number of 128-query tiles: the last CTA repeats a tile).  The small N
    reach the edges of the tiling: one key (N = 1), query blocks past the last one that re-read it (N = 1, 64, 129), a
    full key tile with no masked keys (128), a last tile of one key (129), and a K / V ring that wraps around (385: four
    key tiles through three stages, three CTAs)."""
    g = torch.Generator().manual_seed(N)
    qkv = torch.randn(N, 192, generator=g) * 1.5
    scale = 16 ** -0.5 * math.log(N, 12185)
    qd = qkv.to(dev)
    ws = torch.empty((N + 128) * 224 + 16, device=dev)
    o0 = torch.empty(N, 64, device=dev)
    _lib.call("mvsf_attention_forward", qd, o0, ws, ws.numel() * 4, N, float(scale))
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(3):
        _lib.call("mvsf_attention_forward", qd, o0, ws, ws.numel() * 4, N, float(scale))
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / 3
    q, k, v = [qd[:, i * 64:(i + 1) * 64].double().view(N, 4, 16).transpose(0, 1) for i in range(3)]
    want = torch.empty(4, N, 16, dtype=torch.float64, device=dev)
    for s0 in range(0, N, 2048):
        a = torch.softmax(q[:, s0:s0 + 2048] @ k.transpose(1, 2) * scale, -1)
        want[:, s0:s0 + 2048] = a @ v
    want = want.transpose(0, 1).reshape(N, 64)
    e_tc, sc = max_abs(o0, want), float(want.abs().max())
    rms = float((o0.double() - want).pow(2).mean().sqrt())
    rec(f"attention_N{N}", tc_vs_f64=e_tc, rms=rms, scale=sc, ms_with_operand_tiling=ms)
    # an fp32 one-thread-per-query kernel measured 4.3e-4
    assert e_tc < 4e-4 * sc


def test_prefetching_runner_matches_direct_call(dev):
    """streaming.PrefetchingRunner (copy stream + two device slots) returns what a direct forward_features on
    device-resident inputs returns, for alternating batches, with and without prefetch."""
    import bench
    from mvsformerplusplus_b200.streaming import PrefetchingRunner
    net, _ = bench.make_net()
    net = net.to(dev)
    wl = bench.WORKLOADS["small"]
    batches = []
    for seed in (11, 12, 13):
        f, p, d = bench.make_inputs(wl, seed)
        batches.append(({k: v.pin_memory() for k, v in f.items()}, {k: v.pin_memory() for k, v in p.items()}, d.pin_memory()))
    want = []
    for f, p, d in batches:
        out = net.forward_features({k: v.to(dev) for k, v in f.items()}, {k: v.to(dev) for k, v in p.items()}, d.to(dev), bench.TMP)
        want.append((out["refined_depth"].clone(), out["photometric_confidence"].clone()))
    runner = PrefetchingRunner(net, dev)
    order = [0, 1, 2, 0, 2, 1, 1]
    for i, b in enumerate(order):
        nxt = batches[order[i + 1]] if i + 1 < len(order) and i % 3 != 2 else None   # every third call: no prefetch
        out = runner.run(batches[b], next_batch=nxt, tmp=bench.TMP)
        torch.cuda.synchronize()
        assert torch.equal(out["refined_depth"], want[b][0]), f"call {i} (batch {b})"
        assert torch.equal(out["photometric_confidence"], want[b][1])
