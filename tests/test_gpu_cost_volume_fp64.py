"""Cost-volume kernels against the fp64 reference at the library's own sample coordinates (tests/cost_volume_common.py),
at the sizes where the persistent pipeline kernel and the strided L1 kernel loop, plus the selection kernel's window-miss
count and the standalone warp seam.  Every loop case asserts, from the running device's SM count, that it loops."""
import ctypes

import pytest
import torch

from mvsformerplusplus_b200 import _lib
from tests import cost_volume_common as R
from tests.common import load_golden, max_abs, rec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _case(dev, C, D, H, W, V, th, jit, seed, band=None):
    """channels-last features [V, H, W, C], homographies [V-1, 12] from mvsf_compose_geometry, hypotheses [D, H, W]: the
    first stage's inverse range over 425..931, or `band` = (near, far) spread evenly (a later stage's narrow range)"""
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(V, H, W, C, generator=g).to(dev)
    pm = synth.make_proj_matrices(V, H, W, theta_step=th)["stage4"][0].to(dev)
    dv = synth.make_depth_values(192)
    if band is None:
        base = O.init_inverse_range(dv, D, H, W)[0]
    else:
        base = (band[0] + (band[1] - band[0]) * torch.arange(D, dtype=torch.float32) / (D - 1)).view(D, 1, 1).expand(D, H, W)
    dd = (base * (1.0 + jit * torch.rand(D, H, W, generator=g))).contiguous().to(dev)
    homs = torch.empty(V - 1, 12, device=dev)
    kinv = torch.empty(9, device=dev)
    _lib.call("mvsf_compose_geometry", pm, V, homs, kinv)
    return f, homs, dd


def _entropy_store(dev, mode, f, homs, dd, V, C, D, H, W):
    """pass A of the spill plan with the tile path in `mode`; outputs prefilled with NaN"""
    ent = torch.full((V - 1, H, W), float("nan"), device=dev)
    corr = torch.full((V - 1, D, H, W, 8), float("nan"), device=dev)
    _lib.call("mvsf_warp_corr_set_tile_path", mode)
    try:
        _lib.call("mvsf_warp_corr_entropy_store", f, homs, dd, ent, corr, V, C, 8, D, H, W)
    finally:
        _lib.call("mvsf_warp_corr_set_tile_path", 1)
    return ent, corr


def _last_selection():
    used, miss = ctypes.c_int(-1), ctypes.c_int(-1)
    _lib.call("mvsf_warp_corr_last_selection", ctypes.byref(used), ctypes.byref(miss))
    return used.value, miss.value


def _against_fp64(ref, ent, corr):
    """largest entropy error (absolute) and correlation error (relative to max(1, max|fp64|)) over all source views"""
    e_ent = e_corr = 0.0
    scale = 1.0
    for v in range(ref.V - 1):
        corr64, ent64 = ref.view(v)
        scale = max(scale, float(corr64.abs().max()))
        e_ent = max(e_ent, max_abs(ent[v].reshape(-1), ent64))
        e_corr = max(e_corr, max_abs(corr[v].reshape(ref.D, -1, 8), corr64))
        del corr64, ent64
    return e_ent, e_corr / scale, scale


# 250 x 1000: 32 x 32 tiles with ragged right (8 columns) and bottom (2 rows) tiles, 9 source views = 3 turns of the
# 3-window ring per tile, 1024 tiles = 3-4 per CTA at 132 SMs (4-5 at 114).  1152 x 1536 (DTU stage 4): 6912 tiles,
# 26-27 per CTA at 132 SMs.
@pytest.mark.parametrize("H,W,V", [(250, 1000, 10), (1152, 1536, 5)])
def test_pipeline_kernel_loops(dev, H, W, V):
    C, D = 8, 4
    lo, hi, turns = R.pipeline_coverage(H, W, V, _sms())
    assert lo >= 3, (lo, hi)
    if V == 10:
        assert turns == 3
    torch.cuda.reset_peak_memory_stats()
    f, homs, dd = _case(dev, C, D, H, W, V, 0.1, 0.02, seed=H + V)
    ent, corr = _entropy_store(dev, 2, f, homs, dd, V, C, D, H, W)   # forced: the pipeline kernel
    written = bool(torch.isfinite(ent).all()) and bool(torch.isfinite(corr).all())
    ref = R.CostVolumeRef(f, homs, dd)
    e_ent, e_corr, scale = _against_fp64(ref, ent, corr)
    rec(f"cost_volume_pipeline_{H}x{W}_V{V}", entropy64=e_ent, corr64=e_corr, corr64_scale=scale, tiles_per_cta_min=lo,
        tiles_per_cta_max=hi, ring_turns_per_tile=turns, sms=_sms(), peak_gb=torch.cuda.max_memory_allocated() / 2**30)
    assert written, "the pipeline kernel left entropy or correlations unwritten"
    assert e_ent < R.ENT_TOL and e_corr < R.CORR_TOL, (e_ent, e_corr)


def test_strided_l1_kernel_loops(dev):
    """the adaptive spill plan at a wide baseline: the selection kernel hands the call to the strided L1 kernel, whose
    capped grid (16 CTAs per SM) takes 2-3 trips per CTA at 768 x 1024"""
    C, D, H, W, V = 8, 4, 768, 1024, 3
    lo, hi = R.strided_trips(H, W, _sms())
    assert lo >= 2, (lo, hi)
    torch.cuda.reset_peak_memory_stats()
    f, homs, dd = _case(dev, C, D, H, W, V, 0.6, 0.02, seed=7)
    ent, corr = _entropy_store(dev, 1, f, homs, dd, V, C, D, H, W)
    used, miss = _last_selection()
    ref = R.CostVolumeRef(f, homs, dd)
    want_miss, want_used, tot, nmiss = R.selector_restated(ref)
    written = bool(torch.isfinite(ent).all()) and bool(torch.isfinite(corr).all())
    e_ent, e_corr, scale = _against_fp64(ref, ent, corr)
    rec(f"cost_volume_strided_{H}x{W}_V{V}", entropy64=e_ent, corr64=e_corr, corr64_scale=scale, trips_min=lo, trips_max=hi,
        used_pipeline=used, miss_permille=miss, miss_permille_restated=want_miss, sms=_sms(),
        peak_gb=torch.cuda.max_memory_allocated() / 2**30)
    assert used == 0 and miss == want_miss, (used, miss, want_miss)
    assert written, "the strided L1 kernel left entropy or correlations unwritten"
    assert e_ent < R.ENT_TOL and e_corr < R.CORR_TOL, (e_ent, e_corr)


def test_selector_miss_share(dev):
    """warp_stream_select_kernel's miss share equals the host restatement of its count, its decision is miss <= 60 per
    mille, and a call does not see the previous one (narrow, wide, narrow read back the same for both narrow calls)"""
    C, D, H, W, V = 8, 4, 256, 384, 3
    cases = {"narrow": _case(dev, C, D, H, W, V, 0.1, 0.002, seed=11, band=(600.0, 606.0)),
             "wide": _case(dev, C, D, H, W, V, 0.6, 0.3, seed=12)}
    want = {k: R.selector_restated(R.CostVolumeRef(*c)) for k, c in cases.items()}
    got = []
    for k in ("narrow", "wide", "narrow"):
        _entropy_store(dev, 1, *cases[k], V, C, D, H, W)
        got.append(_last_selection())
    rec("cost_volume_selector", **{f"{k}_restated_permille": w[0] for k, w in want.items()},
        **{f"{k}_restated_taps": w[2] for k, w in want.items()}, narrow_permille=got[0][1], wide_permille=got[1][1],
        narrow_again_permille=got[2][1], narrow_used=got[0][0], wide_used=got[1][0])
    assert got[0] == got[2], got
    for (used, miss), k in zip(got, ("narrow", "wide", "narrow")):
        assert miss == want[k][0], (k, miss, want[k])
        assert used == (1 if miss <= R.MAX_MISS_PERMILLE else 0)
    assert got[0][0] == 1 and got[1][0] == 0, got   # the two cases fall on either side of the threshold


def _homo_warp_cases():
    """(name, src [H, W, C], hom [12], depth [D, H, W]) for the reference-executed seam fixture and both grazing views"""
    g, _ = load_golden("warp_seam")
    src = g["src"][0].permute(1, 2, 0).contiguous()
    yield "warp_seam", src, R.seam_hom(g["src_proj"][0], g["ref_proj"][0]), g["depth_values"][0].contiguous()
    H, W, C, D = 36, 52, 8, 4
    gen = torch.Generator().manual_seed(5)
    src = torch.randn(H, W, C, generator=gen)
    homs = R.compose_homs_fp64(R.grazing_projections(H, W))
    for v in range(2):
        yield f"grazing_view{v + 1}", src, homs[v], R.grazing_depth(D, H, W, seed=v)


def test_homo_warp_at_restated_coordinates(dev):
    """mvsf_homo_warp: the mask is the restated coordinates' comparison, bit for bit, and the samples are the fp64
    bilinear samples at those coordinates up to fp32 rounding"""
    for name, src, hom, depth in _homo_warp_cases():
        H, W, C = src.shape
        D = depth.shape[0]
        warped = torch.empty(C, D, H, W, device=dev)
        mask = torch.empty(D, H, W, dtype=torch.uint8, device=dev)
        src_d, hom_d, depth_d = src.to(dev), hom.to(dev), depth.to(dev)
        _lib.call("mvsf_homo_warp", src_d, hom_d, depth_d, warped, mask, C, D, H, W)
        ix, iy, Z = R.restated_coords(hom_d[None], depth_d)
        ix, iy, Z = ix[0], iy[0], Z[0]
        want_mask = (ix > W - 1) | (ix < 0) | (iy > H - 1) | (iy < 0) | (Z <= 0)
        want = torch.stack([R.sample(src_d.reshape(-1, C).double(), ix[d], iy[d], H, W) for d in range(D)])   # [D, HW, C]
        want = want.permute(2, 0, 1).reshape(C, D, H, W)
        scale = max(1.0, float(want.abs().max()))
        e = max_abs(warped, want) / scale
        mism = int((mask.bool().view(D, -1) != want_mask).sum())
        rec(f"homo_warp_restated_{name}", abs64=e, scale=scale, mask_mismatch=mism,
            masked=int(want_mask.sum()), nonfinite=int((~torch.isfinite(ix)).sum()))
        assert mism == 0, (name, mism)
        assert e < R.WARP_TOL, (name, e)
