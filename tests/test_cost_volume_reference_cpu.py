"""The fp64 cost-volume reference of tests/cost_volume_common.py pinned to the oracle (itself pinned to the
reference-executed fixtures by tests/test_oracle_golden.py) and to the reference-executed warp seam fixture."""
import pytest
import torch

from tests import cost_volume_common as R
from tests.common import load_golden, max_abs

# (C, D, H, W, V, theta step, depth jitter): small shapes of tests/test_gpu_parity.py COST_CASES
CASES = [(8, 4, 37, 53, 3, 0.1, 0.02), (16, 8, 24, 40, 3, 0.1, 0.02), (32, 16, 16, 24, 4, 0.12, 0.02),
         (64, 32, 12, 16, 5, 0.1, 0.02), (8, 4, 31, 45, 3, 0.6, 0.02), (8, 48, 10, 14, 3, 0.1, 0.02)]


def _case(C, D, H, W, V, th, jit):
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    g = torch.Generator().manual_seed(C * 1000 + D)
    feats = torch.randn(1, V, C, H, W, generator=g)
    sc = {8: 1, 16: 2, 32: 4, 64: 8}[C]
    pm = synth.make_proj_matrices(V, H * sc, W * sc, theta_step=th)[f"stage{ {1: 4, 2: 3, 4: 2, 8: 1}[sc] }"]
    dvals = O.init_inverse_range(synth.make_depth_values(192), D, H, W) * (1.0 + jit * torch.rand(1, D, H, W, generator=g))
    return feats, pm, dvals


def _ulps(a, b):
    """|a - b| in units of the fp32 spacing at max(|a|, |b|), over the entries where both are finite"""
    ok = torch.isfinite(a) & torch.isfinite(b)
    a, b = a[ok], b[ok]
    m = torch.maximum(a.abs(), b.abs())
    return float(((a.double() - b.double()).abs() / (torch.nextafter(m, torch.full_like(m, float("inf"))) - m).double()).max())


@pytest.mark.parametrize("C,D,H,W,V,th,jit", CASES)
def test_coordinates_match_oracle(C, D, H, W, V, th, jit):
    """restated coordinates against oracle.hotpath.warp_coordinates fed the same rotation and translation (identity
    reference projection).  The oracle forms the ray with a matmul, whose summation order and FMA use are the BLAS's
    choice; measured: 0 ulp on ix, iy and Z in every case"""
    from oracle import hotpath as O
    _, pm, dvals = _case(C, D, H, W, V, th, jit)
    homs = R.compose_homs_fp64(pm[0])
    ix, iy, Z = R.restated_coords(homs, dvals[0])
    for v in range(V - 1):
        src = torch.eye(4)
        src[:3, :3] = homs[v, :9].view(3, 3)
        src[:3, 3] = homs[v, 9:]
        px, py, z = O.warp_coordinates(src[None], torch.eye(4)[None], dvals, H, W)
        u = (_ulps(ix[v], px[0]), _ulps(iy[v], py[0]), _ulps(Z[v], z[0]))
        assert max(u) <= 4, u


@pytest.mark.parametrize("C,D,H,W,V,th,jit", CASES)
def test_reference_matches_fp32_oracle(C, D, H, W, V, th, jit, monkeypatch):
    """entropy, vis and volume of the fp64 reference against oracle.hotpath.cost_volume in fp32 with the homography
    composed in fp64 and rounded once (the library's rounding): the two agree to the oracle's fp32 noise.  Measured:
    entropy 1.4e-6, vis 2.9e-7, volume 4.1e-7 (relative to max(1, max|volume|))"""
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.params import build_hotpath_params
    from oracle import hotpath as O
    monkeypatch.setattr(O, "HOMOGRAPHY_FP64", True)
    torch.manual_seed(0)
    sd = synth.randomize_state_dict(build_hotpath_params(default_args()).eval(), seed=5)
    feats, pm, dvals = _case(C, D, H, W, V, th, jit)
    want = O.cost_volume(feats, pm, dvals, sd, "fusions.3.", 8)
    ref = R.CostVolumeRef(feats[0].permute(0, 2, 3, 1).contiguous(), R.compose_homs_fp64(pm[0]), dvals[0].contiguous())
    corr, ent = ref.pass_a()
    vis = R.vis_fp64(ent.view(V - 1, H, W), R.state_dict_fp64(sd, "cpu"), "fusions.3.")
    vol = R.aggregate(corr, vis.view(V - 1, -1))
    e_ent = max_abs(ent.view(V - 1, H, W), want["entropy"][0])
    e_vis = max_abs(vis, want["vis_weight"][0])
    scale = max(1.0, float(vol.abs().max()))
    e_vol = max_abs(vol.view(D, H, W, 8).permute(3, 0, 1, 2), want["volume_mean"][0]) / scale
    assert e_ent < 5e-6 and e_vis < 1e-6 and e_vol < 1.5e-6, (e_ent, e_vis, e_vol)


def test_reference_reproduces_warp_seam():
    """bilinear samples at the restated coordinates against the reference-executed warp seam fixture, within the GPU seam
    test's bar (measured 6.9e-6: the fixture's homography is the reference's fp32 inverse); the mask agrees everywhere"""
    g, _ = load_golden("warp_seam")
    src = g["src"][0]
    C, H, W = src.shape
    depth = g["depth_values"][0].contiguous()
    ix, iy, Z = R.restated_coords(R.seam_hom(g["src_proj"][0], g["ref_proj"][0])[None], depth)
    flat = src.permute(1, 2, 0).reshape(-1, C).double()
    got = torch.stack([R.sample(flat, ix[0, d], iy[0, d], H, W) for d in range(depth.shape[0])]).permute(2, 0, 1)
    assert max_abs(got.reshape(g["warped"][0].shape), g["warped"][0]) < 2e-4
    mask = (ix > W - 1) | (ix < 0) | (iy > H - 1) | (iy < 0) | (Z <= 0)
    assert torch.equal(mask.view(g["mask"][0].shape), g["mask"][0])
