"""The fp64 references and the cases of tests/geometry_common.py pinned on the CPU: the restatements agree with
oracle/hotpath.py run in fp64, the confidence restatement is F.interpolate bit for bit, and every case is what it claims
to be (negative hypotheses on the wide range, each extreme in its sample and beyond the first grid-stride trip)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import hotpath as O
from tests import geometry_common as G
from tests.common import max_abs


@pytest.mark.parametrize("D,Dn", [(2, 2), (32, 192), (48, 192), (4, 2)])
def test_init_reference_matches_oracle(D, Dn):
    for lo, hi in (G.DTU_RANGE, G.TT_RANGE, G.WIDE_RANGE):
        dv = G.depth_values(lo, hi, Dn)
        want = 1 / O.init_inverse_range(dv[None].double(), D, 3, 5)[0]
        got = G.init_inv64(dv, D).view(D, 1, 1)
        assert max_abs(got, want) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("H,W,D,ratio,wide", [(288, 384, 16, 2.67, False), (74, 106, 8, 1.5, True), (2, 2, 4, 1.0, False),
                                              (272, 480, 16, 2.67, True)])
def test_schedule_reference_matches_oracle(H, W, D, ratio, wide):
    """in fp64 coordinates the restatement is the oracle's schedule in fp64 (in inverse space); in the kernel's fp32
    coordinates it moves by up to the rounding of a coordinate (ulp(240) = 1.5e-5) times a neighbour difference, far
    more than the kernel's own arithmetic: that is why the kernel is compared at its own coordinates"""
    dv, stage_depth = G.cascade_inputs(G.DTU, wide, seed=H)
    prev = O.init_inverse_range(dv[None], G.NDEPTHS[0], H // 2, W // 2)[0]
    depth = stage_depth(prev)
    want = 1 / O.schedule_inverse_range(depth[None].double(), prev[None].double(), D, G.f32(ratio), H, W)[0]
    got = G.schedule_inv64(depth, prev, D, ratio, H, W, coords=torch.float64)
    scale = float(want.abs().max())
    assert max_abs(got, want) <= 1e-12 * scale
    got32 = G.schedule_inv64(depth, prev, D, ratio, H, W)
    assert max_abs(got32, want) <= 1e-4 * scale


def test_blend_axis_matches_oracle_fp32():
    """the fp32 source coordinates are the ones the fp32 oracle blends at: a plane that is its column (row) index
    upsampled by the oracle equals the restated blend of it"""
    for h, w in ((1, 1), (37, 53), (144, 192), (544, 960)):
        x = torch.arange(w, dtype=torch.float32).expand(1, 1, h, w)
        up = O.upsample2x_align_corners(x, 2 * h, 2 * w)[0, 0, 0]
        x0, x1, w0, w1 = G.blend_axis(w, 2 * w)
        assert torch.equal(up, (x0.float() * w0.float() + x1.float() * w1.float()))


def test_wide_range_drives_the_schedule_negative():
    """dmax / dmin = 100 > 1 + 31 / 2.67: the stage-2 inverse maximum 1/depth - 2.67 itv is < 0 at far pixels, and the
    planes hold negative hypotheses there"""
    for H, W in ((272, 480), (37, 53), (144, 192)):
        planes = G.wide_planes(H, W)
        assert int((planes < 0).sum()) > 0 and bool(torch.isfinite(planes).all())
    dv, stage_depth = G.cascade_inputs(G.TT, True, seed=1)
    prev = O.init_inverse_range(dv[None], G.NDEPTHS[0], 136, 240)[0]
    v = G.schedule_halfres64(stage_depth(prev), prev, 16, 2.67)
    assert int((v[0] < 0).sum()) > 0


@pytest.mark.parametrize("B,D,wide", [(1, 8, False), (2, 8, True), (3, 8, False)])
def test_position_reference_matches_oracle(B, D, wide):
    """positions and fp64 extents of the restatement against get_position_3d in fp64, one K per batch reduced over the
    batch; the fp32 extents are within fp32 rounding of the fp64 ones"""
    H, W = 24, 40
    pm, hyp, dvs, _ = G.position_case(B, H, W, D, "tt", wide, seed=B)
    K = pm[:, 0, 1, :3, :3].double()
    kinv64 = torch.inverse(K).reshape(B, 9)
    want, hmin, hmax, wmin, wmax = O.get_position_3d(B, H, W, K, hyp.double(), dvs.min().double(), dvs.max().double(),
                                                     None, None, None, None)
    ext = G.extents(kinv64, hyp.double())
    assert max_abs(torch.stack(ext), torch.stack([wmin, wmax, hmin, hmax])) <= 1e-12 * float(torch.stack(ext).abs().max())
    stats = [*ext, dvs.min(), dvs.max()]
    for b in range(B):
        got = G.positions64(kinv64[b], hyp[b], stats)
        assert max_abs(got, want[b]) <= 1e-12
    ext32 = G.extents(kinv64.float(), hyp)
    assert all(abs(float(a) - float(b)) <= 1e-6 * abs(float(b)) for a, b in zip(ext32, ext))


@pytest.mark.parametrize("B,H,W,D,kind,wide", [(1, 144, 192, 32, "dtu", False), (2, 144, 192, 32, "dtu", False),
                                               (3, 136, 240, 32, "tt", False), (2, 136, 240, 32, "tt", True),
                                               (3, 137, 239, 32, "tt", False), (2, 75, 243, 48, "dtu", False)])
def test_position_case_extremes(B, H, W, D, kind, wide):
    """each of the six extremes comes from the sample the case names (the last sample among them), the x / y extremes
    from the last grid-stride trip on 132 SMs, and the case exceeds 2 x 132 x 8 x 256 samples; hypotheses lie above
    and below the depth range (the z clamp), and the wide case has negative ones"""
    pm, hyp, dvs, owners = G.position_case(B, H, W, D, kind, wide, seed=7 * B + H)
    assert D * H * W > 2 * G.H100_SMS * G.POS3D_BLOCKS_PER_SM * G.POS3D_THREADS
    assert (D * H * W) % 256 or (H, W) in ((144, 192), (136, 240))
    kinvs = torch.inverse(pm[:, 0, 1, :3, :3].double()).reshape(B, 9).float()
    own = G.extreme_owners(kinvs, hyp, dvs)
    assert {k: b for k, (b, _) in own.items()} == owners
    assert B == 1 or B - 1 in owners.values()
    trips, stride = G.minmax_trips(D, H, W, G.H100_SMS)
    assert trips >= 2
    for k in ("xmin", "xmax", "ymin", "ymax"):
        assert own[k][1] // stride == trips - 1, (k, own[k], stride, trips)
    assert bool((hyp > dvs.max()).any()) and bool((hyp < dvs.min()).any())
    assert bool((hyp < 0).any()) == wide


@pytest.mark.parametrize("sizes", [[(144, 192), (288, 384), (576, 768), (1152, 1536)],
                                   [(136, 240), (272, 480), (544, 960), (1088, 1920)],
                                   [(37, 53), (50, 60), (73, 97), (100, 120)]])
def test_nearest_restatement_is_interpolate(sizes):
    """the restated source indices gather exactly what F.interpolate(mode="nearest") returns, at every stage ratio"""
    Hf, Wf = sizes[-1]
    g = torch.Generator().manual_seed(Hf)
    acc = None
    for h, w in sizes:
        c = torch.rand(h, w, generator=g)
        up = G.nearest_upsample(c, Hf, Wf)
        assert torch.equal(up, F.interpolate(c[None, None], (Hf, Wf), mode="nearest")[0, 0])
        acc = up * 0.25 if acc is None else acc + up * 0.25
    g = torch.Generator().manual_seed(Hf)
    confs = [torch.rand(h, w, generator=g) for h, w in sizes]
    assert torch.equal(acc, G.confidence_average(confs, Hf, Wf))
    # the reference's own order (prob_maps += conf; / 4) gives the same bits
    ref = torch.zeros(Hf, Wf)
    for c in confs:
        ref += F.interpolate(c[None, None], (Hf, Wf), mode="nearest")[0, 0]
    assert torch.equal(ref / 4, acc)


def test_softargmax_cases():
    """the four logit kinds are present in the last partial block of 256 pixels; flat pixels are flat; ties share the
    maximum; peaked pixels lead by 30"""
    D, H, W = 8, 37, 53
    z, flat = G.softargmax_logits(D, H, W, seed=1)
    zf = z.view(D, -1)
    tail = torch.arange(H * W) >= (H * W // 256) * 256
    kind = torch.arange(H * W) % 4
    assert set(kind[tail].tolist()) == {0, 1, 2, 3}
    assert torch.equal(flat.view(-1), kind == 2)
    assert bool((zf[:, kind == 2] == zf[:1, kind == 2]).all())
    top2 = zf.topk(2, 0).values
    assert bool((top2[0, kind == 3] == top2[1, kind == 3]).all())
    assert bool((top2[0, kind == 1] - top2[1, kind == 1] >= 29.99).all())
    p, c, d, s = G.softargmax64(z, G.narrow_planes(D, H, W), 5.0)
    assert bool((p.view(D, -1)[:, kind == 2] == 1 / D).all())
    assert torch.allclose(d, (torch.softmax(z.double() * 5, 0) * G.narrow_planes(D, H, W).double()).sum(0), rtol=1e-6)
