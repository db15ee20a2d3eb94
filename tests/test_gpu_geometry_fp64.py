"""The cascade glue kernels of geometry.cu against fp64 (tests/geometry_common.py) at the shipped stage sizes: projection
composition up to 64 views and 70 batch items, the first stage's hypotheses, the schedule through all four stages of
DTU, T&T and a wide depth range, the 3-D positions through the cascade's batched call sequence with its grid-stride
loop taking 2+ trips, the soft-argmax at every stage size and temperature, and the confidence average.  Every output
is prefilled with NaN, except the homographies of mvsf_homography_from_proj, whose singular item must write NaN itself."""
import pytest
import torch

from mvsformerplusplus_b200 import _lib, synth
from tests import geometry_common as G
from tests.common import rec

pytestmark = pytest.mark.gpu
NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nan(*shape):
    return torch.full(shape, NAN, device="cuda:0")


def _rows34(h):
    """[N, 12] rotation | translation -> [N, 3, 4] rows of the 3 x 4 matrix"""
    h = h.reshape(-1, 12)
    return torch.cat([h[:, :9].reshape(-1, 3, 3), h[:, 9:].reshape(-1, 3, 1)], 2)


# ----------------------------------------------------------------------------------------------- W1 composition
COMPOSE_CASES = [(V, kind) for kind in ("dtu", "tt") for V in (2, 5, 20, 64)] + [(5, "synth")]


@pytest.mark.parametrize("V,kind", COMPOSE_CASES)
def test_compose_geometry(dev, V, kind):
    """every homography element and K^-1 entry within one fp32 ulp of fp64 (plus 1e-14 of its row's largest entry)"""
    if kind == "synth":
        pm = synth.make_proj_matrices(V, *G.DTU)["stage3"][0]
    else:
        pm = G.ring_cameras(V, *(G.DTU if kind == "dtu" else G.TT), kind, seed=V)
    homs, kinv = _nan(V - 1, 12), _nan(9)
    pmd = pm.to(dev)
    _lib.call("mvsf_compose_geometry", pmd, V, homs, kinv)
    want_h, want_k = G.compose64(pm)
    e_h = G.ulp_ratio(_rows34(homs.cpu()), _rows34(want_h), 4)
    e_k = G.ulp_ratio(kinv.cpu(), want_k, 3)
    rec(f"geometry_compose_V{V}_{kind}", homs_ulp_ratio=e_h, kinv_ulp_ratio=e_k)
    assert e_h <= 1.0 and e_k <= 1.0, (e_h, e_k)


@pytest.mark.parametrize("B", [1, 33, 70])
def test_homography_from_proj(dev, B):
    """src_proj @ inverse(ref_proj) per batch item within one fp32 ulp of fp64, every item written (the output is
    prefilled with a finite sentinel, so that the NaN of a singular item is the kernel's); an item with a zero row in
    ref_proj (the middle one) is all NaN and leaves the others as they are"""
    src, ref = [], []
    for b in range(B):
        pm = G.ring_cameras(2, *G.TT, "tt" if b % 2 else "dtu", seed=100 + b).double()
        P = pm[:, 0].clone()
        P[:, :3, :4] = pm[:, 1, :3, :3] @ pm[:, 0, :3, :4]
        ref.append(P[0])
        src.append(P[1])
    src, ref = torch.stack(src).float(), torch.stack(ref).float()
    sing = B // 2 if B > 1 else None
    if sing is not None:
        ref[sing, 2] = 0.0
    homs = torch.full((B, 12), -7.0, device=dev)
    sd, rd = src.to(dev), ref.to(dev)
    _lib.call("mvsf_homography_from_proj", sd, rd, B, homs)
    want = G.homography64(src, ref)
    got = homs.cpu()
    ok = torch.ones(B, dtype=torch.bool)
    if sing is not None:
        ok[sing] = False
        assert torch.isnan(got[sing]).all()
    e = G.ulp_ratio(_rows34(got[ok]), _rows34(want[ok]), 4)
    rec(f"geometry_homography_from_proj_B{B}", ulp_ratio=e)
    assert e <= 1.0, e


# ----------------------------------------------------------------------------------------------- F5 / F6 scheduling
INIT_SIZES = [(144, 192, G.DTU_RANGE), (136, 240, G.TT_RANGE), (37, 53, G.WIDE_RANGE)]


@pytest.mark.parametrize("Dn", [2, 192])
@pytest.mark.parametrize("D", [2, 4, 16, 32, 48])
def test_init_inverse_range(dev, D, Dn):
    """the first stage's planes at the DTU and T&T stage-1 sizes and at 37 x 53 (H W % 256 != 0), in inverse space"""
    for H, W, (lo, hi) in INIT_SIZES:
        dv = G.depth_values(lo, hi, Dn)
        out = _nan(D, H, W)
        dvd = dv.to(dev)
        _lib.call("mvsf_init_inverse_range", dvd, Dn, out, D, H, W)
        want = G.init_inv64(dvd, D).view(D, 1, 1).expand(D, H, W)
        e_inv, e_out, flips = G.inverse_error(out, want, G.INIT_TOL)
        rec(f"geometry_init_D{D}_Dn{Dn}_{H}x{W}", inv=e_inv, out_over_bound=e_out, sign_flips=flips)
        assert e_inv <= G.INIT_TOL and e_out <= 1.0 and flips == 0, (H, W, e_inv, e_out, flips)


def _schedule(dev, depth, prev, D, ratio, H, W):
    out = _nan(D, H, W)
    _lib.call("mvsf_schedule_inverse_range", depth, prev, prev.shape[0], G.f32(ratio), out, D, H, W)
    want = G.schedule_inv64(depth, prev, D, ratio, H, W)
    return out, want


@pytest.mark.parametrize("full,wide", [(G.DTU, False), (G.TT, False), (G.TT, True)], ids=["dtu", "tt", "tt_wide"])
def test_schedule_inverse_range_cascade(dev, full, wide):
    """stages 2-4 with the shipped (D, ratio) pairs, each fed the previous stage's planes as the library made them and a
    depth map drawn from them: W = 384 ... 1920, i.e. 3 to 15 column blocks.  The wide range drives 1/depth - 2.67 itv
    below 0 at far pixels, so the planes hold negative and huge hypotheses there"""
    dv, stage_depth = G.cascade_inputs(full, wide, seed=full[1] + wide)
    H, W = G.stage_size(full, 1)
    prev = _nan(G.NDEPTHS[0], H, W)
    dvd = dv.to(dev)
    _lib.call("mvsf_init_inverse_range", dvd, dv.numel(), prev, G.NDEPTHS[0], H, W)
    for s in (2, 3, 4):
        H, W = G.stage_size(full, s)
        D, ratio = G.NDEPTHS[s - 1], G.RATIOS[s - 1]
        depth = stage_depth(prev)
        out, want = _schedule(dev, depth, prev, D, ratio, H, W)
        e_inv, e_out, flips = G.inverse_error(out, want, G.INV_TOL)
        neg = int((want < 0).sum())
        rec(f"geometry_schedule_{'wide_' if wide else ''}{H}x{W}_D{D}", inv=e_inv, out_over_bound=e_out,
            sign_flips=flips, negative=neg)
        assert e_inv <= G.INV_TOL and e_out <= 1.0 and flips == 0, (s, e_inv, e_out, flips)
        if wide and s == 2:
            assert neg > 0
        prev = out


# H = W = 2 (one source pixel), odd half sizes, W % 128 != 0, and the 12 x 20 -> 24 x 40 step of a toy cascade
@pytest.mark.parametrize("H,W", [(2, 2), (74, 106), (6, 130), (24, 40), (258, 386)])
@pytest.mark.parametrize("D,ratio", [(16, 2.67), (8, 1.5), (4, 1.0)])
def test_schedule_inverse_range_edges(dev, H, W, D, ratio):
    dv, stage_depth = G.cascade_inputs(G.DTU, False, seed=H * W + D)
    h, w = H // 2, W // 2
    prev = _nan(G.NDEPTHS[0], h, w)
    dvd = dv.to(dev)
    _lib.call("mvsf_init_inverse_range", dvd, dv.numel(), prev, G.NDEPTHS[0], h, w)
    g = torch.Generator().manual_seed(D)
    prev = (prev * (1 + 0.01 * torch.rand(prev.shape, generator=g)).to(dev)).contiguous()   # per-pixel planes
    depth = stage_depth(prev)
    out, want = _schedule(dev, depth, prev, D, ratio, H, W)
    e_inv, e_out, flips = G.inverse_error(out, want, G.INV_TOL)
    rec(f"geometry_schedule_{H}x{W}_D{D}", inv=e_inv, out_over_bound=e_out, sign_flips=flips)
    assert e_inv <= G.INV_TOL and e_out <= 1.0 and flips == 0, (e_inv, e_out, flips)


# ----------------------------------------------------------------------------------------------- F7 3-D positions
# (B, H, W, D, camera kind, wide range): the DTU and T&T stage-1 sizes, and odd sizes whose D H W is no multiple of 256
POS_CASES = [(1, 144, 192, 32, "dtu", False), (2, 144, 192, 32, "dtu", False), (3, 144, 192, 32, "dtu", True),
             (1, 136, 240, 32, "tt", True), (2, 136, 240, 32, "tt", True), (3, 136, 240, 32, "tt", False),
             (3, 137, 239, 32, "tt", False), (2, 75, 243, 48, "dtu", False)]


def _kinvs(dev, pm):
    B, V = pm.shape[:2]
    kinvs, homs = _nan(B, 9), _nan(V - 1, 12)
    for b in range(B):
        _lib.call("mvsf_compose_geometry", pm[b], V, homs, kinvs[b])
    return kinvs


@pytest.mark.parametrize("B,H,W,D,kind,wide", POS_CASES)
def test_position3d_batched(dev, B, H, W, D, kind, wide):
    """the call sequence of hotpath.cascade_forward: mode 2 on sample 0, mode 3 on each further sample, mode 4 over the
    B x 192 depth values, mode 5 per sample.  The decoded extents and depth range equal the restatement bit for bit; the
    positions match fp64.  Each extreme comes from a chosen sample, the x / y ones from beyond the first grid-stride trip"""
    trips, stride = G.minmax_trips(D, H, W, _sms())
    assert trips >= 2, trips
    pm, hyp, dvs, owners = G.position_case(B, H, W, D, kind, wide, seed=7 * B + H)
    pm, hyp, dvs = pm.to(dev), hyp.to(dev), dvs.contiguous().to(dev)
    kinvs = _kinvs(dev, pm)
    stats = _nan(8)
    for b in range(B):
        _lib.call("mvsf_position3d", kinvs[b], hyp[b], None, 0, stats, 2 if b == 0 else 3, None, D, H, W)
    _lib.call("mvsf_position3d", None, None, dvs, dvs.numel(), stats, 4, None, D, H, W)
    pos = _nan(B, 3, D, H, W)
    for b in range(B):
        _lib.call("mvsf_position3d", kinvs[b], hyp[b], None, 0, stats, 5, pos[b], D, H, W)
    got_own = G.extreme_owners(kinvs, hyp, dvs)
    want_stats = torch.stack([*G.extents(kinvs, hyp), dvs.min(), dvs.max()])
    e = max(float((pos[b] - G.positions64(kinvs[b], hyp[b], stats[:6])).abs().max()) for b in range(B))
    neg = int((hyp < 0).sum())
    rec(f"geometry_position3d_B{B}_{H}x{W}_D{D}_{kind}{'_wide' if wide else ''}", abs=e, trips=trips, sms=_sms(),
        stats_equal=int(torch.equal(stats[:6], want_stats)), negative=neg)
    assert {k: b for k, (b, _) in got_own.items()} == owners, got_own
    assert all(got_own[k][1] >= stride for k in ("xmin", "xmax", "ymin", "ymax")), (got_own, stride)
    assert torch.equal(stats[:6], want_stats), (stats[:6].tolist(), want_stats.tolist())
    assert e <= G.POS_TOL, e
    assert neg > 0 if wide else neg == 0


@pytest.mark.parametrize("H,W,D", [(144, 192, 32), (137, 239, 32), (12, 16, 8)])
def test_position3d_single(dev, H, W, D):
    """mode 1 (extents of one sample, its depth range, normalise) at the DTU stage-1 size, an odd size and a toy size"""
    pm, hyp, dvs, _ = G.position_case(1, H, W, D, "dtu", False, seed=H)
    pm, hyp, dv = pm.to(dev), hyp.to(dev), dvs[0].contiguous().to(dev)
    kinvs = _kinvs(dev, pm)
    stats, pos = _nan(8), _nan(3, D, H, W)
    _lib.call("mvsf_position3d", kinvs[0], hyp[0], dv, dv.numel(), stats, 1, pos, D, H, W)
    want_stats = torch.stack([*G.extents(kinvs, hyp), dv.min(), dv.max()])
    e = float((pos - G.positions64(kinvs[0], hyp[0], stats[:6])).abs().max())
    rec(f"geometry_position3d_mode1_{H}x{W}_D{D}", abs=e, trips=G.minmax_trips(D, H, W, _sms())[0])
    assert torch.equal(stats[:6], want_stats), (stats[:6].tolist(), want_stats.tolist())
    assert e <= G.POS_TOL, e


# ----------------------------------------------------------------------------------------------- S1 soft-argmax
# (D, tmp, H, W, wide hypotheses): the shipped (D, tmp) at every DTU and T&T stage size; the templated D with the other
# temperature, the generic D = 2, 3, 48, 96 and negative temperatures at 37 x 53 (H W % 256 != 0); the generic D at a
# stage-1 size; the 9 x 21 toy cases
SA_CASES = ([(G.NDEPTHS[s - 1], G.TMP[s - 1], *G.stage_size(full, s), full == G.TT and s == 2)
             for s in (1, 2, 3, 4) for full in (G.DTU, G.TT)] +
            [(D, 6.0 - G.TMP[i], 37, 53, False) for i, D in enumerate(G.NDEPTHS)] +
            [(D, t, 37, 53, D == 3) for D in (2, 3, 48, 96) for t in (5.0, 1.0)] +
            [(8, -1.0, 37, 53, False), (3, -1.0, 37, 53, False), (48, 5.0, 136, 240, True), (96, 5.0, 144, 192, False)] +
            [(D, 5.0, 9, 21, False) for D in (4, 8, 16, 32, 5)])


@pytest.mark.parametrize("D,tmp,H,W,wide", SA_CASES)
def test_softargmax(dev, D, tmp, H, W, wide):
    """probability and confidence against fp64 (absolute), depth against fp64 relative to sum_d w_d |hypo_d|; conf is
    the max of the kernel's own prob bit for bit, and flat pixels give exactly 1/D"""
    z, flat = G.softargmax_logits(D, H, W, seed=D * 1000 + H)
    hyp = G.wide_planes(H, W, D, seed=D) if wide else G.narrow_planes(D, H, W, seed=D)
    zd, hd = z.to(dev), hyp.to(dev)
    prob, depth, conf = _nan(D, H, W), _nan(H, W), _nan(H, W)
    _lib.call("mvsf_softargmax", zd, hd, float(tmp), prob, depth, conf, D, H, W)
    p64, c64, d64, scale = G.softargmax64(zd, hd, tmp)
    e = dict(prob=float((prob - p64).abs().max()), conf=float((conf - c64).abs().max()),
             depth_rel=float(((depth - d64).abs() / scale).max()))
    inv_d = torch.tensor(1.0, device=dev) / torch.tensor(float(D), device=dev)
    fl = flat.to(dev)
    rec(f"geometry_softargmax_D{D}_tmp{tmp:g}_{H}x{W}{'_wide' if wide else ''}", **e)
    assert torch.equal(conf, prob.max(0).values)
    assert bool((prob[:, fl] == inv_d).all()) and bool((conf[fl] == inv_d).all())
    assert e["prob"] <= G.prob_tol(D) and e["conf"] <= G.prob_tol(D) and e["depth_rel"] <= G.depth_tol(D), e


# ----------------------------------------------------------------------------------------------- S2 confidence
CONF_CASES = {"dtu": [G.stage_size(G.DTU, s) for s in (1, 2, 3, 4)], "tt": [G.stage_size(G.TT, s) for s in (1, 2, 3, 4)],
              "odd": [(37, 53), (50, 60), (73, 97), (100, 120)]}


@pytest.mark.parametrize("name", list(CONF_CASES))
def test_conf_accumulate(dev, name):
    """the four-stage average (init, then three accumulations, scale 0.25) into a NaN-filled map equals
    sum_s F.interpolate(conf_s, nearest) x 0.25 in fp32, in stage order, bit for bit"""
    sizes = CONF_CASES[name]
    Hf, Wf = sizes[-1]
    g = torch.Generator().manual_seed(Hf)
    confs = [torch.rand(h, w, generator=g) for h, w in sizes]
    acc = _nan(Hf, Wf)
    cd = [c.to(dev) for c in confs]
    for s, ((h, w), c) in enumerate(zip(sizes, cd)):
        _lib.call("mvsf_conf_accumulate", c, h, w, acc, Hf, Wf, 0.25, 1 if s == 0 else 0)
    want = G.confidence_average(confs, Hf, Wf)
    got = acc.cpu()
    rec(f"geometry_conf_accumulate_{name}", abs=float((got - want).abs().max()), differing=int((got != want).sum()))
    assert torch.equal(got, want)
