"""GPU tests of the depth-map fusion (csrc/fusion.cu, mvsformerplusplus_b200/fusion.py) through the C ABI and through
fuse_scene, against the reference-executed fixtures and the torch restatement oracle/fusion.py on the host.

The mask rule (tests/fusion_common.check_view): a pixel may disagree with the fp32 oracle only where the fp64 oracle puts
one of the pixel's comparisons within 1e-4 relative of its threshold, and fewer than 1e-3 of a view's pixels may do so.
Both numbers go to parity_report.json."""
import ctypes

import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import _lib, fusion as FU, synth
from oracle import fusion as OF
from tests.common import TMP, rec
from tests.fusion_common import FIXTURES, MARGIN, check_view, fixture_view, load_fixture, scatter_points

pytestmark = pytest.mark.gpu
METHODS = ("pcd", "dpcd")


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _dev_scene(scene, dev):
    """the scene on the device; scene["inv"] becomes the kernels' camera inverses (host copy), which check_view hands to
    the fp32 oracle"""
    sc = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in scene.items()}
    scene["inv"] = FU._prepare_cameras(sc["cams"]).cpu()
    return sc


def test_camera_inverses(dev):
    cams = synth.make_fusion_scene(17, 8, 8)["cams"]
    got = FU._prepare_cameras(cams.to(dev)).cpu()
    want = OF.camera_inverses(cams, torch.float64)
    assert float(((got.double() - want).abs() / want.abs().amax(dim=(2, 3), keepdim=True)).max()) < 1e-7


def abi_view(sc, ref, srcs, method, thr=(0.5, 2.0, 1.0, 4.0, 1300.0)):
    """one reference view through the four C entry points -> mask bool [H,W], averaged depth, xyz [M,3], rgb [M,3]"""
    d, c, k, img = sc["depths"], sc["confs"], sc["cams"], sc["images"]
    N, H, W = d.shape
    nbytes = _lib.size("mvsf_fusion_workspace_bytes", H, W)
    assert nbytes == 4 * ((H * W + 255) // 256 + 1)
    ws = torch.empty(nbytes // 4, dtype=torch.int32, device=d.device)
    inv = torch.empty_like(k)
    _lib.call("mvsf_fusion_prepare_cameras", k, N, inv)
    mask = torch.empty(H, W, dtype=torch.uint8, device=d.device)
    avg = torch.empty(H, W, dtype=torch.float32, device=d.device)
    idx = (ctypes.c_int * len(srcs))(*srcs)
    _lib.call("mvsf_fusion_filter", FU.METHODS[method], d, c, k, inv, N, ref, idx, len(srcs), H, W, *thr, mask, avg, ws, nbytes)
    M = int(ws[-1])
    assert M == int(mask.sum())
    xyz = torch.full((M + 1, 3), -7.0, device=d.device)      # one row of room more than the survivors: it must stay untouched
    rgb = torch.full((M + 1, 3), 9, dtype=torch.uint8, device=d.device)
    _lib.call("mvsf_fusion_extract", mask, avg, ws, nbytes, inv[ref], img[ref], xyz, rgb, M, H, W)
    assert bool((xyz[M] == -7.0).all()) and bool((rgb[M] == 9).all())
    return mask.bool(), avg, xyz[:M], rgb[:M]


def expected_rgb(images, ref, mask):
    return (images[ref] * 255).permute(1, 2, 0)[mask.cpu()].to(torch.uint8)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name", FIXTURES)
def test_abi_vs_reference_fixture(dev, name, method):
    scene, meta, z = load_fixture(name)
    sc = _dev_scene(scene, dev)
    for r in meta["refs"]:
        srcs = scene["pairs"][r][1]
        mask, avg, xyz, rgb = abi_view(sc, r, srcs, method)
        got = check_view(mask, avg, r, srcs, scene, method, points=scatter_points(mask, xyz), inv=scene["inv"])
        want_mask, want_avg, want_pts = fixture_view(z, meta, method, r)
        _, _, margin = OF.filter_view(r, srcs, scene["depths"], scene["confs"], scene["cams"], method, dtype=torch.float64)
        bad = mask.cpu() != want_mask
        assert not bad.any() or float(margin[bad].max()) < MARGIN
        both = mask.cpu() & want_mask
        assert float((scatter_points(mask, xyz) - scatter_points(want_mask, want_pts))[both].abs().max()) < 1e-3
        assert torch.equal(rgb.cpu(), expected_rgb(scene["images"], r, mask))
        rec(f"fusion_fixture_{name}_{method}_ref{r}", fixture_disagree=float(bad.float().mean()), **got)


@pytest.mark.parametrize("V", [1, 2, 4, 10, 16])
@pytest.mark.parametrize("method", METHODS)
def test_odd_sizes_and_source_counts(dev, method, V):
    H, W = (37, 53) if V % 4 else (45, 31)
    scene = synth.make_fusion_scene(V + 1, H, W, seed=100 + V, n_src=V)
    sc = _dev_scene(scene, dev)
    for r in (0, V):
        srcs = scene["pairs"][r][1]
        assert len(srcs) == V
        mask, avg, xyz, rgb = abi_view(sc, r, srcs, method)
        got = check_view(mask, avg, r, srcs, scene, method, points=scatter_points(mask, xyz), inv=scene["inv"])
        m2, a2 = FU.filter_view(r, srcs, sc["depths"], sc["confs"], sc["cams"], method)
        assert torch.equal(m2, mask) and torch.equal(a2, avg)
        assert torch.equal(rgb.cpu(), expected_rgb(scene["images"], r, mask))
        rec(f"fusion_{method}_v{V}_{H}x{W}_ref{r}", kept=float(mask.float().mean()), **got)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("name,n_src,H,W", [("dtu", 4, 1152, 1536), ("tt", 10, 1088, 1920)])
def test_full_size(dev, name, n_src, H, W, method):
    scene = synth.make_fusion_scene(n_src + 1, H, W, seed=7, n_src=n_src)
    sc = _dev_scene(scene, dev)
    r, srcs = scene["pairs"][1]
    mask, avg = FU.filter_view(r, srcs, sc["depths"], sc["confs"], sc["cams"], method)
    xyz, rgb = FU.fuse_scene(sc["depths"], sc["confs"], sc["cams"], sc["images"], [(r, srcs)], method)
    assert xyz.shape[0] == int(mask.sum())
    got = check_view(mask, avg, r, srcs, scene, method, points=scatter_points(mask, xyz), inv=scene["inv"])
    assert torch.equal(rgb.cpu(), expected_rgb(scene["images"], r, mask))
    rec(f"fusion_fullsize_{name}_{method}", kept=float(mask.float().mean()), **got)


def _index_images(N, H, W, dev):
    """images whose colour bytes spell the flat pixel index: channel k holds byte k of the index, at (byte + 0.5) / 255"""
    idx = torch.arange(H * W).view(H, W)
    img = torch.stack([(idx >> (8 * k)) & 255 for k in range(3)]).float()
    return ((img + 0.5) / 255.0).expand(N, 3, H, W).contiguous().to(dev)


@pytest.mark.parametrize("method", METHODS)
def test_scene_order_colours_and_ply(dev, method, tmp_path):
    """fuse_scene over a pair list in which every view is a reference view and a source view: views in pair order, pixels
    row-major (the flat pixel index of every point is compared), colours exact, the PLY byte-identical between two runs."""
    scene, meta, _ = load_fixture("fusion_n6_40x72")
    sc = _dev_scene(scene, dev)
    H, W = meta["H"], meta["W"]
    pairs = [scene["pairs"][i] for i in (3, 0, 5, 1, 2, 4)]
    xyz, rgb = FU.fuse_scene(sc["depths"], sc["confs"], sc["cams"], sc["images"], pairs, method)
    _, coded = FU.fuse_scene(sc["depths"], sc["confs"], sc["cams"], _index_images(6, H, W, dev), pairs, method)
    pixel = (coded.long() * torch.tensor([1, 256, 65536], device=dev)).sum(1).cpu()
    want_xyz, want_rgb, want_flat = OF.fuse_scene(scene["depths"], scene["confs"], scene["cams"], scene["images"], pairs, method)
    masks = [FU.filter_view(r, s, sc["depths"], sc["confs"], sc["cams"], method)[0].cpu() for r, s in pairs]
    flat = torch.cat([torch.nonzero(m.reshape(-1)).squeeze(1) + k * H * W for k, m in enumerate(masks)])
    assert torch.equal(pixel, flat % (H * W)), "points are not in pair order / row-major pixel order"
    assert xyz.shape == (len(flat), 3) and rgb.shape == (len(flat), 3) and rgb.dtype == torch.uint8
    for (r, s), m in zip(pairs, masks):
        check_view(m, FU.filter_view(r, s, sc["depths"], sc["confs"], sc["cams"], method)[1], r, s, scene, method, inv=scene["inv"])
    common = torch.isin(flat, want_flat)
    theirs = torch.isin(want_flat, flat)
    assert float(common.float().mean()) > 0.999
    assert float((xyz.cpu()[common] - want_xyz[theirs]).abs().max()) < 1e-3
    assert torch.equal(rgb.cpu()[common], want_rgb[theirs])
    FU.write_ply(tmp_path / "a.ply", xyz, rgb)
    xyz2, rgb2 = FU.fuse_scene(sc["depths"], sc["confs"], sc["cams"], sc["images"], pairs, method)
    FU.write_ply(tmp_path / "b.ply", xyz2, rgb2)
    raw = (tmp_path / "a.ply").read_bytes()
    assert raw == (tmp_path / "b.ply").read_bytes()
    v = np.frombuffer(raw.split(b"end_header\n", 1)[1], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), xyz.cpu().numpy())
    rec(f"fusion_scene_{method}", points=len(flat), common_with_oracle=float(common.float().mean()))


@pytest.mark.parametrize("method", METHODS)
def test_all_rejected_and_all_accepted(dev, method):
    scene = synth.make_fusion_scene(3, 24, 40, seed=9, n_src=2)
    sc = _dev_scene(scene, dev)
    zero = torch.zeros_like(sc["confs"])
    xyz, rgb = FU.fuse_scene(sc["depths"], zero, sc["cams"], sc["images"], scene["pairs"], method)
    assert xyz.shape == (0, 3) and rgb.shape == (0, 3)
    # every view sees the true surface with full confidence; pcd with thres_view = 1 needs no consistent source at all,
    # dpcd is given thresholds no reprojection misses
    clean = torch.ones_like(sc["confs"])
    true = scene["depth_true"].to(dev)
    kw = dict(thres_view=1) if method == "pcd" else dict(dist_base=1e-6, rel_diff_base=1e-6)
    pairs = [(0, [1, 2]), (1, [0, 2])]
    xyz, rgb = FU.fuse_scene(true, clean, sc["cams"], sc["images"], pairs, method, **kw)
    assert xyz.shape == (2 * 24 * 40, 3)
    want = OF.view_points(0, OF.filter_view(0, [1, 2], scene["depth_true"], clean.cpu(), scene["cams"], method, inv=scene["inv"],
                                            **kw)[1], scene["cams"], inv=scene["inv"])
    assert float((xyz[:24 * 40].cpu() - want.reshape(-1, 3)).abs().max()) < 1e-3


def test_non_default_stream_and_views_without_copy(dev):
    scene = synth.make_fusion_scene(5, 40, 56, seed=11, n_src=3)
    sc = _dev_scene(scene, dev)
    want = FU.fuse_scene(sc["depths"], sc["confs"], sc["cams"], sc["images"], scene["pairs"], "dpcd")
    # the scene as views into larger buffers (what a model's batched output is): no copy is made, the result is the same
    big_d = torch.zeros(9, 40, 56, device=dev)
    big_c = torch.zeros(9, 40, 56, device=dev)
    big_d[2:7], big_c[2:7] = sc["depths"], sc["confs"]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        got = FU.fuse_scene(big_d[2:7], big_c[2:7], sc["cams"], sc["images"], scene["pairs"], "dpcd")
    stream.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_error_paths(dev):
    scene = synth.make_fusion_scene(3, 16, 24, seed=3, n_src=2)
    sc = _dev_scene(scene, dev)
    d, c, k, img = sc["depths"], sc["confs"], sc["cams"], sc["images"]
    with pytest.raises(ValueError, match="contiguous float32"):
        FU.filter_view(0, [1], d.transpose(1, 2), c.transpose(1, 2), k, "pcd")
    with pytest.raises(ValueError, match="contiguous float32"):
        FU.filter_view(0, [1], d.double(), c, k, "pcd")
    with pytest.raises(ValueError, match="source views"):
        FU.filter_view(0, [1] * 17, d, c, k, "dpcd")
    with pytest.raises(ValueError, match="source views"):
        FU.filter_view(0, [], d, c, k, "dpcd")
    with pytest.raises(ValueError, match="outside the scene"):
        FU.filter_view(0, [3], d, c, k, "pcd")
    with pytest.raises(ValueError, match="non-empty"):
        FU.filter_view(0, [1], d[:, :0], c[:, :0], k, "pcd")
    with pytest.raises(ValueError, match="images"):
        FU.fuse_scene(d, c, k, img[:, :, :8].contiguous(), scene["pairs"], "pcd")
    # the C ABI reports the same conditions as status codes with a message
    L = _lib.lib()
    ws = torch.empty(8, dtype=torch.int32, device=dev)
    mask, avg = torch.empty(16, 24, dtype=torch.uint8, device=dev), torch.empty(16, 24, device=dev)
    idx = (ctypes.c_int * 17)(*([1] * 17))
    thr = (0.5, 2.0, 1.0, 4.0, 1300.0)
    scene_ptrs = [t.data_ptr() for t in (d, c, k, k)]
    out_ptrs = [t.data_ptr() for t in (mask, avg, ws)]
    assert L.mvsf_fusion_filter(0, *scene_ptrs, 3, 0, idx, 17, 16, 24, *thr, *out_ptrs, 32, None) == -1
    assert b"source views" in L.mvsf_last_error()
    assert L.mvsf_fusion_filter(2, *scene_ptrs, 3, 0, idx, 1, 16, 24, *thr, *out_ptrs, 32, None) == -1
    assert L.mvsf_fusion_filter(0, *scene_ptrs, 3, 0, idx, 1, 16, 24, *thr, *out_ptrs, 4, None) == -3
    assert L.mvsf_fusion_filter(0, *scene_ptrs, 3, 0, idx, 1, 0, 24, *thr, *out_ptrs, 32, None) == -1


def test_model_to_point_cloud(dev):
    """DINOv2MVSNet on a 3-view synthetic set, each view once the reference view; its depth and confidence maps go to
    fuse_scene on the device."""
    from tests.model_common import CASES, cuda_model, make_inputs, model_state_dict
    meta = CASES["model_b1v3_96x128"]
    imgs, proj, dv = make_inputs(meta)
    net = cuda_model(model_state_dict(meta["wseed"]), dev)
    imgs, dv = imgs.to(dev), dv.to(dev)
    proj = {k: v.to(dev) for k, v in proj.items()}
    H, W = meta["H"], meta["W"]
    depths, confs = torch.empty(3, H, W, device=dev), torch.empty(3, H, W, device=dev)
    for r in range(3):
        order = [r] + [v for v in range(3) if v != r]
        out = net(imgs[:, order], {k: v[:, order] for k, v in proj.items()}, dv, TMP)
        depths[r], confs[r] = out["refined_depth"][0], out["photometric_confidence"][0]
    cams = proj["stage4"][0].contiguous()
    cams[:, 1, 3, 3] = 1.0
    colour = ((imgs[0] - imgs[0].amin()) / (imgs[0].amax() - imgs[0].amin())).contiguous()
    pairs = [(r, [v for v in range(3) if v != r]) for r in range(3)]
    conf = float(confs.median())   # seeded weights give no calibrated confidence: split the pixels in two
    for method in METHODS:
        xyz, rgb = FU.fuse_scene(depths, confs, cams, colour, pairs, method, conf=conf, thres_view=1, dist_base=0.01,
                                 rel_diff_base=1.0)
        scene = dict(depths=depths.cpu(), confs=confs.cpu(), cams=cams.cpu())
        inv = FU._prepare_cameras(cams).cpu()
        n = 0
        for r, s in pairs:
            mask, avg = FU.filter_view(r, s, depths, confs, cams, method, conf=conf, thres_view=1, dist_base=0.01, rel_diff_base=1.0)
            check_view(mask, avg, r, s, scene, method, inv=inv, conf=conf, **(dict(thres_view=1) if method == "pcd" else
                                                                     dict(dist_base=0.01, rel_diff_base=1.0)))
            n += int(mask.sum())
        assert xyz.shape[0] == n and 0 < n < 3 * H * W
        assert bool(torch.isfinite(xyz).all())
