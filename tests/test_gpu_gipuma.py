"""GPU tests of the gipuma fusion (csrc/fusion.cu gipuma_*, fusion.gipuma_step / fuse_scene_gipuma) against the torch
restatement oracle/gipuma.py on the host.

Every reference view is checked from the same used state: the device's used marks are copied before the step, the step
runs once on the device and once in the fp32 oracle on the device's own filtered depths and camera table, and
tests/gipuma_common.compare_step applies the rule (decisions differ only at fp64 margin < 1e-4, on < 1e-3 of the pixels;
used marks only where such a decision lands; points to 1e-3, colours exactly)."""
import ctypes

import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import _lib, fusion as FU, synth
from oracle import gipuma as OG
from tests.common import rec
from tests.gipuma_common import compare_step, load_fixture, oracle_steps

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _on(dev, *ts):
    return [t.to(dev).contiguous() for t in ts]


def _steps_vs_oracle(dev, depths, confs, cams, images, disp, nc, prob=0.5):
    d, c, k, img = _on(dev, depths, confs, cams, images)
    scene = FU.gipuma_prepare(d, c, k, img, prob)
    D, rng = OG.filter_depths(depths, confs, prob)
    assert torch.equal(scene.depth.cpu().view(torch.int32), D.view(torch.int32)), "filtered depths differ from the oracle"
    table = scene.cams.cpu()
    t64 = OG.camera_table(cams, torch.float64)
    scale = t64.abs().amax(1, keepdim=True)
    assert float(((table.double() - t64).abs() / scale)[:, :22].max()) < 1e-6
    N = depths.shape[0]
    stats = []
    for r in range(N):
        before = scene.used.cpu()
        xyz, rgb = FU.gipuma_step(scene, r, disp, nc)
        want, truth = oracle_steps(r, D, table, cams, images, before, disp, nc, rng)
        stats.append(compare_step(scene.mask.cpu().bool(), xyz.cpu(), rgb.cpu(), scene.used.cpu(), want, truth))
    return stats


def _summary(name, stats):
    rec(name, worst_disagree=max(s["disagree"] for s in stats), used_disagree=sum(s["used_disagree"] for s in stats),
        worst_xyz=max(s["xyz_err"] for s in stats), points=sum(s["points"] for s in stats))


def test_steps_vs_oracle_fixture(dev):
    scene, meta, _ = load_fixture()
    stats = _steps_vs_oracle(dev, scene["depths"], scene["confs"], scene["cams"], scene["images"], meta["disp_threshold"],
                             meta["num_consistent"])
    _summary("gipuma_fixture", stats)
    assert sum(s["points"] for s in stats) > 1000


@pytest.mark.parametrize("N,H,W,nc", [(1, 19, 33, 0), (3, 27, 45, 1), (17, 23, 37, 3)])
def test_steps_vs_oracle_odd_sizes(dev, N, H, W, nc):
    sc = synth.make_fusion_scene(N, H, W, seed=100 + N)
    stats = _steps_vs_oracle(dev, sc["depths"], sc["confs"], sc["cams"], sc["images"], 0.0015 * W / 72, nc)
    _summary(f"gipuma_{N}x{H}x{W}", stats)
    assert sum(s["points"] for s in stats) > 0


def test_steps_vs_oracle_full_size(dev):
    sc = synth.make_fusion_scene(5, 1152, 1536, seed=105)
    stats = _steps_vs_oracle(dev, sc["depths"], sc["confs"], sc["cams"], sc["images"], 0.03, 2)
    _summary("gipuma_5x1152x1536", stats)
    assert sum(s["points"] for s in stats) > 100000


def test_scene_is_its_steps_and_deterministic(dev):
    scene, meta, _ = load_fixture()
    d, c, k, img = _on(dev, scene["depths"], scene["confs"], scene["cams"], scene["images"])
    kw = dict(disp_threshold=meta["disp_threshold"], num_consistent=meta["num_consistent"])
    xyz, rgb = FU.fuse_scene_gipuma(d, c, k, img, **kw)
    st = FU.gipuma_prepare(d, c, k, img)
    parts = [FU.gipuma_step(st, r, **kw) for r in range(meta["N"])]
    assert torch.equal(xyz, torch.cat([p[0] for p in parts])) and torch.equal(rgb, torch.cat([p[1] for p in parts]))
    xyz2, rgb2 = FU.fuse_scene_gipuma(d, c, k, img, **kw)
    assert torch.equal(xyz.view(torch.int32), xyz2.view(torch.int32)) and torch.equal(rgb, rgb2)
    assert xyz.dtype == torch.float32 and rgb.dtype == torch.uint8 and xyz.shape == rgb.shape and xyz.shape[1] == 3


def test_order_colours_and_ply(dev, tmp_path):
    """no source is ever consistent (negative disparity threshold) and num_consistent = 0: every valid pixel emits itself,
    so index-coded colours spell each point's pixel; views in index order, pixels row-major, xyz the pixel's world point"""
    scene, meta, _ = load_fixture()
    N, H, W = meta["N"], meta["H"], meta["W"]
    idx = torch.arange(H * W).view(H, W)
    coded = (torch.stack([(idx >> (8 * k)) & 255 for k in range(3)]).float() / 255.0).expand(N, 3, H, W).contiguous()
    d, c, k, img = _on(dev, scene["depths"], scene["confs"], scene["cams"], coded)
    xyz, rgb = FU.fuse_scene_gipuma(d, c, k, img, disp_threshold=-1.0, num_consistent=0)
    D, _ = OG.filter_depths(scene["depths"], scene["confs"])
    flat = torch.nonzero((D > 0).reshape(-1)).squeeze(1)
    assert len(rgb) == len(flat)
    pixel = (rgb.long().cpu() * torch.tensor([1, 256, 65536])).sum(1)
    assert torch.equal(pixel, flat % (H * W)), "points are not in view order / row-major pixel order"
    want, _, want_flat, _ = OG.fuse_scene(scene["depths"], scene["confs"], scene["cams"], coded, disp_threshold=-1.0,
                                          num_consistent=0)
    assert torch.equal(want_flat, flat) and float((xyz.cpu() - want).abs().max()) < 1e-3
    FU.write_ply(tmp_path / "g.ply", xyz, rgb)
    raw = (tmp_path / "g.ply").read_bytes()
    v = np.frombuffer(raw.split(b"end_header\n", 1)[1], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), xyz.cpu().numpy())
    assert np.array_equal(np.stack([v["r"], v["g"], v["b"]], 1), rgb.cpu().numpy())


def test_edge_cases(dev):
    scene, meta, _ = load_fixture()
    d, c, k, img = _on(dev, scene["depths"], scene["confs"], scene["cams"], scene["images"])
    xyz, rgb = FU.fuse_scene_gipuma(d, c, k, img, prob_threshold=1.0)
    assert xyz.shape == (0, 3) and rgb.shape == (0, 3)
    # num_consistent = 0: every valid pixel the earlier views left unused emits
    st = FU.gipuma_prepare(d, c, k, img)
    for r in range(meta["N"]):
        before = st.used[r].clone()
        xyz, _ = FU.gipuma_step(st, r, meta["disp_threshold"], 0)
        assert len(xyz) == int(((st.depth[r] > 0) & (before == 0)).sum())
    # a non-default stream
    want = FU.fuse_scene_gipuma(d, c, k, img, disp_threshold=meta["disp_threshold"], num_consistent=meta["num_consistent"])
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        got = FU.fuse_scene_gipuma(d, c, k, img, disp_threshold=meta["disp_threshold"], num_consistent=meta["num_consistent"])
    stream.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_error_paths(dev):
    sc = synth.make_fusion_scene(3, 16, 24, seed=3)
    d, c, k, img = _on(dev, sc["depths"], sc["confs"], sc["cams"], sc["images"])
    with pytest.raises(ValueError, match="contiguous float32"):
        FU.fuse_scene_gipuma(d.transpose(1, 2), c, k, img)
    with pytest.raises(ValueError, match="do not match"):
        FU.fuse_scene_gipuma(d, c[:2].contiguous(), k, img)
    with pytest.raises(ValueError, match="images"):
        FU.fuse_scene_gipuma(d, c, k, img[:, :, :8].contiguous())
    st = FU.gipuma_prepare(d, c, k, img)
    with pytest.raises(ValueError, match="outside the scene"):
        FU.gipuma_step(st, 3)
    # the C ABI reports the same conditions as status codes with a message
    L = _lib.lib()
    ws = st.ws.data_ptr()
    args = [st.depth.data_ptr(), st.used.data_ptr(), st.cams.data_ptr(), 3]
    assert L.mvsf_fusion_gipuma_vote(*args, 3, 16, 24, ctypes.c_float(0.2), 1, st.mask.data_ptr(), ws, 32, None) == -1
    assert b"reference view" in L.mvsf_last_error()
    assert L.mvsf_fusion_gipuma_vote(*args, 0, 16, 24, ctypes.c_float(0.2), -1, st.mask.data_ptr(), ws, 32, None) == -1
    assert L.mvsf_fusion_gipuma_vote(*args, 0, 16, 24, ctypes.c_float(0.2), 1, st.mask.data_ptr(), ws, 4, None) == -3
    assert L.mvsf_fusion_gipuma_emit(st.depth.data_ptr(), st.cams.data_ptr(), img.data_ptr(), 3, 0, 16, 24,
                                     ctypes.c_float(0.2), st.mask.data_ptr(), ws, 4, st.used.data_ptr(), None, None, 0,
                                     None) == -3
    torch.cuda.synchronize()
