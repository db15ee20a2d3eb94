"""Depth-map fusion without a GPU: the torch restatement (oracle/fusion.py) against fixtures the reference's own
misc/fusion.py produced, the PLY writer, the pair-file reader, and argument checks."""
import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import fusion as FU, synth
from oracle import fusion as OF
from oracle import gen_golden_fusion as GG
from tests.fusion_common import FIXTURES, MARGIN, check_view, fixture_view, load_fixture, scatter_points

CASES = [(n, m) for n in FIXTURES for m in ("pcd", "dpcd")]


@pytest.mark.parametrize("name,method", CASES)
def test_oracle_matches_reference_fixture(name, method):
    scene, meta, z = load_fixture(name)
    for r in meta["refs"]:
        mask, avg, pts = fixture_view(z, meta, method, r)
        got = check_view(mask, avg, r, scene["pairs"][r][1], scene, method, points=scatter_points(mask, pts))
        assert 0.05 < float(mask.float().mean()) < 0.95, "the fixture does not exercise both outcomes"
        assert got["disagree_fraction"] == 0.0 or got["worst_margin"] < MARGIN


@pytest.mark.parametrize("name,method", CASES)
def test_reference_arm_reproduces_golden_fixture(name, method):
    ref = GG.reference_fusion_module()
    if ref is None:
        pytest.skip("no reference sources (oracle/_ref/misc/fusion.py is made by build() only where the reference is available)")
    scene, meta, z = load_fixture(name)
    for r in meta["refs"]:
        with GG.on_cpu(), torch.no_grad():
            mask, avg, pts = GG.reference_filter(ref, method, r, scene["pairs"][r][1], scene["depths"], scene["confs"], scene["cams"])
        want_mask, want_avg, want_pts = fixture_view(z, meta, method, r)
        assert torch.equal(mask, want_mask)
        torch.testing.assert_close(avg, want_avg, rtol=1e-6, atol=0)
        torch.testing.assert_close(pts.permute(1, 2, 0)[mask], want_pts, rtol=0, atol=1e-3)


def test_scene_is_seeded_and_damaged():
    a, b = synth.make_fusion_scene(4, 24, 40, seed=5), synth.make_fusion_scene(4, 24, 40, seed=5)
    assert all(torch.equal(a[k], b[k]) for k in ("depths", "confs", "cams", "images")) and a["pairs"] == b["pairs"]
    assert (a["depths"] == 0).any() and (a["confs"] <= 0.5).any() and (a["confs"] > 0.5).any()
    assert torch.equal(a["images"], torch.round(a["images"] * 255) / 255)


def test_long_focal_view_leaves_the_image():
    # the last camera of the ring sees part of the scene: reprojections of the other views fall outside it
    sc = synth.make_fusion_scene(6, 40, 72)
    inv = OF.camera_inverses(sc["cams"], torch.float64)
    u, v = OF.pixel_centres(40, 72, torch.float64, "cpu")
    x, y, _ = OF.reproject(inv[0], sc["cams"][5].double(), u, v, sc["depth_true"][0].double())
    outside = (x < 0) | (x > 72) | (y < 0) | (y > 40)
    assert 0.1 < float(outside.float().mean()) < 0.9


def test_dpcd_single_source_accepts_nothing():
    sc = synth.make_fusion_scene(3, 16, 24)
    mask, avg, _ = OF.filter_view(0, [1], sc["depths"], sc["confs"], sc["cams"], "dpcd")
    assert not mask.any() and torch.equal(avg, sc["depths"][0])


def test_write_ply_round_trip(tmp_path):
    g = torch.Generator().manual_seed(1)
    xyz = torch.randn(37, 3, generator=g)
    rgb = torch.randint(0, 256, (37, 3), generator=g, dtype=torch.uint8)
    FU.write_ply(tmp_path / "a.ply", xyz, rgb)
    FU.write_ply(tmp_path / "b.ply", xyz.numpy(), rgb.numpy())
    raw = (tmp_path / "a.ply").read_bytes()
    assert raw == (tmp_path / "b.ply").read_bytes()
    head, payload = raw.split(b"end_header\n", 1)
    lines = head.decode("ascii").split("\n")
    assert lines[:3] == ["ply", "format binary_little_endian 1.0", "element vertex 37"]
    assert lines[3:9] == ["property float x", "property float y", "property float z", "property uchar red",
                          "property uchar green", "property uchar blue"]
    v = np.frombuffer(payload, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    assert len(payload) == 37 * 15 and len(v) == 37
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), xyz.numpy())
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), rgb.numpy())
    FU.write_ply(tmp_path / "empty.ply", torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.uint8))
    assert (tmp_path / "empty.ply").read_bytes().endswith(b"end_header\n")
    with pytest.raises(ValueError):
        FU.write_ply(tmp_path / "bad.ply", torch.zeros(4, 3), torch.zeros(5, 3, dtype=torch.uint8))


def test_read_pair_file(tmp_path):
    p = tmp_path / "pair.txt"
    p.write_text("3\n0\n3 1 2036.5 2 1696.2 7 10.0\n1\n0\n2\n2 0 5.0 1 4.0\n")
    assert FU.read_pair_file(p) == [(0, [1, 2, 7]), (2, [0, 1])]   # a view without sources is dropped


def test_argument_errors():
    d, c, k = torch.zeros(3, 8, 8), torch.zeros(3, 8, 8), torch.zeros(3, 2, 4, 4)
    with pytest.raises(ValueError, match="method"):
        FU.filter_view(0, [1], d, c, k, "gipuma")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        FU.filter_view(0, [1], d, c, k, "pcd")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        FU.fuse_scene(d, c, k, torch.zeros(3, 3, 8, 8), [(0, [1])], "dpcd")

