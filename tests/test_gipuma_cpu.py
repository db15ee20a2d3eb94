"""The gipuma fusion without a GPU: the torch restatement (oracle/gipuma.py) against the inputs the reference's own
probability_filter and mvsnet_to_gipuma_cam produced, its fp32 run against its fp64 run, the used marks, argument checks,
and the compile-time guard of the kernels."""
import re

import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import fusion as FU, synth
from oracle import gen_golden_gipuma as GG
from oracle import gipuma as OG
from tests.gipuma_common import MARGIN, load_fixture
from tests.ptxas_common import function_props, ptxas_report


def test_camera_table_matches_reference_P():
    scene, meta, z = load_fixture()
    P = torch.from_numpy(z["P"])
    got = OG.camera_table(scene["cams"])[:, :12].reshape(-1, 3, 4)
    ulp = torch.finfo(torch.float32).eps * P.float().abs().clamp_min(torch.finfo(torch.float32).tiny)
    assert bool(((got.double() - P).abs() <= ulp.double()).all()), "P differs from the reference's by more than fp32 rounding"
    # M^-1 and f b of the fp64 table
    t = OG.camera_table(scene["cams"], torch.float64)
    eye = torch.eye(3, dtype=torch.float64).expand(meta["N"], 3, 3)
    assert torch.allclose(t[:, 12:21].reshape(-1, 3, 3) @ P[:, :, :3], eye, atol=1e-9)
    K = scene["cams"][:, 1].double()
    assert torch.allclose(t[:, 21], K[:, 0, 0] / K[:, 2, 2] * 0.54)


def test_filtered_depths_equal_reference_probability_filter():
    scene, meta, z = load_fixture()
    D, _ = OG.filter_depths(scene["depths"], scene["confs"], meta["prob_threshold"])
    want = torch.from_numpy(z["filtered"])
    assert torch.equal(D.view(torch.int32), want.view(torch.int32))
    assert 0.3 < float((D > 0).float().mean()) < 0.95


def test_reference_reproduces_fixture():
    mods = GG.reference_gipuma_modules()
    if mods is None:
        pytest.skip("no reference sources")
    depths, conf_u8, cams, images = GG.scene()
    _, _, z = load_fixture()
    assert np.array_equal(depths, z["depths"]) and np.array_equal(conf_u8, z["conf_u8"]) and np.array_equal(cams, z["cams"])
    filtered, P = GG.reference_inputs(*mods, depths, conf_u8, cams, GG.CASE["prob_threshold"])
    assert np.array_equal(filtered, z["filtered"]) and np.array_equal(P, z["P"])


def test_fp32_oracle_vs_fp64_on_fixture():
    """every view from the fp32 run's used state: the emit decisions of the two precisions differ only where the fp64
    margin is < 1e-4, and both outcomes occur"""
    scene, meta, _ = load_fixture()
    D, rng = OG.filter_depths(scene["depths"], scene["confs"], meta["prob_threshold"])
    t32, t64 = OG.camera_table(scene["cams"]), OG.camera_table(scene["cams"], torch.float64)
    N, H, W = D.shape
    used = torch.zeros(N, H, W, dtype=torch.uint8)
    emitted = 0
    for r in range(N):
        a = OG.step(r, D, t32, scene["images"], used, meta["disp_threshold"], meta["num_consistent"], torch.float32, rng)
        b = OG.step(r, D, t64, scene["images"], used, meta["disp_threshold"], meta["num_consistent"], torch.float64, rng)
        dis = a["keep"] != b["keep"]
        assert not dis.any() or float(b["margin"][dis].max()) < MARGIN
        both = a["keep"] & b["keep"]
        assert float((a["xyz"].double()[both[a["keep"]]] - b["xyz"][both[b["keep"]]]).abs().max()) < 1e-3
        valid = (D[r] > 0) & (used[r] == 0)
        assert (valid & ~a["keep"]).any() or r == 0
        emitted += int(a["keep"].sum())
        used = a["used"]
    assert 0.1 < emitted / float((D > 0).sum()) < 0.9


def _plane_scene():
    """3 ring views of the noise-free synthetic surface at full confidence"""
    sc = synth.make_fusion_scene(3, 24, 40, seed=12)
    return sc["depth_true"], torch.ones_like(sc["confs"]), sc["cams"], sc["images"]


def test_used_marks_consume_later_views():
    d, c, cams, img = _plane_scene()
    D, _ = OG.filter_depths(d, c)
    t = OG.camera_table(cams)
    zero = torch.zeros(D.shape, dtype=torch.uint8)
    first = OG.step(0, D, t, img, zero, 0.01, 1)
    alone = OG.step(1, D, t, img, zero, 0.01, 1)
    after = OG.step(1, D, t, img, first["used"], 0.01, 1)
    assert first["used"][1].any() and first["used"][2].any() and not first["used"][0].any()
    assert int(after["keep"].sum()) < int(alone["keep"].sum())
    assert not (after["keep"] & first["used"][1].bool()).any()
    a = OG.fuse_scene(d, c, cams, img, disp_threshold=0.01, num_consistent=1)
    b = OG.fuse_scene(d, c, cams, img, disp_threshold=0.01, num_consistent=1, order=[1, 0, 2])
    assert len(a[0]) != len(b[0]) or not torch.equal(a[0], b[0])


def test_argument_errors():
    sc = synth.make_fusion_scene(2, 8, 8)
    args = (sc["depths"], sc["confs"], sc["cams"], sc["images"])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        FU.fuse_scene_gipuma(*args)
    for kw in (dict(num_consistent=-1), dict(num_consistent=2.5), dict(depth_min=0.0), dict(depth_min=-1.0),
               dict(prob_threshold=float("nan")), dict(disp_threshold=float("inf")), dict(depth_max=float("nan"))):
        with pytest.raises(ValueError):
            FU.fuse_scene_gipuma(*args, **kw)


def test_gipuma_kernels_compile_without_spills():
    report = ptxas_report("fusion.cu")
    props = {f: (st, ld, r) for f, st, ld, r in function_props(report)}
    for k in ("gipuma_cameras_kernel", "gipuma_depth_kernel", "gipuma_vote_kernel", "gipuma_emit_kernel"):
        assert any(k in f for f in props), k
    for f, (st, ld, _) in props.items():
        assert not (st or ld) or "gipuma" not in f, f
    for k in ("gipuma_depth_kernel", "gipuma_vote_kernel", "gipuma_emit_kernel"):
        m = re.search(r"Function properties for (\w*" + k + r"\w*)\n\s*(\d+) bytes stack frame", report)
        assert m and int(m.group(2)) == 0, (k, m and m.group(2))
