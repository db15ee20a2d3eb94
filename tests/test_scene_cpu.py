"""CPU tests of scene preparation (mvsformerplusplus_b200/scene.py, oracle/image_prep.py) against the reference's own eval
loader and file writers, as the fixtures tests/golden/scene_*.npz hold them, and against cv2.resize where cv2 is
installed: everything bit for bit.  No GPU needed."""
import os

import numpy as np
import pytest

from mvsformerplusplus_b200 import scene as S
from oracle import image_prep as IP
from tests.scene_common import CASES, fixture, load_args, reference_item, write_folder

# (h, w) -> (H, W): DTU and its 864 x 1152 setting, T&T's 1080 -> 1024 and 1088 -> 1152 x 2048, upscales, odd widths,
# exact 2x, a tiny image and the identity
RESIZE_SIZES = [((1200, 1600), (1152, 1536)), ((1200, 1600), (864, 1152)), ((576, 768), (512, 640)),
                ((1080, 1920), (1024, 1920)), ((100, 130), (160, 224)), ((64, 64), (96, 97)), ((1088, 1920), (1152, 2048)),
                ((1200, 1600), (1150, 1001)), ((1200, 1600), (1152, 1537)), ((37, 53), (29, 41)), ((192, 256), (96, 128)),
                ((96, 128), (96, 128))]


def _images(case):
    blob, meta = fixture(case)
    return {v: blob[f"decoded_{v}"] for v in sorted({v for ids in meta["items"] for v in ids})}


@pytest.mark.parametrize("src,dst", RESIZE_SIZES)
def test_resize_oracle_equals_cv2(src, dst):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(src[0] * 7 + dst[1]).integers(0, 256, (*src, 3), dtype=np.uint8)
    assert np.array_equal(IP.resize_u8(img, *dst), cv2.resize(img, (dst[1], dst[0])))


@pytest.mark.parametrize("case", CASES)
def test_resize_oracle_equals_cv2_on_fixture(case):
    cv2 = pytest.importorskip("cv2")
    _, meta = fixture(case)
    pad = S.TT_PAD_ROWS if meta["dataset"] == "tt" else 0
    for img in _images(case).values():
        padded = np.pad(img, ((pad, pad), (0, 0), (0, 0)), "edge")
        want = cv2.resize(padded, (meta["max_w"], meta["max_h"]))
        assert np.array_equal(IP.resize_u8(img, meta["max_h"], meta["max_w"], pad), want)


@pytest.mark.parametrize("case", CASES)
def test_oracle_prepares_the_loaders_images(case):
    """pad + resize + ToTensor + Normalize of the oracle reproduce the loader's imgs bit for bit"""
    blob, meta = fixture(case)
    pad = S.TT_PAD_ROWS if meta["dataset"] == "tt" else 0
    for v, img in _images(case).items():
        x = IP.normalize(IP.resize_u8(img, meta["max_h"], meta["max_w"], pad))
        assert x.dtype == np.float32 and np.array_equal(x, blob[f"img_{v}"]), v


def test_fusion_colour_is_test_py_array():
    """trunc(clip((norm std + mean) 255)) / 255 as test.py:287-292 computes it from the model's input, read back as
    read_img does (float32 / 255)"""
    blob, _ = fixture("dtu")
    img = blob["img_0"]
    c = img * IP.STD.reshape(3, 1, 1) + IP.MEAN.reshape(3, 1, 1)
    want = np.clip(c.transpose(1, 2, 0) * 255, 0, 255).astype(np.uint8).astype(np.float32) / 255.
    u8 = IP.resize_u8(blob["decoded_0"], 96, 128)
    assert np.array_equal(IP.fusion_colour(u8), want.transpose(2, 0, 1))


@pytest.mark.parametrize("case", CASES)
def test_cameras_view_sets_and_depth_values_equal_the_loader(case, tmp_path):
    blob, meta = fixture(case)
    a = load_args(meta)
    plan = S.ScenePlan(write_folder(case, str(tmp_path)), a["scan"], a["dataset"], a["nviews"], a["use_short_range"])
    assert [[r] + s for r, s in plan.view_sets] == meta["items"]
    sizes = [blob[f"decoded_{v}"].shape[:2] for v in plan.view_ids]
    projs, dvals = plan.cameras(sizes, a["ndepths"], a["interval_scale"], a["max_h"], a["max_w"])
    for k in range(len(meta["items"])):
        _, proj, dv = reference_item(case, k)
        assert dvals[k].dtype == np.float32 and np.array_equal(dvals[k], dv), k
        for s, m in proj.items():
            assert projs[k][s].dtype == np.float32 and np.array_equal(projs[k][s], m), (k, s)


def test_view_sets_pad_and_truncate(tmp_path):
    p = tmp_path / "pair.txt"
    p.write_text("3\n0\n1 4 9.0\n1\n4 0 9.0 2 8.0 3 7.0 4 6.0\n2\n0\n")
    assert S.build_view_sets(str(p), 4) == [(0, [4, 4, 4]), (1, [0, 2, 3])]


@pytest.mark.parametrize("case", CASES)
def test_writers_reproduce_reference_bytes(case, tmp_path):
    blob, meta = fixture(case)
    S.save_pfm(str(tmp_path / "d.pfm"), blob["pfm_depth"])
    assert (tmp_path / "d.pfm").read_bytes() == blob["pfm_bytes"].tobytes()
    dv = blob["dv_0"]
    S.write_cam(str(tmp_path / "c.txt"), blob["proj_0_stage4"][0], (dv[0], dv[-1]) if meta["dataset"] == "tt" else None)
    assert (tmp_path / "c.txt").read_bytes() == blob["cam_bytes"].tobytes()


def test_load_scene_rejects_sizes_that_are_not_multiples_of_32(tmp_path):
    _, meta = fixture("dtu")
    a = load_args(meta)
    datapath = write_folder("dtu", str(tmp_path))
    for bad in (dict(max_h=100), dict(max_w=0), dict(max_h=96.5)):
        with pytest.raises(ValueError, match="multiple of 32"):
            S.load_scene(datapath, **dict(a, **bad))


def test_load_scene_names_a_missing_view(tmp_path):
    _, meta = fixture("eth3d")
    datapath = write_folder("eth3d", str(tmp_path))
    os.remove(os.path.join(datapath, meta["scan"], "images", "00000002.jpg"))
    with pytest.raises(FileNotFoundError, match="00000002.jpg"):
        S.load_scene(datapath, **load_args(meta))


def test_load_scene_rejects_a_cpu_device(tmp_path):
    _, meta = fixture("eth3d")
    with pytest.raises(RuntimeError, match="CUDA"):
        S.load_scene(write_folder("eth3d", str(tmp_path)), **load_args(meta), device="cpu")
