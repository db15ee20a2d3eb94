"""GPU tests of scene preparation and reconstruction (csrc/image_prep.cu, mvsformerplusplus_b200/scene.py), all bit for bit:
  * mvsf_image_resize_u8 against the oracle and cv2.resize, on the fixtures' decoded images and on random images;
  * load_scene + Scene.item(k) against every item of the reference's own loader (tests/golden/scene_*.npz);
  * reconstruct_scene against the composition a user writes today: DINOv2MVSNet on the loader's items, the confidence
    quantised in numpy as test.py does, then fuse_scene / fuse_scene_gipuma, and its out_dir files against the writers;
  * malformed input raises."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import _lib
from mvsformerplusplus_b200 import scene as S
from oracle import image_prep as IP
from tests.common import TMP
from tests.scene_common import CASES, fixture, load_args, reference_item, write_folder
from tests.test_scene_cpu import RESIZE_SIZES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _views(meta):
    return sorted({v for ids in meta["items"] for v in ids})


@pytest.mark.parametrize("case", CASES)
def test_resize_kernel_on_fixture(dev, case):
    blob, meta = fixture(case)
    pad = S.TT_PAD_ROWS if meta["dataset"] == "tt" else 0
    imgs = np.stack([blob[f"decoded_{v}"] for v in _views(meta)])
    got = S.resize_u8(torch.from_numpy(imgs).to(dev), meta["max_h"], meta["max_w"], pad).cpu().numpy()
    for n, img in enumerate(imgs):
        want = IP.resize_u8(img, meta["max_h"], meta["max_w"], pad)
        assert np.array_equal(got[n], want), n
        try:
            import cv2
        except ImportError:
            continue
        assert np.array_equal(got[n], cv2.resize(np.pad(img, ((pad, pad), (0, 0), (0, 0)), "edge"),
                                                 (meta["max_w"], meta["max_h"])))


@pytest.mark.parametrize("src,dst", RESIZE_SIZES)
@pytest.mark.parametrize("pad", [0, 4])
def test_resize_kernel_sizes(dev, src, dst, pad):
    imgs = np.random.default_rng(src[1] + dst[0] + pad).integers(0, 256, (2, *src, 3), dtype=np.uint8)
    got = S.resize_u8(torch.from_numpy(imgs).to(dev), *dst, pad_rows=pad).cpu().numpy()
    for n in range(2):
        assert np.array_equal(got[n], IP.resize_u8(imgs[n], *dst, pad)), n


@pytest.mark.parametrize("case", CASES)
def test_normalize_and_colour(dev, case):
    blob, meta = fixture(case)
    pad = S.TT_PAD_ROWS if meta["dataset"] == "tt" else 0
    u8 = np.stack([IP.resize_u8(blob[f"decoded_{v}"], meta["max_h"], meta["max_w"], pad) for v in _views(meta)])
    views = [len(u8) - 1, 0, 0]
    norm, colour = S.normalize(torch.from_numpy(u8).to(dev), views, norm=True, colour=True)
    assert np.array_equal(norm.cpu().numpy(), IP.normalize(u8[views]))
    assert np.array_equal(colour.cpu().numpy(), IP.fusion_colour(u8[views]))


@pytest.mark.parametrize("case", CASES)
def test_load_scene_items_equal_the_loader(dev, case, tmp_path):
    from PIL import Image
    blob, meta = fixture(case)
    datapath = write_folder(case, str(tmp_path))
    for v in _views(meta):   # a different libjpeg would show here, not as a kernel mismatch
        p = os.path.join(datapath, meta["scan"], "images", f"{v:08d}.jpg")
        assert np.array_equal(np.asarray(Image.open(p).convert("RGB")), blob[f"decoded_{v}"]), f"PIL decodes view {v} differently"
    sc = S.load_scene(datapath, **load_args(meta), device=dev)
    assert len(sc) == len(meta["items"])
    for k in range(len(sc)):
        imgs, proj, dv = sc.item(k)
        want_imgs, want_proj, want_dv = reference_item(case, k)
        assert imgs.dtype == torch.float32 and imgs.is_cuda and np.array_equal(imgs.cpu().numpy(), want_imgs[None]), k
        assert dv.is_cuda and np.array_equal(dv.cpu().numpy(), want_dv[None]), k
        for s, m in want_proj.items():
            assert proj[s].is_cuda and np.array_equal(proj[s].cpu().numpy(), m[None]), (k, s)


@pytest.fixture(scope="module")
def model(dev):
    from tests.model_common import cuda_model, model_state_dict
    return cuda_model(model_state_dict(401), dev)


def _composition(case, datapath, model, dev, method, conf_choose, combine, fusion_args):
    """what a user writes today: the model on the loader's items, test.py's numpy quantisation, then the fusion"""
    from mvsformerplusplus_b200.fusion import fuse_scene, fuse_scene_gipuma
    blob, meta = fixture(case)
    depths, confs, cams, colours = [], [], [], []
    for k in range(len(meta["items"])):
        imgs, proj, dv = reference_item(case, k)
        with torch.no_grad():
            out = model(torch.from_numpy(imgs)[None].to(dev), {s: torch.from_numpy(m)[None].to(dev) for s, m in proj.items()},
                        torch.from_numpy(dv)[None].to(dev), TMP)
        c = (out["photometric_confidence"] if conf_choose == "mean" else out["stage4"]["photometric_confidence"])[0].cpu().numpy()
        if combine:
            c = (c * 3 + out["stage4"]["photometric_confidence"][0].cpu().numpy()) / 4
        confs.append((c * 255).astype(np.uint8))
        depths.append(out["refined_depth"][0].cpu().numpy())
        cams.append(proj["stage4"][0])
        img = imgs[0] * IP.STD.reshape(3, 1, 1) + IP.MEAN.reshape(3, 1, 1)
        colours.append(np.clip(img * 255, 0, 255).astype(np.uint8).astype(np.float32) / 255.)
    cams_rb = np.stack(cams).copy()
    cams_rb[:, 1, 3, 3] = 1.0
    t = lambda x: torch.from_numpy(np.ascontiguousarray(np.stack(x) if isinstance(x, list) else x)).to(dev)  # noqa: E731
    conf = t([c.astype(np.float32) / 255 for c in confs])
    if method == "gipuma":
        xyz, rgb = fuse_scene_gipuma(t(depths), conf, t(cams_rb), t(colours), **fusion_args)
    else:
        item = {ids[0]: k for k, ids in enumerate(meta["items"])}
        from mvsformerplusplus_b200.fusion import read_pair_file
        pairs = []
        for ref, srcs in read_pair_file(os.path.join(datapath, meta["scan"], "pair.txt")):
            srcs = [item[s] for s in srcs if s in item]
            if ref in item and srcs:
                pairs.append((item[ref], srcs))
        xyz, rgb = fuse_scene(t(depths), conf, t(cams_rb), t(colours), pairs, method, **fusion_args)
    return xyz, rgb, depths, confs, cams


RECON = [("dtu", "pcd", "mean", False), ("dtu", "dpcd", "mean", False), ("dtu", "gipuma", "mean", False),
         ("tt_short_range", "pcd", "stage4", False), ("tt_short_range", "gipuma", "mean", True),
         ("eth3d", "dpcd", "stage4", True)]
# thresholds loose enough for random weights' depth maps to leave points
FUSION_ARGS = {"pcd": dict(conf=0.0, thres_view=1, thres_disp=100.0), "dpcd": dict(conf=0.0, dist_base=1e-3, rel_diff_base=1e-3),
               "gipuma": dict(prob_threshold=0.0, disp_threshold=10.0, num_consistent=1)}


@pytest.mark.parametrize("case,method,conf_choose,combine", RECON)
def test_reconstruct_scene_equals_composition(dev, model, case, method, conf_choose, combine, tmp_path):
    blob, meta = fixture(case)
    datapath = write_folder(case, str(tmp_path / "in"))
    xyz_w, rgb_w, depths, confs, cams = _composition(case, datapath, model, dev, method, conf_choose, combine,
                                                     FUSION_ARGS[method])
    sc = S.load_scene(datapath, **load_args(meta), device=dev)
    out_dir = str(tmp_path / "out")
    xyz, rgb = S.reconstruct_scene(model, sc, method, tmp=TMP, conf_choose=conf_choose, combine_reg_conf=combine,
                                   out_dir=out_dir, **FUSION_ARGS[method])
    assert xyz.is_cuda and rgb.is_cuda and xyz.shape[0] > 0
    assert torch.equal(xyz, xyz_w) and torch.equal(rgb, rgb_w)
    # the files: byte for byte what the writers make of the composition's depth, confidence and camera
    for k, ids in enumerate(meta["items"]):
        ref = ids[0]
        S.save_pfm(str(tmp_path / "d.pfm"), depths[k])
        assert (tmp_path / "d.pfm").read_bytes() == open(os.path.join(out_dir, "depth_est", f"{ref:08d}.pfm"), "rb").read()
        c = np.load(os.path.join(out_dir, "confidence", f"{ref:08d}.npy"))
        assert c.dtype == np.uint8 and np.array_equal(c, confs[k])
        np.save(str(tmp_path / "c.npy"), confs[k])
        assert (tmp_path / "c.npy").read_bytes() == open(os.path.join(out_dir, "confidence", f"{ref:08d}.npy"), "rb").read()
        dv = blob[f"dv_{k}"]
        S.write_cam(str(tmp_path / "c.txt"), cams[k], (dv[0], dv[-1]) if meta["dataset"] == "tt" else None)
        assert (tmp_path / "c.txt").read_bytes() == open(os.path.join(out_dir, "cams", f"{ref:08d}_cam.txt"), "rb").read()


def test_malformed_input(dev):
    with pytest.raises(ValueError, match="uint8"):
        S.resize_u8(torch.zeros(1, 8, 8, 3, device=dev), 32, 32)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.resize_u8(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), 32, 32)
    scene_u8 = torch.zeros(2, 32, 32, 3, dtype=torch.uint8, device=dev)
    with pytest.raises(ValueError, match="65 views"):
        S.normalize(scene_u8, [0] * 65)
    with pytest.raises(ValueError, match="uint8"):
        S.normalize(scene_u8.float(), [0])
    out = torch.empty(65, 3, 32, 32, device=dev)
    for views in ([0] * 65, [0, 2]):   # the C entry point checks V and the indices itself
        idx = (ctypes.c_int * len(views))(*views)
        with pytest.raises(RuntimeError, match="image_normalize"):
            _lib.call("mvsf_image_normalize", scene_u8, 2, idx, len(views), 32, 32, out, None)
    with pytest.raises(RuntimeError, match="image_resize_u8"):
        _lib.call("mvsf_image_resize_u8", scene_u8, 2, 32, 32, -1, scene_u8, 32, 32)
    torch.cuda.synchronize()
