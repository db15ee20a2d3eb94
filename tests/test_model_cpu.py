"""CPU tests of the whole-model seam (hotpath.DINOv2MVSNet, DINOv2_mvsformer_model.py:22-179): the oracle composition
(oracle/model.py) against the reference-executed fixtures tests/golden/model_*.npz at the north-star bars, the state-dict
keys of the module against the reference's, the ViT grid arithmetic, and the construction and input errors."""
import os

import pytest
import torch

from oracle import model as OM
from tests.common import GOLDEN
from tests.model_common import CASES, fixture, fixture_errors, model_args, model_state_dict, within_bars


@pytest.fixture(scope="module")
def net():
    from mvsformerplusplus_b200 import DINOv2MVSNet
    return DINOv2MVSNet(model_args()).eval()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_model(name):
    gold, meta, imgs, proj, dv = fixture(name)
    out = OM.model_forward(imgs, proj, dv, model_state_dict(meta["wseed"]), model_args())
    e = fixture_errors(meta, out, out["features_fpn"], gold)
    assert not within_bars(e), within_bars(e)


def test_state_dict_keys_are_the_reference_model_keys(net):
    """the four key lists of the seams add up to the reference DINOv2MVSNet's 779 keys"""
    want = {}
    for part in ("hotpath", "fpn", "vit", "vit_decoder"):
        with open(os.path.join(GOLDEN, f"{part}_state_dict_keys.txt")) as f:
            for line in f:
                k, shape = line.strip().split(" ", 1)
                want[k] = shape
    got = {k: str(tuple(v.shape)) for k, v in net.state_dict().items()}
    assert len(want) == 779
    assert got == want


@pytest.mark.parametrize("H,W,grid", [(1152, 1536, (36, 48)), (1088, 1920, (34, 60)), (864, 1152, (27, 36)),
                                      (96, 128, (3, 4)), (64, 96, (2, 3))])
def test_vit_grid(net, H, W, grid):
    """DTU, Tanks & Temples and test.py's default size, and the fixtures: the shipped rescale 0.4375 gives a grid of exactly
    H/32 x W/32, so vit_feat (4x the grid) is already H/8 x W/8 and the bilinear resize never runs"""
    vh, vw = OM.vit_size(H, W, 0.4375)
    assert net.vit_grid(H, W) == grid == (vh // 14, vw // 14) == (H // 32, W // 32)


def _inputs(B=1, V=2, H=64, W=96):
    from mvsformerplusplus_b200 import synth
    return (torch.zeros(B, V, 3, H, W), synth.make_proj_matrices(V, H, W, batch=B),
            synth.make_depth_values(48, 425.0, 10.0, batch=B))


def test_cpu_tensor_raises(net):
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        net(*_inputs())


@pytest.mark.parametrize("H,W", [(72, 96), (64, 80), (16, 32)])
def test_size_not_a_multiple_of_32_raises(net, H, W):
    with pytest.raises(ValueError, match="multiples of 32"):
        net(*_inputs(H=H, W=W))


def test_training_mode_raises():
    from mvsformerplusplus_b200 import DINOv2MVSNet
    m = DINOv2MVSNet(model_args())
    assert m.training
    with pytest.raises(NotImplementedError, match="eval"):
        m(*_inputs())


def test_rescale_needing_the_bilinear_resize_raises():
    from mvsformerplusplus_b200 import DINOv2MVSNet
    m = DINOv2MVSNet(model_args(rescale=0.25)).eval()
    with pytest.raises(NotImplementedError, match="bilinear"):
        m(*_inputs())


@pytest.mark.parametrize("change", [dict(inverse_depth=False), dict(feat_chs=[8, 16, 32, 32]), dict(out_ch=32)])
def test_unsupported_config_raises(change):
    from mvsformerplusplus_b200 import DINOv2MVSNet
    with pytest.raises(NotImplementedError):
        DINOv2MVSNet(model_args(**change))
