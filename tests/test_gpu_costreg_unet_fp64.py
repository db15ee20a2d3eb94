"""The U-Net regularisers of stages 2-4 (CostRegNet, CostRegNet3D: csrc/costreg_unet.cu, csrc/conv3d_tc.cu) against fp64
on the device, at the sizes where their persistent CTAs loop:
  * every layer launch of both U-Nets at the DTU and Tanks & Temples stage sizes, through the layer seam
    mvsf_conv3d_tc_layer (fp16 hi|lo split output), plus sizes whose right and bottom tiles are ragged and larger cases
    for the layers that do not loop at a shipped size;
  * a test that asserts, from this device's SM count, which kernel instances those cases drive through more than one
    tile per CTA;
  * both whole U-Nets against oracle.hotpath.costreg_unet in fp64, at the three stage sizes of both datasets: the fp32
    epilogues (the skip add of the input volume, the fused 1x1x1 `prob` conv), prob3_kernel and the packing of all
    nine layers are reached only here and in test_costreg_unet_two_part(_pipelined)."""
import pytest
import torch

from tests import conv3d_common as C
from tests.common import rec

pytestmark = pytest.mark.gpu

PREFIX = {0: "fusions.1.cost_reg.", 1: "fusions.2.cost_reg."}   # stage 2: CostRegNet, stages 3-4: CostRegNet3D


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _unet_sd(seed, prob_gain=1.0):
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    torch.manual_seed(0)
    return synth.randomize_state_dict(build_hotpath_params(default_args()).eval(), seed=seed, prob_gain=prob_gain)


@pytest.fixture(scope="module")
def unet_sd():
    return _unet_sd(23)


# whole U-Nets: both kinds at the three stage sizes of each dataset (CostRegNet needs D % 8 == 0, so it takes D = 8 at
# the stage-4 size), and sizes with H, W multiples of 8 but not of 16, whose tiles are ragged at the right and bottom
UNET_CASES = [(f"{name}_s{st}", kind, D if kind == 1 or D % 8 == 0 else 8, H // s, W // s)
              for name, (H, W) in C.DATASETS.items() for kind in (0, 1) for st, _, D, s in C.UNET_STAGES] + \
             [("odd", 0, 16, 264, 440), ("odd", 1, 8, 520, 904)]

# single layers: every launch of the U-Nets at their shipped stage sizes and at the odd sizes above, and layers that do
# not loop there: CostRegNet conv5 / conv6 / conv7 at the T&T stage-4 size, CostRegNet3D conv5 / conv6 at NT = 4
_layers = {}
for _, _, kind, D, H, W in C.stage_shapes():
    _layers.update(dict.fromkeys(C.unet_layers(kind, D, H, W)))
for _, kind, D, H, W in UNET_CASES[-2:]:
    _layers.update(dict.fromkeys(C.unet_layers(kind, D, H, W)))
_layers.update(dict.fromkeys(C.unet_layers(0, 8, 1088, 1920)[4:7]))
_layers.update(dict.fromkeys([(C.CONV_S2, 1, 32, 64, 8, 296, 136, False, C.OUT_SPLIT),
                              (C.CONV_S1, 1, 64, 64, 8, 216, 40, False, C.OUT_SPLIT)]))
LAYER_CASES = [lay[:8] for lay in _layers]


def _layer_id(case):
    mode, sd, cin, cout, ID, IH, IW, skip = case
    return f"m{mode}sd{sd}_{cin}to{cout}_{ID}x{IH}x{IW}" + ("_skip" if skip else "")


def test_cases_loop_on_this_device(sms):
    """Every kernel instance the U-Nets run at the shipped sizes on this device runs two or more tiles on some CTA, in a
    case below whose CTAs run different numbers of tiles; some looping tile
    kernel CTA runs tiles with different numbers of units (depth edge and interior); the tile kernel's right and
    bottom tiles are ragged in some case of every mode."""
    shipped = {r["instance"] for _, _, kind, D, H, W in C.stage_shapes() for _, r in C.unet_coverage(kind, D, H, W, sms)}
    runs = [C.launch(*case[:7], sms) for case in LAYER_CASES] + \
        [r for _, kind, D, H, W in UNET_CASES for _, r in C.unet_coverage(kind, D, H, W, sms)]
    for inst in shipped:
        assert any(r["instance"] == inst and r["trips"][1] >= 2 and r["trips"][0] != r["trips"][1] for r in runs), inst
    tile = [r for r in runs if r["kernel"] == "tile"]
    assert any(r["mixed_depth"] for r in tile)
    for mode in (C.CONV_S1, C.CONV_S2, C.DECONV_S2):
        assert any(r["instance"][0] == mode and r["ragged_w"] and r["trips"][1] >= 2 for r in tile), mode
        assert any(r["instance"][0] == mode and r["ragged_h"] and r["trips"][1] >= 2 for r in tile), mode


@pytest.mark.parametrize("case", LAYER_CASES, ids=[_layer_id(c) for c in LAYER_CASES])
def test_unet_layer_vs_fp64(dev, sms, case):
    mode, sd, cin, cout, ID, IH, IW, skip = case
    e, scale = C.layer_vs_fp64(dev, mode, sd, cin, cout, ID, IH, IW, skip, seed=ID * 1009 + IH * 7 + IW + cin)
    r = C.launch(mode, sd, cin, cout, ID, IH, IW, sms)
    rec(f"unet_layer_{_layer_id(case)}", abs=e, scale=scale, kernel=r["kernel"], work=r["work"], trips=r["trips"][1])
    assert e < C.LAYER_TOL * max(1.0, scale)


@pytest.mark.parametrize("name,kind,D,H,W", UNET_CASES)
def test_costreg_unet_vs_fp64(dev, unet_sd, name, kind, D, H, W):
    e, scale = C.unet_vs_fp64(dev, unet_sd, PREFIX[kind], kind, D, H, W, seed=kind * 101 + D + H, twice=True)
    rec(f"costreg_unet_fp64_{name}_kind{kind}_{D}x{H}x{W}", abs=e, scale=scale)
    assert e < C.UNET_TOL * max(1.0, scale)


@pytest.mark.parametrize("kind", [0, 1])
def test_costreg_unet_harsh_vs_fp64(dev, kind):
    """up-scaled `prob` weights and a 6x larger volume: logits in the tens"""
    sd = _unet_sd(29, prob_gain=2.0)
    D, H, W = (16, 136, 240) if kind == 0 else (8, 272, 480)
    e, scale = C.unet_vs_fp64(dev, sd, PREFIX[kind], kind, D, H, W, seed=77 + kind, vol_scale=3.0, twice=True)
    rec(f"costreg_unet_fp64_harsh_kind{kind}_{D}x{H}x{W}", abs=e, scale=scale)
    assert scale > 10
    assert e < C.UNET_TOL * max(1.0, scale)
