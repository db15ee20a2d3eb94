"""The pipelined U-Net convolutions against torch's fp64 convolutions, at the limits of test_gpu_parity:
  * the depth-streaming kernel (conv3d_col_kernel: a 3-slice accumulator window moved down one slice per input slice)
    over depth runs that start and end at the volume edges (one run) and inside the volume (the launcher splits the
    depth into runs of DC < D slices when the plane has few tiles);
  * the transposed convs (one N = 4 * NPAD product per input shift, zero blocks for the classes it does not feed) with
    odd numbers of tiles in H and W;
  * both U-Net kinds end to end against the fp64 oracle, with the fused OUT_F32 (CostRegNet) and OUT_PROB
    (CostRegNet3D) epilogues."""
import pytest
import torch

from tests import conv3d_common as C
from tests.common import rec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _col_depth_run(D, IH, IW, mode, cin, cout):
    """depth run DC the depth-streaming launcher (conv3d_tc.cu launch_col) picks on this device"""
    return C.col_launch(mode, cin, cout, D, IH, IW, torch.cuda.get_device_properties(0).multi_processor_count)["dc"]


# (mode, cin, cout, D, IH, IW): stride-1 convs (mode 0) and CostRegNet3D's (1, 2, 2) strided convs (mode 1, sd 1)
COL_CASES = [(0, 16, 16, D, 64, 600) for D in (1, 2, 3, 4, 5, 8, 16)] + \
            [(0, 16, 16, D, 16, 24) for D in (2, 3, 5, 16)] + \
            [(0, 32, 32, 5, 40, 56), (0, 32, 32, 8, 64, 200), (1, 8, 16, 4, 48, 80), (1, 8, 16, 16, 32, 40),
             (1, 16, 32, 5, 64, 88), (1, 8, 16, 1, 40, 56)]


def test_col_cases_cover_single_and_split_depth_runs(dev):
    dcs = [(D, _col_depth_run(D, IH, IW, mode, cin, cout)) for mode, cin, cout, D, IH, IW in COL_CASES]
    assert any(D > 2 and dc == D for D, dc in dcs), dcs
    assert any(dc < D - 1 for D, dc in dcs), dcs


@pytest.mark.parametrize("mode,cin,cout,D,IH,IW", COL_CASES)
def test_depth_streaming_conv(dev, mode, cin, cout, D, IH, IW):
    e, scale = C.layer_vs_fp64(dev, mode, 1, cin, cout, D, IH, IW, False, seed=31 * D + cin + mode)
    dc = _col_depth_run(D, IH, IW, mode, cin, cout)
    rec(f"conv3d_col_mode{mode}_{cin}to{cout}_{D}x{IH}x{IW}_dc{dc}", abs=e, scale=scale)
    assert e < C.LAYER_TOL * max(1.0, scale)


# odd tile counts in H (16-row tiles) and W (8 * NT-column tiles) of the input cells
@pytest.mark.parametrize("sd,cin,cout,ID,IH,IW,skip", [
    (2, 32, 16, 3, 40, 72, True), (1, 16, 8, 5, 48, 88, True), (1, 64, 32, 3, 24, 56, True), (2, 16, 8, 1, 40, 40, False),
    (1, 8, 16, 3, 24, 40, False), (1, 32, 64, 2, 17, 23, False)])
def test_transposed_conv_odd_tiles(dev, sd, cin, cout, ID, IH, IW, skip):
    e, scale = C.layer_vs_fp64(dev, 2, sd, cin, cout, ID, IH, IW, skip, seed=7 * ID + cin + IW)
    rec(f"conv3d_deconv_sd{sd}_{cin}to{cout}_{ID}x{IH}x{IW}_skip{int(skip)}", abs=e, scale=scale)
    assert e < C.LAYER_TOL * max(1.0, scale)


def _rand_sd(seed):
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    torch.manual_seed(0)
    return synth.randomize_state_dict(build_hotpath_params(default_args()).eval(), seed=seed)


# stage 1 = CostRegNet (fp32 OUT_F32 epilogue + prob3), stages 2, 3 = CostRegNet3D (fused OUT_PROB epilogue)
@pytest.mark.parametrize("stage,D,H,W", [(1, 8, 40, 24), (1, 16, 24, 56), (2, 5, 40, 56), (3, 1, 24, 24), (3, 16, 16, 8)])
def test_costreg_unet_two_part_pipelined(dev, stage, D, H, W):
    e, scale = C.unet_vs_fp64(dev, _rand_sd(17), f"fusions.{stage}.cost_reg.", 0 if stage == 1 else 1, D, H, W,
                              seed=stage * 11 + D + H)
    rec(f"costreg_unet_pipelined_stage{stage}_{D}x{H}x{W}", abs=e, scale=scale)
    assert e < C.UNET_TOL * max(1.0, scale)
