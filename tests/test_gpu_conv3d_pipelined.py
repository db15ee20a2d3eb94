"""The pipelined U-Net convolutions against torch's fp64 convolutions, at the limits of test_gpu_parity:
  * the depth-streaming kernel (conv3d_col_kernel: a 3-slice accumulator window moved down one slice per input slice)
    over depth runs that start and end at the volume edges (one run) and inside the volume (the launcher splits the
    depth into runs of DC < D slices when the plane has few tiles);
  * the transposed convs (one N = 4 * NPAD product per input shift, zero blocks for the classes it does not feed) with
    odd numbers of tiles in H and W;
  * both U-Net kinds end to end, with the fused OUT_F32 (CostRegNet) and OUT_PROB (CostRegNet3D) epilogues."""
import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import _lib
from tests.common import max_abs, rec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _col_depth_run(D, IH, IW, mode, cin, cout):
    """depth run DC the depth-streaming launcher (conv3d_tc.cu launch_col) picks on this device"""
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    npad = max(cout, 16)
    OH, OW = (IH, IW) if mode == 0 else ((IH - 1) // 2 + 1, (IW - 1) // 2 + 1)
    best, best_cost = None, 1e30
    for nt in (4, 2, 1):
        if 3 * nt * npad > 128:
            continue
        div = 1
        while div <= 8:
            dc = -(-D // div)
            if div == 1 or dc != -(-D // (div // 2)):
                items = -(-OW // (8 * nt)) * -(-OH // 16) * -(-D // dc)
                eff = items / (-(-items // num_sms) * num_sms)
                halo_w = (8 * nt + 2) / (8 * nt) if mode == 0 else (16 * nt + 1) / (16 * nt)
                cost = halo_w * (1.0 if dc >= D else (dc + 2) / dc) / eff
                if cost < best_cost:
                    best, best_cost = dc, cost
            div *= 2
    return best


def _layer(dev, mode, sd, cin, cout, ID, IH, IW, skip, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(ID, IH, IW, cin, generator=g)
    w = torch.randn(27, cin, cout, generator=g) / (27 * cin) ** 0.5 * 1.7
    b = torch.randn(cout, generator=g) * 0.2
    xin = x.permute(3, 0, 1, 2)[None].double()
    if mode == 2:
        wt = w.reshape(3, 3, 3, cin, cout).permute(3, 4, 0, 1, 2).double()
        y = F.conv_transpose3d(xin, wt, stride=(sd, 2, 2), padding=1, output_padding=(sd - 1, 1, 1))
    else:
        wt = w.reshape(3, 3, 3, cin, cout).permute(4, 3, 0, 1, 2).double()
        y = F.conv3d(xin, wt, stride=(1, 1, 1) if mode == 0 else (sd, 2, 2), padding=1)
    y = torch.relu(y + b.double().view(1, -1, 1, 1, 1))[0].permute(1, 2, 3, 0).contiguous()
    sk = torch.randn(y.shape, generator=g) if skip else None
    if skip:
        y = y + sk.double()
    x_d, wb_d = x.contiguous().to(dev), torch.cat([w.reshape(-1), b]).to(dev)
    sk_d = sk.contiguous().to(dev) if skip else None
    out = torch.empty(y.shape, device=dev)
    ws = torch.empty((2 * x.numel() + 4 * y.numel()) // 2 + 27 * cin * max(cout, 16) * 4 + 1024, device=dev)
    _lib.call("mvsf_conv3d_tc_layer", mode, sd, x_d, wb_d, sk_d, out, ws, ws.numel() * 4, cin, cout, ID, IH, IW)
    e = float((out.cpu().double() - y).abs().max())
    return e, float(y.abs().max())


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
    e, scale = _layer(dev, mode, 1, cin, cout, D, IH, IW, False, seed=31 * D + cin + mode)
    dc = _col_depth_run(D, IH, IW, mode, cin, cout)
    rec(f"conv3d_col_mode{mode}_{cin}to{cout}_{D}x{IH}x{IW}_dc{dc}", abs=e, scale=scale)
    assert e < 1e-5 * max(1.0, scale)


# odd tile counts in H (16-row tiles) and W (8 * NT-column tiles) of the input cells
@pytest.mark.parametrize("sd,cin,cout,ID,IH,IW,skip", [
    (2, 32, 16, 3, 40, 72, True), (1, 16, 8, 5, 48, 88, True), (1, 64, 32, 3, 24, 56, True), (2, 16, 8, 1, 40, 40, False),
    (1, 8, 16, 3, 24, 40, False), (1, 32, 64, 2, 17, 23, False)])
def test_transposed_conv_odd_tiles(dev, sd, cin, cout, ID, IH, IW, skip):
    e, scale = _layer(dev, 2, sd, cin, cout, ID, IH, IW, skip, seed=7 * ID + cin + IW)
    rec(f"conv3d_deconv_sd{sd}_{cin}to{cout}_{ID}x{IH}x{IW}_skip{int(skip)}", abs=e, scale=scale)
    assert e < 1e-5 * max(1.0, scale)


def _rand_sd(seed):
    from mvsformerplusplus_b200 import synth
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    torch.manual_seed(0)
    return synth.randomize_state_dict(build_hotpath_params(default_args()).eval(), seed=seed)


# stage 1 = CostRegNet (fp32 OUT_F32 epilogue + prob3), stages 2, 3 = CostRegNet3D (fused OUT_PROB epilogue)
@pytest.mark.parametrize("stage,D,H,W", [(1, 8, 40, 24), (1, 16, 24, 56), (2, 5, 40, 56), (3, 1, 24, 24), (3, 16, 16, 8)])
def test_costreg_unet_two_part_pipelined(dev, stage, D, H, W):
    from mvsformerplusplus_b200 import packing
    from mvsformerplusplus_b200.hotpath import pack_unet_tc
    from oracle import hotpath as O
    sd = _rand_sd(17)
    g = torch.Generator().manual_seed(stage * 11 + D + H)
    vol = torch.randn(1, 8, D, H, W, generator=g) * 0.5
    p = f"fusions.{stage}.cost_reg."
    want = O.costreg_unet(vol, sd, p)[0, 0]
    kind, conv, small = packing.pack_costreg_unet(sd, p)
    assert kind == (0 if stage == 1 else 1)
    ws = _lib.workspace("mvsf_costreg_unet_workspace_bytes", kind, 8, D, H, W, device=dev)
    logits = torch.empty(D, H, W, device=dev)
    v = vol[0].permute(1, 2, 3, 0).contiguous().to(dev)
    tc = pack_unet_tc(kind, conv.to(dev))
    _lib.call("mvsf_costreg_unet_forward", kind, v, small.to(dev), tc, logits, ws, ws.numel() * 4, 8, D, H, W)
    e = max_abs(logits.cpu(), want)
    rec(f"costreg_unet_pipelined_stage{stage}_{D}x{H}x{W}", abs=e, scale=float(want.abs().max()))
    assert e < 2e-4 * max(1.0, float(want.abs().max()))
