"""Shared helpers of the U-Net convolution tests (csrc/conv3d_tc.cu, csrc/costreg_unet.cu): a host restatement of the
launchers' tile choices, the U-Net layer schedule, the tile coverage that follows from them, one fp64 check of a single
layer through the `mvsf_conv3d_tc_layer` seam and one of a whole U-Net.  tests/test_conv3d_cpu.py pins every
constant restated here to the sources."""
import numpy as np
import torch
import torch.nn.functional as F

CONV_S1, CONV_S2, DECONV_S2 = 0, 1, 2             # ConvTcMode (conv3d_tc.cuh)
OUT_SPLIT, OUT_F32, OUT_PROB = 0, 1, 2            # ConvTcOut
SMEM, MAX_STAGES = 227 * 1024, 8                  # dynamic shared memory of one CTA, mbarrier ring slots
WRES_BYTES = 112 * 1024                           # depth-streaming kernel: weight slabs stay resident up to this size

# |out - fp64| <= tol * max(1, max |fp64|) for one layer and for a whole U-Net.  Worst measured on an H100 SXM (132 SMs,
# 700 W): 7.2e-6 (a 64 -> 64 layer) and 1.34e-6; a layer's KG = 1 products without w_lo cost >= 1.6e-4 and CostRegNet
# >= 1.5e-5 (DESIGN.md "Numerics")
LAYER_TOL = 1e-5
UNET_TOL = 3.8e-6

# costreg_unet.cu kLayerCh / kLayerMode: conv1 conv2 conv3 conv4 conv5 conv6 conv7 conv9 conv11 of module.py:367-504
LAYER_CH = ((8, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 32), (32, 16), (16, 8))
LAYER_MODE = (CONV_S2, CONV_S1, CONV_S2, CONV_S1, CONV_S2, CONV_S1, DECONV_S2, DECONV_S2, DECONV_S2)

# the depth maps the U-Nets regularise: (stage, kind, D, image scale); kind 0 = CostRegNet (depth stride 2), kind 1 =
# CostRegNet3D (depth stride 1); image sizes of DTU and Tanks & Temples (1080 rows padded to 1088)
UNET_STAGES = ((2, 0, 16, 4), (3, 1, 8, 2), (4, 1, 4, 1))
DATASETS = {"dtu": (1152, 1536), "tt": (1088, 1920)}


def cdiv(a, b):
    return -(-a // b)


def align_up(x, a):
    return cdiv(x, a) * a


def npad(cout):
    return max(cout, 16)


def kg(mode, cin):
    """channel octets per pipeline unit: conv3d_tc_kg"""
    return 2 if mode != CONV_S2 and cin >= 16 else 1


def uses_col(mode, sd, cout):
    """conv3d_tc_col: the depth-streaming kernel runs the depth-stride-1 convolutions with Cout <= 32"""
    return (mode == CONV_S1 or (mode == CONV_S2 and sd == 1)) and npad(cout) <= 32


def oct_bytes(mode, nt):
    """c3::Geo<MODE, NT>::OCT_BYTES: the hi and lo planes of one channel octet (four parity planes for strided convs)"""
    pr = 18 if mode == CONV_S1 else 17
    pc = 8 * nt + 2 if mode == CONV_S1 else 8 * nt + 1
    return (4 if mode == CONV_S2 else 1) * align_up(2 * pr * pc * 16, 128)


def slab_bytes(mode, cout):
    return npad(cout) * (1024 if mode == DECONV_S2 else 576)


def out_shape(mode, sd, ID, IH, IW):
    if mode == CONV_S1:
        return ID, IH, IW
    if mode == CONV_S2:
        return (ID - 1) // sd + 1, (IH - 1) // 2 + 1, (IW - 1) // 2 + 1
    return ID * sd, 2 * IH, 2 * IW


def depth_taps(mode, sd, od, ID):
    """number of input depth slices that feed output slice od (conv3d_tc.cu depth_taps)"""
    n = 0
    for kd in range(3):
        if mode == CONV_S1:
            i, ok = od + kd - 1, True
        elif mode == CONV_S2:
            i, ok = od * sd + kd - 1, True
        else:
            num = od + 1 - kd
            i, ok = (num, True) if sd == 1 else (num >> 1, num % 2 == 0)
        n += ok and 0 <= i < ID
    return n


def tile_launch(mode, sd, cin, cout, ID, IH, IW, sms, out=OUT_SPLIT):
    """conv3d_tc.cu launch_mode: tile width NT (8 NT cells wide, 16 high), tile count and grid of conv3d_tc_kernel"""
    OD, OH, OW = out_shape(mode, sd, ID, IH, IW)
    cells_h, cells_w = (IH, IW) if mode == DECONV_S2 else (OH, OW)
    ncls = 4 if mode == DECONV_S2 else 1
    best_nt, best_eff = 0, -1.0
    for nt in (4, 2, 1):
        stage = align_up(kg(mode, cin) * oct_bytes(mode, nt) + slab_bytes(mode, cout), 128)
        if nt * ncls * npad(cout) > 256 or 2 * stage + 256 > SMEM:
            continue
        t = cdiv(cells_w, 8 * nt) * cdiv(cells_h, 16) * OD
        eff = t / (cdiv(t, sms) * sms)
        if eff >= 0.85:
            best_nt = nt
            break
        if eff > best_eff:
            best_eff, best_nt = eff, nt
    assert best_nt > 0
    nt = best_nt
    tiles_w, tiles_h = cdiv(cells_w, 8 * nt), cdiv(cells_h, 16)
    ntiles = tiles_w * tiles_h * OD
    grid = min(ntiles, sms)
    # units (input depth slice x channel group) of each tile, per CTA (tile, tile + grid, ...)
    units = np.array([depth_taps(mode, sd, od, ID) for od in range(OD)])[np.arange(ntiles) // (tiles_w * tiles_h)]
    cta = np.arange(ntiles) % grid
    lo, hi = np.full(grid, 99), np.zeros(grid, dtype=int)
    np.minimum.at(lo, cta, units)
    np.maximum.at(hi, cta, units)
    trips = np.bincount(cta, minlength=grid)
    return dict(kernel="tile", instance=(mode, nt, out, npad(cout)), work=ntiles, grid=grid,
                trips=(int(trips.min()), int(trips.max())), mixed_depth=bool(((hi > lo) & (trips >= 2)).any()),
                ragged_w=cells_w % (8 * nt) != 0, ragged_h=cells_h % 16 != 0)


def col_launch(mode, cin, cout, D, IH, IW, sms):
    """conv3d_tc.cu launch_col: tile width NT and depth run DC (items = tiles x depth runs) of conv3d_col_kernel"""
    OH, OW = (IH, IW) if mode == CONV_S1 else ((IH - 1) // 2 + 1, (IW - 1) // 2 + 1)
    slab = npad(cout) * 1728
    wres_bytes = align_up(cin // 8 // kg(mode, cin) * slab, 128)
    wres = wres_bytes <= WRES_BYTES
    best, best_cost = None, 1e30
    for nt in (4, 2, 1):
        if 3 * nt * npad(cout) > 128:
            continue
        stage = align_up(kg(mode, cin) * oct_bytes(mode, nt) + (0 if wres else slab), 128)
        ns = min(MAX_STAGES, (SMEM - (wres_bytes if wres else 0) - 256) // stage)
        if ns < 2:
            continue
        div = 1
        while div <= 8:
            dc = cdiv(D, div)
            if div == 1 or dc != cdiv(D, div // 2):
                items = cdiv(OW, 8 * nt) * cdiv(OH, 16) * cdiv(D, dc)
                eff = items / (cdiv(items, sms) * sms)
                halo_w = (8 * nt + 2) / (8 * nt) if mode == CONV_S1 else (16 * nt + 1) / (16 * nt)
                cost = halo_w * (1.0 if dc >= D else (dc + 2) / dc) / eff
                if cost < best_cost:
                    best, best_cost = (nt, dc, items), cost
            div *= 2
    assert best is not None
    nt, dc, items = best
    grid = min(items, sms)
    return dict(kernel="col", instance=(mode, nt, OUT_SPLIT, npad(cout)), dc=dc, work=items, grid=grid,
                trips=(items // grid, cdiv(items, grid)), mixed_depth=False, ragged_w=OW % (8 * nt) != 0,
                ragged_h=OH % 16 != 0)


def launch(mode, sd, cin, cout, ID, IH, IW, sms, out=OUT_SPLIT):
    """what launch_conv3d_tc runs for one layer"""
    if out == OUT_SPLIT and uses_col(mode, sd, cout):
        return col_launch(mode, cin, cout, ID, IH, IW, sms)
    return tile_launch(mode, sd, cin, cout, ID, IH, IW, sms, out)


def unet_layers(kind, D, H, W):
    """the 9 launches of unet_forward_tc: (mode, sd, cin, cout, ID, IH, IW, skip, out) per layer"""
    sd = 2 if kind == 0 else 1
    dims = [(D, H, W)]
    for _ in range(3):
        d, h, w = dims[-1]
        dims.append(((d - 1) // sd + 1, h // 2, w // 2))
    ins = (dims[0], dims[1], dims[1], dims[2], dims[2], dims[3], dims[3], dims[2], dims[1])
    last = OUT_F32 if kind == 0 else OUT_PROB
    return [(LAYER_MODE[l], sd, LAYER_CH[l][0], LAYER_CH[l][1]) + ins[l] + (l >= 6, last if l == 8 else OUT_SPLIT)
            for l in range(9)]


def unet_coverage(kind, D, H, W, sms):
    """[(layer, launch(...))] of one U-Net forward on this many SMs"""
    return [(l, launch(m, sd, ci, co, ID, IH, IW, sms, out))
            for l, (m, sd, ci, co, ID, IH, IW, _, out) in enumerate(unet_layers(kind, D, H, W))]


def stage_shapes():
    """(dataset, stage, kind, D, H, W) of every U-Net a DTU or Tanks & Temples depth map runs"""
    return [(name, st, kind, D, H // s, W // s) for name, (H, W) in DATASETS.items() for st, kind, D, s in UNET_STAGES]


# ---------------------------------------------------------------------------------------------- fp64 checks (GPU)
def layer_vs_fp64(dev, mode, sd, cin, cout, ID, IH, IW, skip, seed):
    """One 3x3x3 layer through mvsf_conv3d_tc_layer (fp16 hi|lo split, pack, tensor-core layer, merge) against torch's
    fp64 convolution on the device: conv / strided conv / transposed conv with output_padding = stride - 1, bias, ReLU,
    skip added after the ReLU.  The output is NaN-filled before the call.  -> (max |out - fp64|, max |fp64|)"""
    from mvsformerplusplus_b200 import _lib
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(ID, IH, IW, cin, generator=g)
    w = torch.randn(27, cin, cout, generator=g) / (27 * cin) ** 0.5 * 1.7
    b = torch.randn(cout, generator=g) * 0.2
    OD, OH, OW = out_shape(mode, sd, ID, IH, IW)
    sk = torch.randn(OD, OH, OW, cout, generator=g) if skip else None
    x_d, wb_d = x.to(dev), torch.cat([w.reshape(-1), b]).to(dev)
    sk_d = sk.to(dev) if skip else None
    out = torch.full((OD, OH, OW, cout), float("nan"), device=dev)
    ws = torch.empty((2 * x.numel() + 4 * out.numel()) // 2 + 27 * cin * npad(cout) * 4 + 1024, device=dev)
    _lib.call("mvsf_conv3d_tc_layer", mode, sd, x_d, wb_d, sk_d, out, ws, ws.numel() * 4, cin, cout, ID, IH, IW)
    del ws
    with torch.no_grad():
        xin = x_d.double().permute(3, 0, 1, 2)[None]
        w5 = w.to(dev, torch.float64).reshape(3, 3, 3, cin, cout)
        if mode == DECONV_S2:
            y = F.conv_transpose3d(xin, w5.permute(3, 4, 0, 1, 2), stride=(sd, 2, 2), padding=1,
                                   output_padding=(sd - 1, 1, 1))
        else:
            y = F.conv3d(xin, w5.permute(4, 3, 0, 1, 2), stride=(1, 1, 1) if mode == CONV_S1 else (sd, 2, 2), padding=1)
        y = torch.relu(y + b.to(dev, torch.float64).view(1, -1, 1, 1, 1))[0].permute(1, 2, 3, 0)
        if skip:
            y = y + sk_d.double()
        return float((out.double() - y).abs().max()), float(y.abs().max())   # a NaN left in `out` gives NaN


def unet_vs_fp64(dev, sd, p, kind, D, H, W, seed, vol_scale=0.5, twice=False):
    """Both parts of a U-Net (packing.pack_costreg_unet, pack_unet_tc) through mvsf_costreg_unet_forward against
    oracle.hotpath.costreg_unet in fp64 on the device, with the state dict (keys under `p`) and the volume promoted to
    fp64.  The logits
    are NaN-filled before the call; with `twice` a second call must give the same bits.
    -> (max |logits - fp64|, max |fp64|)"""
    from mvsformerplusplus_b200 import _lib, packing
    from mvsformerplusplus_b200.hotpath import pack_unet_tc
    from oracle import hotpath as O
    k, conv, small = packing.pack_costreg_unet(sd, p)
    assert k == kind
    g = torch.Generator().manual_seed(seed)
    vol = (torch.randn(1, 8, D, H, W, generator=g) * vol_scale)[0].permute(1, 2, 3, 0).contiguous().to(dev)   # NDHWC
    ws = _lib.workspace("mvsf_costreg_unet_workspace_bytes", kind, 8, D, H, W, device=dev)
    tc, small = pack_unet_tc(kind, conv.to(dev)), small.to(dev)
    logits = torch.full((D, H, W), float("nan"), device=dev)
    _lib.call("mvsf_costreg_unet_forward", kind, vol, small, tc, logits, ws, ws.numel() * 4, 8, D, H, W)
    if twice:
        again = torch.full((D, H, W), float("nan"), device=dev)
        _lib.call("mvsf_costreg_unet_forward", kind, vol, small, tc, again, ws, ws.numel() * 4, 8, D, H, W)
        assert torch.equal(again, logits), "two calls differ"
        del again
    del ws, tc
    with torch.no_grad():
        sd64 = {key: v.to(dev) for key, v in O.state_dict_to({key: v for key, v in sd.items() if key.startswith(p)},
                                                             torch.float64).items()}
        want = O.costreg_unet(vol.double().permute(3, 0, 1, 2)[None], sd64, p)[0, 0]
        return float((logits.double() - want).abs().max()), float(want.abs().max())
