"""ORACLE - TEST INFRASTRUCTURE ONLY.  The FPN feature pyramid of models/module.py:208-270 (FPNEncoder / FPNDecoder,
eval mode, norm_type 'BN') restated with plain torch ops on a state dict, in the dtype of the inputs (fp32 or fp64), on
any device.  Pinned to the reference's own modules by tests/golden/fpn_*.npz (tests/test_fpn_cpu.py).
"""
import torch
import torch.nn.functional as F

# name, stride, padding (module.py:211-224)
ENCODER_LAYERS = (("conv00", 1, 3), ("conv01", 1, 2), ("downsample1", 2, 2), ("conv10", 1, 1), ("conv11", 1, 1),
                  ("downsample2", 2, 2), ("conv20", 1, 1), ("conv21", 1, 1), ("downsample3", 2, 1), ("conv30", 1, 1),
                  ("conv31", 1, 1))


def _bn(x, sd, p, eps=1e-5):
    t = lambda k: sd[p + k].to(x.dtype).to(x.device)
    return F.batch_norm(x, t("running_mean"), t("running_var"), t("weight"), t("bias"), False, 0.0, eps)


def _w(sd, k, x):
    return sd[k].to(x.dtype).to(x.device)


def fpn_encoder(x, sd, p="encoder."):
    """module.py:226-239: Conv2d(bias=False) -> BatchNorm -> LeakyReLU(0.1) per layer -> [conv01, conv11, conv21, conv31]"""
    outs = {}
    for name, stride, pad in ENCODER_LAYERS:
        x = F.conv2d(x, _w(sd, f"{p}{name}.conv.weight", x), stride=stride, padding=pad)
        x = F.leaky_relu(_bn(x, sd, f"{p}{name}.bn."), 0.1)
        outs[name] = x
    return [outs["conv01"], outs["conv11"], outs["conv21"], outs["conv31"]]


def _swish(x):
    return x * torch.sigmoid(x)


def up2_fp32_coords(x):
    """F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True) in the dtype of x, but at the source
    coordinates an fp32 tensor gets: ATen computes scale = (in - 1) / (out - 1) and src = scale * dst in the tensor's
    opmath type, so fp32 rounds them and fp64 does not.  At 1088 x 1920 the rounded coordinates move fp32 results by up
    to 2e-5 of a feature map's range, an fp32 property of the operation rather than of any arithmetic in the layers."""
    h, w = x.shape[-2:]

    def axis(n):
        i = torch.arange(2 * n, device=x.device)
        s = torch.tensor(n - 1, dtype=torch.float32) / torch.tensor(2 * n - 1, dtype=torch.float32)
        src = (s.to(x.device) * i.float()).to(x.dtype)
        a = src.floor().long()
        return a, (a + 1).clamp(max=n - 1), src - a
    ya, yb, ly = axis(h)
    xa, xb, lx = axis(w)
    ly, lx = ly.view(-1, 1), lx.view(1, -1)
    r0, r1 = x[..., ya, :], x[..., yb, :]
    return (1 - ly) * ((1 - lx) * r0[..., xa] + lx * r0[..., xb]) + ly * ((1 - lx) * r1[..., xa] + lx * r1[..., xb])


def fpn_decoder(conv01, conv11, conv21, conv31, sd, p="decoder.", up2=None):
    """module.py:257-270: out0 = Swish(BN(conv1x1(conv31))); intra_k = up2(intra_{k-1}) (bilinear, align_corners=True)
    + inner_k(lateral_k); out_k = Swish(BN(conv3x3(intra_k))).  up2: the upsampling, by default F.interpolate in the
    dtype of the inputs (up2_fp32_coords: fp64 values at the source coordinates fp32 uses)"""
    up2 = up2 or (lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True))
    x = conv31
    outs = [_swish(_bn(F.conv2d(x, _w(sd, p + "out0.0.weight", x), _w(sd, p + "out0.0.bias", x)), sd, p + "out0.1."))]
    for k, lat in ((1, conv21), (2, conv11), (3, conv01)):
        x = up2(x) + F.conv2d(lat, _w(sd, f"{p}inner{k}.weight", lat), _w(sd, f"{p}inner{k}.bias", lat))
        y = F.conv2d(x, _w(sd, f"{p}out{k}.0.weight", x), _w(sd, f"{p}out{k}.0.bias", x), padding=1)
        outs.append(_swish(_bn(y, sd, f"{p}out{k}.1.")))
    return outs
