"""GPU tests of the FPN feature pyramid (csrc/fpn.cu through hotpath.FPNEncoder / FPNDecoder) against the fp64 torch
restatement of models/module.py:208-270 (oracle/fpn.py, run on the GPU), the reference-executed fixtures, and downstream
through the hot path.  Errors go to rec().

Bar: every output within FPN_BAR * max(1, max|fp64|), the encoder outputs against the fp64 encoder of the same images
and the decoder outputs against the fp64 decoder of the same fp32 maps the CUDA decoder was given, so neither carries
the other's error.  The decoder's bilinear upsampling takes its source coordinates in fp32, as ATen does for an fp32
tensor (fpn.cu IntraSrc); the fp64 reference uses the same coordinates, since fp64 ones move the full-size outputs by
2e-5.
All 13 tensor-core convolutions run on fp16 hi + lo operands (conv2d_tc.cuh) and the SIMT parts (conv00, inner_k, out0)
are fp32, so the bar is fp32-class: about 3x the worst error measured on an H100 SXM (132 SMs, 700 W power limit) over
every case here, FPN_WORST_MEASURED, and below a quarter of what the smallest value mutation of the kernels measured
(dropping the x_lo x w_hi product, the w_lo rows of the 8-channel layers, every CTA's second tile or the vit_feat view
n % V: 1.4e-4 or more in every case it reaches).  An fp16-only operand in one layer costs 1e-4 .. 3e-4 at these
inputs.  The reference-executed fixtures measure parity with the fp32 reference, not the kernels' arithmetic, and keep
1e-4."""
import pytest
import torch

from mvsformerplusplus_b200 import synth
from oracle import fpn as OF
from tests.common import TMP, load_golden, max_abs, rec, rel_linf
from tests.fpn_common import (FPN_CASES, FPN_TC_LAYERS, Pyramid, fixture_crop, fpn_coverage, fpn_inputs, fpn_state_dict,
                              sub_sd)

pytestmark = pytest.mark.gpu
NAMES = ("conv01", "conv11", "conv21", "conv31", "out0", "out1", "out2", "out3")
FPN_BAR = 1.5e-5
FPN_WORST_MEASURED = dict(encoder=5.1e-6, decoder=2.4e-6)   # conv31 / out2 at 10 x 1088 x 1920
# (N, H, W) of the fp64 cases.  14 x 264 x 456 makes every one of the 13 tensor-core layers run more tiles than its grid
# can hold and leaves both its right and bottom edge tiles partial (test_fpn_fp64_cases_cover_every_layer)
FP64_CASES = [(2, 64, 96), (1, 40, 72), (1, 8, 8), (2, 136, 240), (1, 24, 40), (14, 264, 456)]


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _modules(sd, dev):
    from mvsformerplusplus_b200.hotpath import FPNDecoder, FPNEncoder
    enc, dec = FPNEncoder([8, 16, 32, 64]), FPNDecoder([8, 16, 32, 64])
    enc.load_state_dict(sub_sd(sd, "encoder."), strict=True)
    dec.load_state_dict(sub_sd(sd, "decoder."), strict=True)
    return enc.to(dev).eval(), dec.to(dev).eval()


def _coverage(N, H, W):
    p = torch.cuda.get_device_properties(0)
    return fpn_coverage(N, H, W, p.multi_processor_count, p.shared_memory_per_multiprocessor,
                        p.max_threads_per_multi_processor)


def _run_cuda(enc, dec, x, vit):
    c = enc(x)
    o = dec(c[0], c[1], c[2], c[3] + vit)
    return list(c) + list(o)


def _rel(g, w):
    """max |g - w| / max(1, max |w|), inf where g is not finite"""
    assert tuple(g.shape) == tuple(w.shape)
    w = w.to(g.device, torch.float64)
    if not bool(torch.isfinite(g).all()):
        return float("inf")
    return float((g.double() - w).abs().max()) / max(1.0, float(w.abs().max()))


def _errors(got, want):
    return {k: _rel(g, w) for k, g, w in zip(NAMES, got, want)}


def _fp64_errors(enc, dec, sd, x, vit):
    """CUDA encoder against the fp64 encoder of x; CUDA decoder against the fp64 decoder of the same fp32 maps
    (conv01, conv11, conv21, conv31 + vit) it was given, upsampling at fp32's source coordinates as the kernel and the
    fp32 reference do (oracle.fpn.up2_fp32_coords).  x, vit fp32 on the GPU; the fp64 reference runs there too."""
    with torch.no_grad():
        c = enc(x)
        e = _errors(c, OF.fpn_encoder(x.double(), sd))
        ins = [c[0], c[1], c[2], c[3] + vit]
        o = dec(*ins)
        want = OF.fpn_decoder(*[t.double() for t in ins], sd, up2=OF.up2_fp32_coords)
        e.update({k: _rel(g, w) for k, g, w in zip(NAMES[4:], o, want)})
    return e


def test_fpn_fp64_cases_cover_every_layer(dev):
    """on this device, the fp64 cases together run a second tile on some CTA of each of the 13 tensor-core layers and a
    partial tile at its right and at its bottom edge"""
    cov = [_coverage(*c) for c in FP64_CASES]
    missing = []
    for name, *_ in FPN_TC_LAYERS:
        if not any(c[name][0] > c[name][1] for c in cov):
            missing.append(f"{name}: a second tile per CTA")
        if not any(c[name][2] for c in cov):
            missing.append(f"{name}: a ragged right edge")
        if not any(c[name][3] for c in cov):
            missing.append(f"{name}: a ragged bottom edge")
    assert not missing, missing


@pytest.mark.parametrize("N,H,W", FP64_CASES)
def test_fpn_vs_fp64_oracle(dev, N, H, W):
    sd = fpn_state_dict(21)
    x = synth.make_images(N, H, W, seed=H * W).to(dev)
    vit = torch.randn(N, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(3)).to(dev)
    enc, dec = _modules(sd, dev)
    e = _fp64_errors(enc, dec, sd, x, vit)
    rec(f"fpn_fp64_{N}x{H}x{W}", **e)
    assert max(e.values()) < FPN_BAR, e


def test_fpn_encoder_with_vit_feat_vs_fp64(dev):
    """FPNEncoder.forward(x, vit_feat) (mvsf_fpn_encoder_vit_forward, the encoder the model runs): conv31 =
    LeakyReLU(conv31) + vit_feat[n % V] in the last layer's epilogue, N = B V images of B = 2 samples of V = 3 views,
    at a size where conv31 runs a second tile on some CTA"""
    B, V, H, W = 2, 3, 328, 560
    N = B * V
    tiles, bound, _, _ = _coverage(N, H, W)["conv31"]
    assert tiles > bound, (tiles, bound)
    sd = fpn_state_dict(26)
    x = synth.make_images(N, H, W, seed=27).to(dev)
    vit = torch.randn(V, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(28)).to(dev)
    enc, _ = _modules(sd, dev)
    got = enc(x, vit)
    for t, (c, s) in zip(got, ((8, 1), (16, 2), (32, 4), (64, 8))):
        assert tuple(t.shape) == (N, c, H // s, W // s) and not bool(torch.isnan(t).any())
    with torch.no_grad():
        want = OF.fpn_encoder(x.double(), sd)
    want[3] = want[3] + vit.double().repeat(B, 1, 1, 1)   # image n = b V + v takes view v = n % V
    e = _errors(got, want)
    rec(f"fpn_encoder_vit_{B}x{V}x{H}x{W}", **e)
    assert max(e.values()) < FPN_BAR, e


@pytest.mark.parametrize("name", FPN_CASES)
def test_fpn_vs_reference_fixture(dev, name):
    gold, meta = load_golden(name)
    sd = fpn_state_dict(meta["wseed"])
    x, vit = fpn_inputs(gold, meta)
    enc, dec = _modules(sd, dev)
    got = _run_cuda(enc, dec, x.to(dev), vit.to(dev))
    e = _errors([fixture_crop(k, g) for k, g in zip(NAMES, got)], [gold[k] for k in NAMES])
    rec(f"fpn_fixture_{name}", **e)
    assert max(e.values()) < 1e-4, e


@pytest.mark.parametrize("V,H,W", [(5, 1152, 1536), (10, 1088, 1920)])
def test_fpn_full_size_vs_fp64(dev, V, H, W):
    sd = fpn_state_dict(22)
    enc, dec = _modules(sd, dev)
    worst = {}
    for v0 in range(0, V, 5):   # the fp64 restatement holds every full-resolution intermediate: 5 views at a time
        n = min(5, V - v0)
        x = synth.make_images(n, H, W, seed=v0 + 1).to(dev)
        vit = torch.randn(n, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(v0)).to(dev)
        for k, v in _fp64_errors(enc, dec, sd, x, vit).items():
            worst[k] = max(worst.get(k, 0.0), v)
        del x, vit
        torch.cuda.empty_cache()
    rec(f"fpn_fullsize_{V}x{H}x{W}", **worst)
    assert max(worst.values()) < FPN_BAR, worst


def test_fpn_bf16_and_strided_inputs(dev):
    sd = fpn_state_dict(23)
    enc, dec = _modules(sd, dev)
    N, H, W = 2, 64, 96
    big = synth.make_images(N, H, 2 * W, seed=5).to(dev)
    x = big[..., ::2]                                # non-contiguous view
    assert not x.is_contiguous()
    vit = torch.randn(N, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(4)).to(dev)
    e = {}
    for tag, xi, vi in (("strided_fp32", x, vit), ("bf16", x.bfloat16(), vit.bfloat16()),
                        ("channels_last_fp16", x.half().contiguous(memory_format=torch.channels_last), vit.half())):
        c = enc(xi)
        c31 = c[3] + vi                                   # fp32 + bf16 -> fp32, as under autocast
        lat = [t.bfloat16() if tag == "bf16" else t for t in c[:3]]   # bf16 / channels-last views into the decoder
        got = list(c) + list(dec(lat[0], lat[1], lat[2], c31))
        c64 = OF.fpn_encoder(xi.double().cpu(), sd)
        lat64 = [t.double().cpu() for t in lat]
        want = c64 + OF.fpn_decoder(lat64[0], lat64[1], lat64[2], c31.double().cpu(), sd, up2=OF.up2_fp32_coords)
        # encoder outputs against the encoder on the same (rounded) input; decoder against the same decoder inputs
        e[tag] = max(_errors(got, want).values())
    rec("fpn_input_dtypes_strides", **e)
    assert max(e.values()) < FPN_BAR, e


def _hotpath_net(dev, seed=7):
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.hotpath import HotPathNet
    from mvsformerplusplus_b200.params import build_hotpath_params
    args = default_args()
    params = build_hotpath_params(args).eval()
    sd = synth.randomize_state_dict(params, seed=seed)
    net = HotPathNet(args).eval()
    net.load_state_dict(sd, strict=True)
    return args, net.to(dev)


def test_downstream_hotpath_from_cuda_fpn_features(dev):
    """HotPathNet fed from CUDA-FPN features against HotPathNet fed from fp64-oracle-FPN features (fixture size)."""
    gold, meta = load_golden("fpn_n2_64x96")
    sd = fpn_state_dict(meta["wseed"])
    V, H, W = 3, 64, 96
    imgs = synth.make_images(V, H, W, seed=77).unsqueeze(0)
    vit = torch.randn(V, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(78))
    enc, dec = _modules(sd, dev)
    feats_cuda = Pyramid(enc, dec)(imgs.to(dev), vit.to(dev))

    class _E(torch.nn.Module):
        def forward(self, x):
            return OF.fpn_encoder(x, sd)

    class _D(torch.nn.Module):
        def forward(self, *c):
            return OF.fpn_decoder(*c, sd)

    feats_ref = Pyramid(_E(), _D())(imgs.double(), vit.double())
    feats_ref = {k: v.float().to(dev) for k, v in feats_ref.items()}
    args, net = _hotpath_net(dev)
    proj = {k: v.to(dev) for k, v in synth.make_proj_matrices(V, H, W, theta_step=0.12).items()}
    dv = synth.make_depth_values(48, 425.0, 2.65 * 4).to(dev)
    a = net.forward_features(feats_cuda, proj, dv, TMP)
    b = net.forward_features(feats_ref, proj, dv, TMP)
    e = dict(depth_rel=rel_linf(a["refined_depth"].cpu(), b["refined_depth"].cpu()),
             conf=max_abs(a["photometric_confidence"].cpu(), b["photometric_confidence"].cpu()),
             prob4=max_abs(a["stage4"]["prob_volume"].cpu(), b["stage4"]["prob_volume"].cpu()),
             feat=max(max_abs(feats_cuda[k].cpu(), feats_ref[k].cpu()) for k in feats_ref))
    rec("fpn_downstream_hotpath", **e)
    assert e["depth_rel"] < 1e-3 and e["conf"] < 1e-4 and e["prob4"] < 1e-4, e


def test_install_feature_pyramid_under_bf16_autocast(dev):
    """install(model, feature_pyramid=True) on a stub with the reference's glue (encoder -> + vit_feat -> decoder -> FMT ->
    cascade), run under bf16 autocast as test.py:250 does, against the CUDA modules called directly in fp32."""
    from mvsformerplusplus_b200 import hotpath
    from mvsformerplusplus_b200.hotpath import cascade_forward
    from tests.fpn_common import fpn_params
    sd = fpn_state_dict(24)
    args, net = _hotpath_net(dev, seed=8)

    class Stub(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.args = args
            p = fpn_params()
            self.encoder, self.decoder = p.encoder, p.decoder   # parameter containers with the reference's keys
            self.FMT_module, self.fusions = net.FMT_module, net.fusions

        def forward(self, imgs, vit_feat, proj, dv):
            feats = Pyramid(self.encoder, self.decoder)(imgs, vit_feat)
            return cascade_forward(self.FMT_module, self.fusions, self.args, feats, proj, dv, TMP)

    stub = Stub()
    wrap = torch.nn.Module()
    wrap.encoder, wrap.decoder = stub.encoder, stub.decoder
    wrap.load_state_dict(sd, strict=True)
    hotpath.install(stub, feature_pyramid=True)
    stub = stub.to(dev).eval()
    V, H, W = 3, 64, 96
    imgs = synth.make_images(V, H, W, seed=91).unsqueeze(0).to(dev)
    vit = torch.randn(V, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(92)).to(dev)
    proj = {k: v.to(dev) for k, v in synth.make_proj_matrices(V, H, W, theta_step=0.12).items()}
    dv = synth.make_depth_values(48, 425.0, 2.65 * 4).to(dev)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        a = stub(imgs, vit, proj, dv)
    enc, dec = _modules(sd, dev)
    feats = Pyramid(enc, dec)(imgs, vit)
    b = cascade_forward(net.FMT_module, net.fusions, args, feats, proj, dv, TMP)
    e = dict(depth_rel=rel_linf(a["refined_depth"].cpu(), b["refined_depth"].cpu()),
             conf=max_abs(a["photometric_confidence"].cpu(), b["photometric_confidence"].cpu()),
             feat=max(max_abs(a["features"][k].float().cpu(), b["features"][k].float().cpu()) for k in ("stage1", "stage4")))
    rec("fpn_install_autocast", **e)
    assert e["depth_rel"] < 1e-3 and e["conf"] < 1e-4, e
