"""GPU tests of the FPN feature pyramid (csrc/fpn.cu through hotpath.FPNEncoder / FPNDecoder) against the fp64 torch
restatement of models/module.py:208-270 (oracle/fpn.py), the reference-executed fixtures, the fp32 restatement at full
size, and downstream through the hot path.  Bar: every output within 1e-4 * max(1, max|ref|); errors go to rec()."""
import pytest
import torch

from mvsformerplusplus_b200 import synth
from oracle import fpn as OF
from tests.common import TMP, load_golden, max_abs, rec, rel_linf
from tests.fpn_common import FPN_CASES, Pyramid, fixture_crop, fpn_inputs, fpn_state_dict, sub_sd

pytestmark = pytest.mark.gpu
NAMES = ("conv01", "conv11", "conv21", "conv31", "out0", "out1", "out2", "out3")


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


def _run_cuda(enc, dec, x, vit):
    c = enc(x)
    o = dec(c[0], c[1], c[2], c[3] + vit)
    return list(c) + list(o)


def _run_oracle(sd, x, vit):
    c = OF.fpn_encoder(x, sd)
    return c + OF.fpn_decoder(c[0], c[1], c[2], c[3] + vit, sd)


def _errors(got, want):
    e = {}
    for k, g, w in zip(NAMES, got, want):
        assert tuple(g.shape) == tuple(w.shape), k
        e[k] = max_abs(g.cpu(), w.cpu()) / max(1.0, float(w.abs().max()))
    return e


@pytest.mark.parametrize("N,H,W", [(2, 64, 96), (1, 40, 72), (1, 8, 8), (2, 136, 240), (1, 24, 40)])
def test_fpn_vs_fp64_oracle(dev, N, H, W):
    sd = fpn_state_dict(21)
    x = synth.make_images(N, H, W, seed=H * W)
    vit = torch.randn(N, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(3))
    enc, dec = _modules(sd, dev)
    got = _run_cuda(enc, dec, x.to(dev), vit.to(dev))
    want = _run_oracle(sd, x.double(), vit.double())
    e = _errors(got, want)
    rec(f"fpn_fp64_{N}x{H}x{W}", **e)
    assert max(e.values()) < 1e-4, e


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
def test_fpn_full_size_vs_fp32_torch(dev, V, H, W):
    sd = fpn_state_dict(22)
    enc, dec = _modules(sd, dev)
    worst = {}
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for v0 in range(0, V, 5):   # the fp32 torch restatement holds every full-resolution intermediate: 5 views at a time
            n = min(5, V - v0)
            x = synth.make_images(n, H, W, seed=v0 + 1).to(dev)
            vit = torch.randn(n, 64, H // 8, W // 8, generator=torch.Generator().manual_seed(v0)).to(dev)
            got = _run_cuda(enc, dec, x, vit)
            with torch.no_grad():
                want = _run_oracle(sd, x, vit)
            for k, g, w in zip(NAMES, got, want):
                worst[k] = max(worst.get(k, 0.0), float((g - w).abs().max()) / max(1.0, float(w.abs().max())))
            del got, want
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    rec(f"fpn_fullsize_{V}x{H}x{W}", **worst)
    assert max(worst.values()) < 1e-4, worst


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
        want = c64 + OF.fpn_decoder(lat64[0], lat64[1], lat64[2], c31.double().cpu(), sd)
        # encoder outputs against the encoder on the same (rounded) input; decoder against the same decoder inputs
        e[tag] = max(_errors(got, want).values())
    rec("fpn_input_dtypes_strides", **e)
    assert max(e.values()) < 1e-4, e


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
