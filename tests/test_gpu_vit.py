"""GPU tests of the DINOv2 ViT backbone (csrc/vit.cu through hotpath.DinoVisionTransformer) and of its softmax attention
(csrc/vit_attention.cuh, mvsf_vit_attention_forward) against fp64 references, up to the shipped sizes, the
reference-executed fixtures, and through install() with the reference's glue.
Bars: attention within 2e-4 * max|ref| (fp16 P, measured worst 1.2e-4); every module output within
1e-4 * max(1, max|ref|).  Errors go to rec()."""

import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import _lib, synth
from oracle import vit as OVT
from tests.common import load_golden, max_abs, rec
from tests.fpn_common import fpn_state_dict
from tests.vit_common import CASES, OracleViT, cuda_vit, dino_cfg, make_images, vit_state_dict
from tests.vit_decoder_common import (OracleFPNDecoder, OracleFPNEncoder, OracleViTDecoder, shipped_args,
                                      vit_state_dict as decoder_state_dict)

pytestmark = pytest.mark.gpu
ATT_BAR, BAR = 2e-4, 1e-4


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _attention(qkv, n, N, ldo=776):
    """qkv [n*N][ldq] (row stride ldq >= 2304) -> out [n*N][ldo] NaN-filled, valid columns [:768]"""
    out = torch.full((n * N, ldo), float("nan"), device=qkv.device)
    ws = torch.empty(n * 12 * ((N + 127) // 128) * 100352 // 4 + 64, device=qkv.device)
    _lib.call("mvsf_vit_attention_forward", qkv, qkv.stride(0), out, ldo, ws, ws.numel() * 4, n, N)
    return out


def _attention_ref(qkv, n, N):
    x = qkv[:, :2304].double().reshape(n, N, 3, 12, 64).permute(2, 0, 3, 1, 4)
    out = torch.empty(n, N, 768, dtype=torch.float64, device=qkv.device)
    for b in range(n):
        a = torch.softmax((x[0, b] * 0.125) @ x[1, b].transpose(-2, -1), dim=-1)
        out[b] = (a @ x[2, b]).transpose(0, 1).reshape(N, 768)
    return out.reshape(n * N, 768)


def _check_attention(tag, qkv, n, N):
    out = _attention(qkv, n, N)
    got = out[:, :768]
    assert bool(torch.isfinite(got).all()), tag
    assert bool(torch.isnan(out[:, 768:]).all()), tag
    want = _attention_ref(qkv, n, N)
    e = float((got.double() - want).abs().max()) / float(want.abs().max())
    rec(f"vit_attention_{tag}", rel=e, max_ref=float(want.abs().max()))
    assert e < ATT_BAR, (tag, e)
    return e


@pytest.mark.parametrize("N", [2, 13, 127, 128, 129, 1370, 1729, 2041])
@pytest.mark.parametrize("n", [1, 3, 5])
def test_vit_attention_vs_fp64(dev, n, N):
    g = torch.Generator(device=dev).manual_seed(n * 10000 + N)
    qkv = 1.5 * torch.randn(n * N, 2304 + 12, device=dev, generator=g)   # strided rows, logits of a few units
    _check_attention(f"n{n}_N{N}", qkv, n, N)


def test_vit_attention_harsh_logits(dev):
    """logits up to about +-40 and one key that dominates most rows"""
    n, N = 2, 1729
    g = torch.Generator(device=dev).manual_seed(7)
    qkv = 3.5 * torch.randn(n * N, 2304, device=dev, generator=g)
    x = qkv.view(n, N, 3, 12, 64)
    u = F.normalize(torch.randn(12, 64, device=dev, generator=g), dim=-1)
    x[:, :, 0] += 3.0 * u
    x[:, 7, 1] = 30.0 * u
    logits = torch.einsum("bqhd,bkhd->bhqk", x[:, :, 0], x[:, :, 1]) * 0.125
    assert float(logits.abs().max()) > 35.0
    del logits
    _check_attention("harsh", qkv, n, N)


def test_vit_attention_underflowing_rows(dev):
    """every score of some rows below -150 (online-softmax underflow): those rows must still be the softmax average"""
    n, N = 1, 1370
    g = torch.Generator(device=dev).manual_seed(8)
    qkv = torch.randn(n * N, 2304, device=dev, generator=g)
    x = qkv.view(N, 3, 12, 64)
    v = F.normalize(torch.randn(12, 64, device=dev, generator=g), dim=-1)
    x[:, 1] = 0.05 * x[:, 1] + 5.0 * v
    x[::5, 0] = -270.0 * v + 0.2 * x[::5, 0]
    logits = torch.einsum("qhd,khd->hqk", x[::5, 0], x[:, 1]) * 0.125
    assert float(logits.max()) < -150.0
    _check_attention("underflow", qkv, n, N)


def _fwd(m, img):
    return m.forward_interval_features(img)


def _errors(got, want):
    return [float((g.double() - w.double()).abs().max()) / max(1.0, float(w.abs().max())) for g, w in zip(got, want)]


GRIDS = [(1, 2, 3), (2, 3, 4), (3, 5, 7), (1, 37, 37), (2, 9, 11), (1, 4, 4)]
SHIPPED = [(5, 36, 48), (10, 34, 60)]   # the ViT inputs of DTU and Tanks and Temples
# kind "uniform": measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), worst 6.9e-6 (1 x 4 x 4)
UNIFORM_BAR = 2e-5


@pytest.mark.parametrize("n,gh,gw,kind", [(1, 2, 3, ""), (2, 3, 4, ""), (3, 5, 7, ""), (1, 37, 37, ""), (2, 9, 11, ""),
                                          (1, 4, 4, "harsh"), (2, 9, 11, "small")] +
                         [g + ("",) for g in SHIPPED] + [g + ("uniform",) for g in GRIDS + SHIPPED])
def test_vit_vs_fp64_oracle(dev, n, gh, gw, kind):
    """The interval features against the fp64 oracle, computed by torch on the device (its attention matrix is about
    4 GB at 10 x 34 x 60).
    kind "small": images, patch bias, pos_embed and cls token scaled by 1e-2, so the tokens entering block 0 have a
    variance near 1e-4, where the LayerNorm eps (1e-6 in the ViT, not the decoder's 1e-5) changes the result.
    kind "uniform": the query projection (attn.qkv.weight[:768] and its bias) zeroed in every block, so every score is
    exactly 0, P is exactly 2^14 and the whole ViT is an fp32-class computation held to UNIFORM_BAR: its GEMMs,
    LayerNorms, the cls-last token rows and the hi|lo attention output.  Uniform attention gives every token of an image
    the same attention output, so a row permutation inside the proj GEMM's input would not show here; the normal
    weights and test_gpu_attention_exact.py cover how tokens mix."""
    sd = vit_state_dict(41, kind == "harsh")
    img = synth.make_images(n, 14 * gh, 14 * gw, seed=n * 100 + gh * 10 + gw).to(dev)
    if kind == "small":
        img = 1e-2 * img
        for k in ("vit.patch_embed.proj.bias", "vit.pos_embed", "vit.cls_token"):
            sd[k] = 1e-2 * sd[k]
    if kind == "uniform":
        for i in range(12):
            for k in (f"vit.blocks.{i}.attn.qkv.weight", f"vit.blocks.{i}.attn.qkv.bias"):
                sd[k] = sd[k].clone()
                sd[k][:768] = 0.0
    got = _fwd(cuda_vit(sd, dev), img)
    with torch.no_grad():
        want = OVT.vit_interval_features(img.double(), sd)
    for o in got:
        assert o.shape == (n, gh * gw, 768) and o.dtype == torch.float32 and o.is_contiguous() and o.data_ptr() % 16 == 0
    e = _errors(got, want)
    del want
    rec(f"vit_fp64_{n}x{gh}x{gw}{'_' + kind if kind else ''}", out0=e[0], out1=e[1], out2=e[2])
    assert max(e) < (UNIFORM_BAR if kind == "uniform" else BAR), e


@pytest.mark.parametrize("name", sorted(CASES))
def test_vit_vs_reference_fixture(dev, name):
    gold, meta = load_golden(name)
    got = _fwd(cuda_vit(vit_state_dict(meta["wseed"], meta["harsh"]), dev), make_images(meta).to(dev))
    e = [max_abs(got[i].cpu(), gold[f"out{i}"]) / max(1.0, float(gold[f"out{i}"].abs().max())) for i in range(3)]
    rec(f"vit_fixture_{name}", out0=e[0], out1=e[1], out2=e[2])
    assert max(e) < BAR, e


def test_vit_bf16_and_strided_inputs(dev):
    sd = vit_state_dict(43)
    m = cuda_vit(sd, dev)
    n, gh, gw = 2, 4, 6
    img = synth.make_images(n, 14 * gh + 3, 14 * gw, seed=3).to(dev)
    strided = img[:, :, 3:]
    assert not strided.is_contiguous()
    e = {}
    for tag, x in (("strided_fp32", strided), ("bf16", strided.bfloat16())):
        got = _fwd(m, x)
        want = OVT.vit_interval_features(x.double(), sd)
        e[tag] = max(_errors(got, want))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        got = _fwd(m, strided)
    assert all(o.dtype == torch.float32 for o in got)
    e["autocast"] = max(_errors(got, OVT.vit_interval_features(strided.double(), sd)))
    rec("vit_input_dtypes_strides", **e)
    assert max(e.values()) < BAR, e


def test_install_vit_decoder_and_fpn_under_bf16_autocast(dev):
    """install(stub, feature_pyramid=True, vit_decoder=True, vit=True) on a stub with the reference's glue (bicubic resize
    -> ViT -> vit_forward's reshape -> decoder -> bilinear resize to H/8 x W/8 -> conv31 + vit_feat -> FPN decoder,
    DINOv2_mvsformer_model.py:55-98) under bf16 autocast, against the unswapped stub (fp32 torch) outside autocast."""
    from mvsformerplusplus_b200 import hotpath
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params

    class Stub(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.args = default_args()
            self.vit_args = dict(shipped_args(), rescale=0.4375)
            self.vit_args["dino_cfg"] = dict(dino_cfg(), decoder_cfg=self.vit_args["dino_cfg"]["decoder_cfg"])
            hp = build_hotpath_params(self.args)
            self.FMT_module, self.fusions = hp.FMT_module, hp.fusions
            self.encoder, self.decoder, self.decoder_vit = OracleFPNEncoder(), OracleFPNDecoder(), OracleViTDecoder()
            self.vit = OracleViT()

        def forward(self, imgs):
            B, V, _, H, W = imgs.shape
            vh, vw = int(H * self.vit_args["rescale"] // 14 * 14), int(W * self.vit_args["rescale"] // 14 * 14)
            vit_imgs = F.interpolate(imgs.reshape(B * V, 3, H, W), (vh, vw), mode="bicubic", align_corners=False)
            vit_out = [v.reshape(B, V, -1, self.vit.embed_dim) for v in self.vit.forward_interval_features(vit_imgs)]
            vit_feat = self.decoder_vit(vit_out, vit_shape=[B, V, vh // 14, vw // 14, 768])
            vit_feat = F.interpolate(vit_feat, size=(H // 8, W // 8), mode="bilinear", align_corners=False)
            feats = [[], [], [], []]
            for vi in range(V):
                c01, c11, c21, c31 = self.encoder(imgs[:, vi])
                c31 = c31 + vit_feat[vi].unsqueeze(0)
                for k, f in enumerate(self.decoder.forward(c01, c11, c21, c31)):
                    feats[k].append(f)
            return [torch.stack(f, 1) for f in feats]

    stub = Stub()
    for name, sd in (("fpn", fpn_state_dict(25)), ("decoder_vit", decoder_state_dict(26)), ("vit", vit_state_dict(27))):
        wrap = torch.nn.Module()
        if name == "fpn":
            wrap.encoder, wrap.decoder = stub.encoder, stub.decoder
        else:
            setattr(wrap, name, getattr(stub, name))
        wrap.load_state_dict(sd, strict=True)
    stub = stub.to(dev).eval()
    V, H, W = 3, 128, 192        # ViT input 56 x 84 (4 x 6 patches) -> decoder 16 x 24 -> resized to 16 x 24
    imgs = synth.make_images(V, H, W, seed=95).unsqueeze(0).to(dev)
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            want = stub(imgs)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    hotpath.install(stub, feature_pyramid=True, vit_decoder=True, vit=True)
    assert isinstance(stub.vit, hotpath.DinoVisionTransformer) and isinstance(stub.decoder_vit, hotpath.CrossVITDecoder)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        got = stub(imgs)
    e = {f"stage{k + 1}": float((g_.float() - w_).abs().max()) / max(1.0, float(w_.abs().max()))
         for k, (g_, w_) in enumerate(zip(got, want))}
    rec("vit_install_autocast", **e)
    assert max(e.values()) < BAR, e
