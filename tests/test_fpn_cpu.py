"""CPU tests of the FPN feature pyramid (models/module.py:208-270): the torch restatement in oracle/fpn.py against the
reference-executed fixtures, state-dict keys, BN folding of the packed weights, argument checks, loud failure on the CPU
and the install() seam."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import packing, synth
from mvsformerplusplus_b200.params import FPN_ENCODER_LAYERS
from oracle import fpn as OF
from tests.common import ROOT, load_golden, max_abs
from tests.fpn_common import FPN_CASES, fixture_crop, fpn_inputs, fpn_params, fpn_state_dict, sub_sd

OUT_NAMES = ("conv01", "conv11", "conv21", "conv31", "out0", "out1", "out2", "out3")


@pytest.mark.parametrize("name", FPN_CASES)
def test_oracle_fpn_matches_reference_fixture(name):
    gold, meta = load_golden(name)
    x, vit = fpn_inputs(gold, meta)
    assert max_abs(x, synth.make_images(meta["N"], meta["H"], meta["W"], seed=meta["iseed"])) < 1e-5
    sd = fpn_state_dict(meta["wseed"])
    enc = OF.fpn_encoder(x, sd)
    dec = OF.fpn_decoder(enc[0], enc[1], enc[2], enc[3] + vit, sd)
    for k, out in zip(OUT_NAMES, enc + dec):
        got, want = fixture_crop(k, out), gold[k]
        assert got.shape == want.shape, k
        assert max_abs(got, want) <= 1e-5 * max(1.0, float(want.abs().max())), k


def test_fpn_state_dict_keys_match_reference_inventory():
    from mvsformerplusplus_b200.hotpath import FPNDecoder, FPNEncoder
    ref = {}
    for line in open(os.path.join(ROOT, "tests", "golden", "fpn_state_dict_keys.txt")):
        k, s = line.strip().split(" ", 1)
        ref[k] = eval(s)
    mine = {k: tuple(v.shape) for k, v in fpn_params().state_dict().items()}
    assert mine == ref
    mods = {"encoder.": FPNEncoder([8, 16, 32, 64]), "decoder.": FPNDecoder([8, 16, 32, 64])}
    got = {p + k: tuple(v.shape) for p, m in mods.items() for k, v in m.state_dict().items()}
    assert got == ref


def test_fpn_two_part_packing_folds_conv_bn():
    sd = fpn_state_dict(5)
    x = torch.randn(1, 8, 11, 13, dtype=torch.float64)
    conv, small = (t.double() for t in packing.pack_fpn_encoder(sd))
    # layer 1 (conv01): the first weights of the conv part; its shift follows conv00's [49][3][8] + 8 in the small part
    w = conv[:25 * 64].view(5, 5, 8, 8).permute(3, 2, 0, 1)
    b = small[49 * 3 * 8 + 8:49 * 3 * 8 + 16]
    got = F.conv2d(x, w, b, padding=2)
    want = OF._bn(F.conv2d(x, sd["encoder.conv01.conv.weight"].double(), padding=2), sd, "encoder.conv01.bn.")
    assert max_abs(got, want) < 1e-5
    assert conv.numel() == sum(k * k * ci * co for _, ci, co, k, _ in FPN_ENCODER_LAYERS[1:]) == 132800
    assert small.numel() == 49 * 3 * 8 + sum(co for _, ci, co, k, _ in FPN_ENCODER_LAYERS) == 1528
    conv, small = (t.double() for t in packing.pack_fpn_decoder(sd))
    # out1: the first weights of the conv part, w [9][64][32]; its shift follows out0 (64*64 + 64) and inner1
    # (32*64 + 64) in the small part
    off = 64 * 64 + 64 + 32 * 64 + 64
    x = torch.randn(1, 64, 7, 9, dtype=torch.float64)
    w = conv[:9 * 64 * 32].view(3, 3, 64, 32).permute(3, 2, 0, 1)
    b = small[off:off + 32]
    got = F.conv2d(x, w, b, padding=1)
    want = OF._bn(F.conv2d(x, sd["decoder.out1.0.weight"].double(), sd["decoder.out1.0.bias"].double(), padding=1), sd,
                  "decoder.out1.1.")
    assert max_abs(got, want) < 1e-5
    assert (conv.numel(), small.numel()) == (32256, 7992)


def test_fpn_rejects_unsupported_configurations_and_sizes():
    from mvsformerplusplus_b200.build import build
    build()
    from mvsformerplusplus_b200 import _lib
    from mvsformerplusplus_b200.hotpath import FPNDecoder, FPNEncoder
    with pytest.raises(NotImplementedError, match="feat_chs"):
        FPNEncoder([8, 16, 32, 32])
    with pytest.raises(NotImplementedError, match="norm_type"):
        FPNEncoder([8, 16, 32, 64], norm_type="IN")
    with pytest.raises(NotImplementedError, match="feat_chs"):
        FPNDecoder([16, 32, 64, 128])
    enc = FPNEncoder([8, 16, 32, 64]).eval()
    with pytest.raises(ValueError, match="multiples of 8"):
        enc(torch.zeros(1, 3, 36, 64))
    dec = FPNDecoder([8, 16, 32, 64]).eval()
    with pytest.raises(ValueError, match="multiples of 8"):
        dec(torch.zeros(1, 8, 20, 16), torch.zeros(1, 16, 10, 8), torch.zeros(1, 32, 5, 4), torch.zeros(1, 64, 2, 2))
    L = _lib.lib()
    need = ctypes.c_size_t(0)
    assert L.mvsf_fpn_encoder_workspace_bytes(1, 1080, 1916, ctypes.byref(need)) == -1
    assert b"multiples of 8" in L.mvsf_last_error()
    assert L.mvsf_fpn_decoder_workspace_bytes(1, 36, 64, ctypes.byref(need)) == -1
    rc = L.mvsf_fpn_encoder_forward(None, None, None, None, None, None, None, None, ctypes.c_size_t(0), 1, 36, 64, None)
    assert rc == -1
    assert L.mvsf_fpn_encoder_workspace_bytes(5, 1152, 1536, ctypes.byref(need)) == 0
    assert need.value == 2 * 5 * 1152 * 1536 * 16
    assert L.mvsf_fpn_decoder_workspace_bytes(1, 1080, 1920, ctypes.byref(need)) == 0
    for part in (0, 1):
        assert L.mvsf_fpn_tc_bytes(part, ctypes.byref(need)) == 0 and need.value % 16 == 0 and need.value > 0


def test_fpn_modules_fail_loudly_on_cpu():
    from mvsformerplusplus_b200.hotpath import FPNDecoder, FPNEncoder
    enc = FPNEncoder([8, 16, 32, 64]).eval()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        enc(torch.zeros(1, 3, 16, 16))
    dec = FPNDecoder([8, 16, 32, 64]).eval()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        dec(torch.zeros(1, 8, 16, 16), torch.zeros(1, 16, 8, 8), torch.zeros(1, 32, 4, 4), torch.zeros(1, 64, 2, 2))


def _reference_model():
    from oracle import reference
    if reference.root("models", reference.CONFIG) is None:
        pytest.skip("no reference sources (oracle/_ref is made by build() only where the reference is available)")
    reference.import_models()
    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    torch.manual_seed(0)
    model = DINOv2MVSNet(reference.config()).eval()
    synth.randomize_state_dict(model.FMT_module, seed=3)
    synth.randomize_state_dict(model.fusions, seed=4)
    return model


def test_install_feature_pyramid_keeps_the_checkpoint_contract():
    """install(model, feature_pyramid=True) on a reference-built DINOv2MVSNet swaps encoder / decoder too; every
    state-dict key and value is unchanged, so a reference checkpoint still loads with strict=True."""
    from mvsformerplusplus_b200 import hotpath
    model = _reference_model()
    wrap = torch.nn.Module()
    wrap.encoder, wrap.decoder = model.encoder, model.decoder
    synth.randomize_state_dict(wrap, seed=6)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    old_encoder, old_decoder = model.encoder, model.decoder
    hotpath.install(model)
    assert model.encoder is old_encoder and model.decoder is old_decoder   # default: the FPN stays as it was
    hotpath.install(model, feature_pyramid=True)
    assert isinstance(model.encoder, hotpath.FPNEncoder) and isinstance(model.decoder, hotpath.FPNDecoder)
    after = model.state_dict()
    assert sorted(after.keys()) == sorted(before.keys())
    for k in before:
        assert torch.equal(after[k], before[k]), k
    model.load_state_dict(before, strict=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.encoder(torch.zeros(1, 3, 64, 96))


def test_plain_install_leaves_the_fpn_untouched():
    """Without the reference: a stub carrying the FPN parameter containers keeps them through install()."""
    from mvsformerplusplus_b200 import hotpath
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    args = default_args()
    model = build_hotpath_params(args)
    p = fpn_params()
    model.encoder, model.decoder = p.encoder, p.decoder
    model.args = args
    hotpath.install(model)
    assert model.encoder is p.encoder and model.decoder is p.decoder
    assert isinstance(model.FMT_module, hotpath.FMT_with_pathway)
    sd = synth.randomize_state_dict(p, seed=9)
    hotpath.install(model, feature_pyramid=True)
    assert isinstance(model.encoder, hotpath.FPNEncoder)
    for k, v in sub_sd(sd, "encoder.").items():
        assert torch.equal(model.encoder.state_dict()[k], v), k
    for k, v in sub_sd(sd, "decoder.").items():
        assert torch.equal(model.decoder.state_dict()[k], v), k


def _source(name):
    return " ".join(open(os.path.join(ROOT, "mvsformerplusplus_b200", "csrc", name)).read().split())


def test_fpn_tile_coverage_restates_the_layer_table():
    """tests/fpn_common.py restates the tiling of the 13 tensor-core layers; a retiling of csrc/fpn.cu or a change of
    conv2d_tc.cuh's shared-memory layout fails here until the restatement follows it"""
    from tests.fpn_common import FPN_TC_LAYERS, fpn_coverage
    src = _source("fpn.cu")
    enc = src[src.index("constexpr LayerDesc kEnc[11] = {"):]
    enc = [tuple(int(v) for v in t.split(",")) for t in enc[enc.index("{") + 2:enc.index("}};")].split("}, {")]
    dec = src[src.index("constexpr LayerDesc kDec[3] = {"):]
    dec = [tuple(int(v) for v in t.split(",")) for t in dec[dec.index("{") + 2:dec.index("}};")].split("}, {")]
    mine = [(ci, co, ks, ns) for _, ci, co, ks, _, _, ns, _, _ in FPN_TC_LAYERS]
    assert mine == enc[1:] + [(64, co, 3, ns) for _, co, _, ns in dec]
    assert ("using EncL = Conv<kEnc[I].ci, kEnc[I].co, kEnc[I].ks, (I == 2 || I == 5 || I == 8) ? 2 : 1, "
            "(I >= 8) ? 8 : 16, kEnc[I].ns>;") in src
    assert "using DecL = Conv<64, kDec[K].co, 3, 1, K == 0 ? 8 : 16, kDec[K].ns>;" in src
    assert "constexpr int kLat[3] = {32, 16, 8};" in src
    conv = _source("conv2d_tc.cuh")
    for line in ("PAD = (KS - 1) / 2, HALO = (KS - 1) / S;", "PR = TR + HALO, PC = 32 + HALO;",
                 "NO = CI / 8, NP = S * S, NG = CI < 16 ? 1 : CI / 16, NB = CO / NS;",
                 "PLANE = PR * PC * 16, PITCH = PC * 16;", "BT = 64 * NS;", "WBYTES = KS * KS * NG * BT;",
                 "OFF_W = NP * NO * 2 * PLANE, SMEM = OFF_W + WBYTES;",
                 "long long cap = (long long)per_sm * device_sm_count(dev) / L::NB;"):
        assert line in conv, line
    assert "IR = L::PR + 6, IC = L::PC + 6, NW = 49 * 3 * 8 + 8;" in src and "EXTRA = (3 * IR * IC + NW) * 4;" in src
    assert "EXTRA = (CL * 64 + 64) * 4;" in src
    # an H100 SXM (132 SMs, 228 KB of shared memory per SM): 14 x 264 x 456 loops and is ragged in every layer
    cov = fpn_coverage(14, 264, 456, 132, 228 * 1024)
    assert all(t > b and rx and ry for t, b, rx, ry in cov.values()), cov
    assert cov["downsample2"][:2] == (280, 132) and cov["conv20"][:2] == (280, 264) and cov["conv30"][:2] == (140, 66)
