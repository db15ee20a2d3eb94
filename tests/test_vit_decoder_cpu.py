"""CPU tests of the ViT feature decoder (models/module.py:273-364): the torch restatement in oracle/vit_decoder.py against
the reference-executed fixtures, state-dict keys, the packed weights (BN folding, gather-form transposed convs), config
and argument checks, loud failure on the CPU and the install() seam."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import packing
from oracle import vit_decoder as OV
from tests.common import ROOT, load_golden, max_abs
from tests.vit_decoder_common import CASES, make_tokens, shipped_args, sub_sd, vit_params, vit_state_dict


@pytest.fixture(scope="module")
def lib():
    from mvsformerplusplus_b200.build import build
    build()
    from mvsformerplusplus_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_vit_decoder_matches_reference_fixture(name):
    gold, meta = load_golden(name)
    x = make_tokens(meta)
    sd = vit_state_dict(meta["wseed"])
    with torch.no_grad():
        got = OV.vit_decoder(x, sd, (meta["B"], meta["V"], meta["h"], meta["w"], 768))
    want = gold["out"]
    assert got.shape == want.shape
    assert max_abs(got, want) <= 1e-5 * max(1.0, float(want.abs().max()))


def test_vit_decoder_state_dict_keys_match_reference_inventory():
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    ref = {}
    for line in open(os.path.join(ROOT, "tests", "golden", "vit_decoder_state_dict_keys.txt")):
        k, s = line.strip().split(" ", 1)
        ref[k] = eval(s)
    assert {k: tuple(v.shape) for k, v in vit_params().state_dict().items()} == ref
    got = {"decoder_vit." + k: tuple(v.shape) for k, v in CrossVITDecoder(shipped_args()).state_dict().items()}
    assert got == ref


def test_vit_decoder_two_part_packing_folds_bn_and_gathers_transposed_convs():
    sd = sub_sd(vit_state_dict(5), "decoder_vit.")
    gemm, small = (t.double() for t in packing.pack_vit_decoder(sd))
    D, G_BLK = 768, 9216 * 768
    ng = 5 * G_BLK + 256 * 9 * D + 4 * 128 * 1024 + 4 * 64 * 512
    sb = 8 * D + 3072   # small parameters per block: 8 vectors of 768 and the fc1 bias
    cb = 5 * sb + 4 * D + 8
    assert gemm.numel() == ng == packing.VIT_DECODER_GEMM_WTS
    assert small.numel() == cb + 448 == packing.VIT_DECODER_SMALL_WTS
    assert float(small[cb - 8]) == pytest.approx(float(sd["prev_values.0"])) and float(small[cb - 7]) == pytest.approx(
        float(sd["prev_values.1"]))
    # the proj conv: [256][tap * 768 + ci] with the BN scale folded, the folded shift at the conv biases
    x = torch.randn(1, D, 5, 6, dtype=torch.float64)
    w = gemm[5 * G_BLK:5 * G_BLK + 256 * 9 * D].view(256, 3, 3, D).permute(0, 3, 1, 2)
    got = F.conv2d(x, w, small[cb:cb + 256], padding=1)
    t = lambda k: sd["proj.1." + k].double()
    want = F.batch_norm(F.conv2d(x, sd["proj.0.weight"].double(), sd["proj.0.bias"].double(), padding=1),
                        t("running_mean"), t("running_var"), t("weight"), t("bias"), False, 0.0, 1e-5)
    assert max_abs(got, want) < 1e-4
    # upsampler0, every parity class: out[2y+py, 2x+px] = sum over the 2 x 2 gather taps of in[y+dy, x+dx] . W_class
    off = 5 * G_BLK + 256 * 9 * D
    x = torch.randn(1, 256, 4, 5, dtype=torch.float64)
    t = lambda k: sd["upsampler0.1." + k].double()
    want = F.batch_norm(F.conv_transpose2d(x, sd["upsampler0.0.weight"].double(), sd["upsampler0.0.bias"].double(),
                                           stride=2, padding=1),
                        t("running_mean"), t("running_var"), t("weight"), t("bias"), False, 0.0, 1e-5)
    xp = F.pad(x, (1, 1, 1, 1))
    for cls in range(4):
        py, px = cls >> 1, cls & 1
        wc = gemm[off + cls * 128 * 1024:off + (cls + 1) * 128 * 1024].view(128, 4, 256)
        acc = small[cb + 256:cb + 384].view(1, 128, 1, 1).expand(1, 128, 4, 5).clone()
        for ti, (dy, _) in enumerate(packing.deconv_class_taps(py)):
            for tj, (dx, _) in enumerate(packing.deconv_class_taps(px)):
                src = xp[:, :, 1 + dy:1 + dy + 4, 1 + dx:1 + dx + 5]
                acc += torch.einsum("nchw,oc->nohw", src, wc[:, 2 * ti + tj])
        assert max_abs(acc, want[:, :, py::2, px::2]) < 1e-4, cls


@pytest.mark.parametrize("key,value", [
    ("ffn_type", "glu"), ("attention_type", "FLASH2"), ("attention_type", "XFormers"),
    ("self_cross_types", ["Linear", "FLASH2"]), ("post_norm", True), ("no_combine_norm", True), ("pre_norm_query", False),
    ("d_model", 1024), ("nhead", 16), ("init_values", None)])
def test_vit_decoder_rejects_unsupported_decoder_cfg(key, value):
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    with pytest.raises(NotImplementedError, match=key):
        CrossVITDecoder(shipped_args(**{key: value}))


def test_vit_decoder_rejects_other_widths_and_interval_layers():
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    for k, v in (("vit_ch", 1024), ("out_ch", 32)):
        a = shipped_args()
        a[k] = v
        with pytest.raises(NotImplementedError, match=k):
            CrossVITDecoder(a)
    a = shipped_args()
    a["dino_cfg"]["cross_interval_layers"] = 4
    with pytest.raises(NotImplementedError, match="cross_interval_layers"):
        CrossVITDecoder(a)


def test_vit_decoder_fails_loudly_on_cpu():
    from mvsformerplusplus_b200.hotpath import CrossVITDecoder
    m = CrossVITDecoder(shipped_args()).eval()
    x = [torch.zeros(1, 2, 12, 768) for _ in range(3)]
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(x, vit_shape=(1, 2, 3, 4, 768))


def test_vit_decoder_entry_points_refuse_bad_arguments_without_touching_the_gpu(lib):
    need = ctypes.c_size_t(0)
    ptr = ctypes.c_void_p(1 << 20)
    lib.mvsf_launch_count(1)
    for B, V, h, w in ((0, 3, 4, 4), (1, 1, 4, 4), (1, 3, 0, 4), (1, 3, 4, 0), (1, 3, 2048, 4), (64, 10, 1000, 1000)):
        assert lib.mvsf_vit_decoder_workspace_bytes(B, V, h, w, ctypes.byref(need)) == -1, (B, V, h, w)
        assert b"vit_decoder" in lib.mvsf_last_error()
        assert lib.mvsf_vit_decoder_forward(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ctypes.c_size_t(1 << 40), B, V, h, w,
                                            None) == -1
    assert lib.mvsf_vit_decoder_workspace_bytes(1, 5, 36, 48, None) == -1
    assert lib.mvsf_vit_decoder_forward(None, ptr, ptr, ptr, ptr, ptr, ptr, ctypes.c_size_t(1 << 40), 1, 3, 4, 4,
                                        None) == -1
    assert b"null pointer" in lib.mvsf_last_error()
    odd = ctypes.c_void_p((1 << 20) + 4)
    assert lib.mvsf_vit_decoder_forward(ptr, odd, ptr, ptr, ptr, ptr, ptr, ctypes.c_size_t(1 << 40), 1, 3, 4, 4,
                                        None) == -1
    assert b"16-byte aligned" in lib.mvsf_last_error()
    assert lib.mvsf_vit_decoder_workspace_bytes(1, 3, 4, 4, ctypes.byref(need)) == 0
    assert lib.mvsf_vit_decoder_forward(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ctypes.c_size_t(need.value - 1), 1, 3, 4, 4,
                                        None) == -3

    # the streamed-weight GEMM seam
    BIAS, GELU, RES, LN, SILU = 0, 1, 3, 5, 6

    def call(epi, M=128, N=768, K=768, lda=None, res=True, gamma=True, C=ptr, ldc=None, C2=None, ldc2=None,
             ws_bytes=1 << 40):
        return lib.mvsf_linear_tc_streamed_epilogue(epi, ptr, lda or K, ptr, ptr, ptr if res else None, N,
                                                    ptr if gamma else None, 0, C, ldc or N, C2, ldc2 or 2 * N, ptr,
                                                    ctypes.c_size_t(ws_bytes), M, N, K, None)

    bad = [
        (dict(epi=LN), b"unknown epilogue"), (dict(epi=4), b"unknown epilogue"), (dict(epi=7), b"unknown epilogue"),
        (dict(epi=BIAS, N=100), b"N % 64 == 0"), (dict(epi=GELU, K=96), b"cin % 64 == 0"),
        (dict(epi=BIAS, C=None), b"bad arguments"), (dict(epi=RES, res=False), b"residual epilogue needs"),
        (dict(epi=RES, gamma=False), b"residual epilogue needs"),
        (dict(epi=SILU, C=ctypes.c_void_p((1 << 20) + 4)), b"C must be 16-byte aligned"),
        (dict(epi=BIAS, C2=ptr, ldc2=1540), b"C2 must be 16-byte aligned"), (dict(epi=BIAS, lda=700), b"need lda >= K"),
        (dict(epi=BIAS, M=0), b"empty shape"),
    ]
    for kw, msg in bad:
        assert call(**kw) == -1, kw
        assert msg in lib.mvsf_last_error(), (kw, lib.mvsf_last_error())
    assert call(BIAS, ws_bytes=1024) == -3 and b"workspace" in lib.mvsf_last_error()
    assert lib.mvsf_launch_count(0) == 0


def _stub():
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    args = default_args()
    model = build_hotpath_params(args)
    model.decoder_vit = vit_params().decoder_vit
    model.args = args
    model.vit_args = shipped_args()
    return model


def test_install_vit_decoder_keeps_the_checkpoint_contract():
    """install(model) leaves decoder_vit alone; install(model, vit_decoder=True) swaps it with every state-dict key and
    value unchanged, so a reference checkpoint still loads with strict=True."""
    from mvsformerplusplus_b200 import hotpath
    model = _stub()
    wrap = torch.nn.Module()
    wrap.decoder_vit = model.decoder_vit
    sd = vit_state_dict(9)
    wrap.load_state_dict(sd, strict=True)
    old = model.decoder_vit
    before = {k: v.clone() for k, v in model.state_dict().items()}
    hotpath.install(model)
    assert model.decoder_vit is old
    hotpath.install(model, feature_pyramid=False, vit_decoder=True)
    assert isinstance(model.decoder_vit, hotpath.CrossVITDecoder)
    after = model.state_dict()
    assert sorted(after) == sorted(before)
    for k in sub_sd(sd, ""):
        assert torch.equal(after[k], before[k]), k
    model.load_state_dict(before, strict=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.decoder_vit([torch.zeros(1, 2, 4, 768)] * 3, vit_shape=(1, 2, 2, 2, 768))


def test_decoder_gemm_tiles_restate_the_streamed_launch():
    """tests/vit_decoder_common.decoder_gemm_tiles restates how the streamed GEMM tiles the decoder's products; a change
    of the tile shape, the grid or the head's GEMM shapes fails here until the restatement follows it"""
    from tests.vit_decoder_common import decoder_gemm_tiles
    src = lambda n: " ".join(open(os.path.join(ROOT, "mvsformerplusplus_b200", "csrc", n)).read().split())
    lin, dec = src("linear_tc.cu"), src("vit_decoder.cu")
    assert "const int ntiles = cdiv(a.M, TC_BM) * (a.N / BN), num_sms = device_sm_count(dev);" in lin
    assert "<<<ntiles < num_sms ? ntiles : num_sms, TC_THREADS, smem, s>>>(a);" in lin
    assert "return a.N % 128 == 0 ? launch_tcs_bn<128>(a, epi, s) : launch_tcs_bn<64>(a, epi, s);" in lin
    for shape in ("a.M = imgs * L; a.N = 256; a.K = 9 * D;", "a.M = imgs * L; a.N = 128; a.K = 1024;",
                  "a.M = imgs * 4 * L; a.N = 64; a.K = 512;", "TcsArgs a = gemm(ws, ws.xn2, 2 * D, D, wb + G_QKV, D, M);",
                  "TcsArgs f1 = gemm(ws, ws.xn2, 2 * D, D, wb + G_FC1, HID, M);"):
        assert shape in dec, shape
    # V = 10 views of 34 x 60 tokens on an H100 SXM's 132 SMs: upsampler0 is the GEMM with the fewest tiles
    t = decoder_gemm_tiles(1, 10, 34, 60)
    assert min(t.values()) == t["upsampler0_class0"] == 160 and t["head_conv"] == 320
