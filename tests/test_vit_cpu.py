"""CPU tests of the DINOv2 ViT backbone (models/dino/dinov2.py:249-266): the torch restatement in oracle/vit.py against
the reference-executed fixtures, state-dict keys, the packed weights and the cached pos embed, config and argument
checks, loud failure on the CPU and the install() seam."""
import ctypes
import math
import os

import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import packing
from oracle import vit as OVT
from tests.common import ROOT, load_golden, max_abs
from tests.vit_common import CASES, VIT_KW, dino_cfg, make_images, sub_sd, vit_params, vit_state_dict


@pytest.fixture(scope="module")
def lib():
    from mvsformerplusplus_b200.build import build
    build()
    from mvsformerplusplus_b200 import _lib
    return _lib.lib()


def _vit(**kw):
    from mvsformerplusplus_b200 import vit_base
    a = dict(VIT_KW)
    cfg = dino_cfg()
    for k, v in kw.items():
        (a if k in a or k not in cfg else cfg)[k] = v
    return vit_base(**a, **cfg)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_vit_matches_reference_fixture(name):
    gold, meta = load_golden(name)
    sd = vit_state_dict(meta["wseed"], meta["harsh"])
    with torch.no_grad():
        got = OVT.vit_interval_features(make_images(meta), sd)
    for i in range(3):
        want = gold[f"out{i}"]
        assert got[i].shape == want.shape == (meta["n"], meta["gh"] * meta["gw"], 768)
        assert max_abs(got[i], want) <= 1e-5 * max(1.0, float(want.abs().max())), i


def test_vit_state_dict_keys_match_reference_inventory():
    ref = {}
    for line in open(os.path.join(ROOT, "tests", "golden", "vit_state_dict_keys.txt")):
        k, s = line.strip().split(" ", 1)
        ref[k] = eval(s)
    assert {k: tuple(v.shape) for k, v in vit_params().state_dict().items()} == ref
    assert {"vit." + k: tuple(v.shape) for k, v in _vit().state_dict().items()} == ref


def test_pack_vit_two_part_layout():
    sd = sub_sd(vit_state_dict(5), "vit.")
    gemm, small = packing.pack_vit(sd)
    assert gemm.dtype == small.dtype == torch.float32
    assert gemm.numel() == packing.VIT_GEMM_WTS and small.numel() == packing.VIT_SMALL_WTS
    D, HID = 768, 3072
    pw = gemm[:D * 640].view(D, 640)
    assert torch.equal(pw[:, :588], sd["patch_embed.proj.weight"].reshape(D, 588))
    assert not pw[:, 588:].any()
    blk = 4 * D * D + 2 * HID * D
    for i in (0, 11):
        o = D * 640 + i * blk
        assert torch.equal(gemm[o:o + 3 * D * D].view(3 * D, D), sd[f"blocks.{i}.attn.qkv.weight"])
        assert torch.equal(gemm[o + 3 * D * D:o + 4 * D * D].view(D, D), sd[f"blocks.{i}.attn.proj.weight"])
        o += 4 * D * D
        assert torch.equal(gemm[o:o + HID * D].view(HID, D), sd[f"blocks.{i}.mlp.fc1.weight"])
        assert torch.equal(gemm[o + HID * D:o + 2 * HID * D].view(D, HID), sd[f"blocks.{i}.mlp.fc2.weight"])
    sb = 15 * D
    assert torch.equal(small[2 * D:5 * D], sd["blocks.0.attn.qkv.bias"])
    assert torch.equal(small[11 * sb + 14 * D:12 * sb], sd["blocks.11.ls2.gamma"])
    assert torch.equal(small[12 * sb:12 * sb + D], sd["patch_embed.proj.bias"])
    assert torch.equal(small[12 * sb + D:12 * sb + 2 * D], sd["cls_token"].reshape(D))
    assert torch.equal(small[12 * sb + 3 * D:], sd["norm.bias"])


@pytest.mark.parametrize("gh,gw", [(3, 4), (36, 48), (5, 5), (37, 37), (1, 1369)])
def test_cached_pos_embed_is_the_reference_formula(gh, gw):
    """dinov2.py:176-200: the 37 x 37 grid of a square image keeps pos_embed; every other grid (also a square one, and
    1 x 1369) is bicubic with scale_factor ((gh + 0.1) / 37, (gw + 0.1) / 37) - not size=(gh, gw)"""
    pos = vit_state_dict(6)["vit.pos_embed"]
    got = packing.vit_pos_embed(pos, gh, gw)
    assert got.shape == (gh * gw + 1, 768) and got.dtype == torch.float32 and got.is_contiguous()
    if gh == gw == 37:
        assert torch.equal(got, pos[0])
        return
    N = pos.shape[1] - 1
    w0, h0 = gh + 0.1, gw + 0.1
    want = F.interpolate(pos[:, 1:].float().reshape(1, 37, 37, 768).permute(0, 3, 1, 2),
                         scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)), mode="bicubic")
    want = torch.cat([pos[:, :1], want.permute(0, 2, 3, 1).view(1, -1, 768)], 1)[0]
    assert torch.equal(got, want)
    if (gh, gw) == (36, 48):
        by_size = F.interpolate(pos[:, 1:].reshape(1, 37, 37, 768).permute(0, 3, 1, 2), size=(gh, gw), mode="bicubic")
        assert float((by_size.permute(0, 2, 3, 1).reshape(-1, 768) - got[1:]).abs().max()) > 1e-2


@pytest.mark.parametrize("kw", [
    dict(patch_size=16), dict(img_size=224), dict(block_chunks=1), dict(ffn_layer="swiglufused"), dict(init_values=None),
    dict(softmax_scale="entropy_invariance"), dict(dino_layer_idxs=[2, 5, 8]), dict(cross_interval_layers=4),
    dict(embed_dim=1024), dict(depth=24), dict(num_heads=16)])
def test_vit_rejects_unsupported_config(kw):
    from mvsformerplusplus_b200.hotpath import DinoVisionTransformer
    k = next(iter(kw))
    with pytest.raises(NotImplementedError, match=k):
        if k in ("embed_dim", "depth", "num_heads"):   # vit_base fixes these, as in the reference
            a = dict(VIT_KW, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4)
            a.update(kw)
            DinoVisionTransformer(**a, **dino_cfg())
        else:
            _vit(**kw)


def test_vit_accepts_flash2_flag_with_the_same_state_dict():
    a, b = _vit(use_flash2_dino=True), _vit()
    assert list(a.state_dict()) == list(b.state_dict())
    assert a.embed_dim == 768 and a.patch_size == 14


def test_vit_call_time_refusals():
    m = _vit().eval()
    x = torch.zeros(1, 3, 28, 42)
    with pytest.raises(NotImplementedError, match="masks"):
        m.forward_interval_features(x, masks=torch.zeros(1, 6, dtype=torch.bool))
    with pytest.raises(NotImplementedError, match="list"):
        m.forward_interval_features([x])
    with pytest.raises(AssertionError, match="height"):
        m.forward_interval_features(torch.zeros(1, 3, 27, 42))
    with pytest.raises(AssertionError, match="width"):
        m.forward_interval_features(torch.zeros(1, 3, 28, 40))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.forward_interval_features(x)
    with pytest.raises(NotImplementedError, match="eval"):
        m.train().forward_interval_features(x)


def test_vit_and_split_abi_refuse_bad_arguments_without_touching_the_gpu(lib):
    need = ctypes.c_size_t(0)
    ptr = ctypes.c_void_p(1 << 20)
    big = ctypes.c_size_t(1 << 40)
    lib.mvsf_launch_count(1)
    for n, gh, gw in ((0, 3, 4), (-1, 3, 4), (1, 0, 4), (1, 3, 0), (1, -2, 4), (1, 3, -1), (1, 1025, 4),
                      (64, 200, 200)):
        assert lib.mvsf_vit_workspace_bytes(n, gh, gw, ctypes.byref(need)) == -1, (n, gh, gw)
        assert b"vit" in lib.mvsf_last_error()
        assert lib.mvsf_vit_forward(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, big, n, gh, gw, None) == -1
    assert lib.mvsf_vit_workspace_bytes(1, 3, 4, None) == -1
    for k in range(7):   # every output / input pointer null in turn
        args = [ptr] * 8
        args[k] = None
        assert lib.mvsf_vit_forward(*args, big, 1, 3, 4, None) == -1
        assert b"null pointer" in lib.mvsf_last_error()
    odd = ctypes.c_void_p((1 << 20) + 4)
    assert lib.mvsf_vit_forward(odd, ptr, ptr, ptr, ptr, ptr, ptr, ptr, big, 1, 3, 4, None) == -1
    assert b"16-byte aligned" in lib.mvsf_last_error()
    assert lib.mvsf_vit_workspace_bytes(2, 3, 4, ctypes.byref(need)) == 0
    assert lib.mvsf_vit_forward(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ctypes.c_size_t(need.value - 1), 2, 3, 4,
                                None) == -3
    assert b"workspace" in lib.mvsf_last_error()
    # the split that makes wts_tc
    assert lib.mvsf_split_weights_f16(None, ptr, ctypes.c_size_t(packing.VIT_GEMM_WTS), None) == -1
    assert lib.mvsf_split_weights_f16(ptr, ptr, ctypes.c_size_t(packing.VIT_GEMM_WTS + 4), None) == -1
    assert b"split_weights_f16" in lib.mvsf_last_error()
    # the attention seam
    for n, N in ((0, 10), (1, 0), (-1, 10), (1, -5)):
        assert lib.mvsf_vit_attention_forward(ptr, 2304, ptr, 768, ptr, big, n, N, None) == -1
    assert lib.mvsf_vit_attention_forward(None, 2304, ptr, 768, ptr, big, 1, 10, None) == -1
    assert lib.mvsf_vit_attention_forward(ptr, 2304, None, 768, ptr, big, 1, 10, None) == -1
    assert lib.mvsf_vit_attention_forward(ptr, 2300, ptr, 768, ptr, big, 1, 10, None) == -1
    assert lib.mvsf_vit_attention_forward(ptr, 2304, odd, 768, ptr, big, 1, 10, None) == -1
    assert lib.mvsf_vit_attention_forward(ptr, 2304, ptr, 768, ptr, ctypes.c_size_t(12 * 100352 - 1), 1, 10,
                                          None) == -3
    assert lib.mvsf_launch_count(0) == 0


def _stub():
    from mvsformerplusplus_b200.config import default_args
    from mvsformerplusplus_b200.params import build_hotpath_params
    args = default_args()
    model = build_hotpath_params(args)
    model.vit = vit_params().vit
    model.args = args
    model.vit_args = dict(args, dino_cfg=dino_cfg())
    return model


def _check_install(model, sd):
    from mvsformerplusplus_b200 import hotpath
    old = model.vit
    before = {k: v.clone() for k, v in model.state_dict().items()}
    hotpath.install(model)
    assert model.vit is old
    hotpath.install(model, vit=True)
    assert isinstance(model.vit, hotpath.DinoVisionTransformer) and not model.vit.training
    assert model.vit.embed_dim == 768 and model.vit.patch_size == 14
    after = model.state_dict()
    assert sorted(after) == sorted(before)
    for k in sd:
        assert torch.equal(after[k], before[k]), k
    model.load_state_dict(before, strict=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.vit.forward_interval_features(torch.zeros(1, 3, 28, 28))


def test_install_vit_keeps_the_checkpoint_contract():
    """install(model) leaves model.vit alone; install(model, vit=True) swaps it with every state-dict key and value
    unchanged, so a reference checkpoint still loads with strict=True."""
    model = _stub()
    wrap = torch.nn.Module()
    wrap.vit = model.vit
    sd = vit_state_dict(9)
    wrap.load_state_dict(sd, strict=True)
    _check_install(model, sd)


def test_install_vit_on_the_reference_model():
    from oracle.ref_hotpath import reference_root
    root = reference_root()
    if root is None or not os.path.isdir(os.path.join(root, "config")):
        pytest.skip("reference modules not available")
    from oracle.gen_golden_vit import reference_vit_base
    reference_vit_base(root)
    import json
    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    cfg = json.load(open(os.path.join(root, "config", "mvsformer++.json")))["arch"]["args"]
    model = DINOv2MVSNet(cfg).eval()
    wrap = torch.nn.Module()
    wrap.vit = model.vit
    sd = {k: v for k, v in vit_state_dict(10).items()}
    wrap.load_state_dict(sd, strict=True)
    _check_install(model, sd)
