"""GPU tests of the whole model (hotpath.DINOv2MVSNet: images to depth maps, DINOv2_mvsformer_model.py:68-179):
  * against the reference-executed fixtures tests/golden/model_*.npz, at the north-star bars (1e-3 relative depth, 1e-4
    probability) or 3x the full-model oracle's own fp32-versus-fp64 floor where that floor is above a third of a bar;
  * against the path there was before it, the reference's glue around install(feature_pyramid, vit_decoder, vit), on the
    same weights at the fixture sizes and at DTU full size: one ViT / encoder / decoder call for all views, the fused
    conv31 + vit_feat and the direct feature layout change nothing beyond the resize's operation order;
  * the bicubic resize fused into the ViT's patch embedding against F.interpolate + forward_interval_features;
  * bf16 autocast changes nothing; the error paths; PrefetchingRunner with image batches.
Errors go to rec()."""
import pytest
import torch
import torch.nn.functional as F

from mvsformerplusplus_b200 import synth
from oracle import model as OM
from tests.common import TMP, max_abs, rec, rel_linf
from tests.model_common import (CASES, cuda_model, fixture, fixture_errors, fixture_outputs, installed_glue_model,
                                make_inputs, model_args, model_state_dict, to_double, within_bars)
from tests.vit_common import cuda_vit, vit_state_dict

pytestmark = pytest.mark.gpu
# stage features of two GPU paths, relative to max(1, max|feature|).  Measured on an H100: 0 (bit-identical) at every size,
# for the features, the outputs and the fused resize against F.interpolate
FEATURE_BAR = 1e-4


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


def _to(x, dev):
    return {k: v.to(dev) for k, v in x.items()} if isinstance(x, dict) else x.to(dev)


@pytest.mark.parametrize("name", sorted(CASES))
def test_model_vs_reference_fixture(dev, name):
    gold, meta, imgs, proj, dv = fixture(name)
    sd = model_state_dict(meta["wseed"])
    net = cuda_model(sd, dev)
    out = net(imgs.to(dev), _to(proj, dev), dv.to(dev), TMP)
    fpn = net.extract_features(imgs.to(dev))
    e = fixture_errors(meta, out, fpn, gold)
    # the reference's own noise on this fixture: the oracle in fp32 against the oracle in fp64
    args = model_args()
    o32 = OM.model_forward(imgs, proj, dv, sd, args)
    o64 = OM.model_forward(imgs.double(), {k: v.double() for k, v in proj.items()}, dv.double(), to_double(sd), args)
    floor = fixture_errors(meta, o32, o32["features_fpn"], fixture_outputs(meta, o64, o64["features_fpn"]))
    rec(f"model_fixture_{name}", **e, **{f"floor_{k}": v for k, v in floor.items()})
    over = within_bars(e, floor)
    assert not over, over


def _compare(out, want, fpn, fpn_want):
    e = {f"features_{k}": max_abs(fpn[k], fpn_want[k]) / max(1.0, float(fpn_want[k].abs().max())) for k in fpn_want}
    e["refined_depth"] = rel_linf(out["refined_depth"], want["refined_depth"])
    e["photometric_confidence"] = max_abs(out["photometric_confidence"], want["photometric_confidence"])
    for s in range(1, 5):
        so, sw = out[f"stage{s}"], want[f"stage{s}"]
        e[f"s{s}_depth"] = rel_linf(so["depth"], sw["depth"])
        e[f"s{s}_prob"] = max_abs(so["prob_volume"], sw["prob_volume"])
        e[f"s{s}_conf"] = max_abs(so["photometric_confidence"], sw["photometric_confidence"])
    return e


SIZES = {name: CASES[name] for name in CASES}
SIZES["dtu"] = dict(B=1, V=5, H=1152, W=1536, numdepth=192, iseed=321, wseed=322)


@pytest.mark.parametrize("name", sorted(SIZES))
def test_model_vs_installed_seams(dev, name):
    c = SIZES[name]
    sd = model_state_dict(c["wseed"])
    imgs, proj, dv = (_to(x, dev) for x in make_inputs(c))
    glue = installed_glue_model(sd, dev)
    want = glue(imgs, proj, dv, TMP)
    fpn_want = glue.extract_features(imgs)
    del glue
    net = cuda_model(sd, dev)
    out = net(imgs, proj, dv, TMP)
    fpn = net.extract_features(imgs)
    for k in fpn:
        assert fpn[k].shape == fpn_want[k].shape and fpn[k].is_contiguous()
    e = _compare(out, want, fpn, fpn_want)
    rec(f"model_vs_installed_{name}", **e)
    assert max(v for k, v in e.items() if k.startswith("features")) < FEATURE_BAR, e
    assert e["refined_depth"] < 1e-3, e
    for s in (1, 2):
        assert e[f"s{s}_prob"] < 1e-4 and e[f"s{s}_conf"] < 1e-4 and e[f"s{s}_depth"] < 1e-3, (s, e)


@pytest.mark.parametrize("n,H,W", [(5, 1152, 1536), (10, 1088, 1920), (2, 96, 128)])
def test_vit_fused_bicubic_resize(dev, n, H, W):
    vit = cuda_vit(vit_state_dict(44), dev)
    imgs = synth.make_images(n, H, W, seed=H + W).to(dev)
    size = OM.vit_size(H, W, 0.4375)
    got = vit.forward_interval_features_resized(imgs, size)
    resized = F.interpolate(imgs, size, mode="bicubic", align_corners=False)
    want = vit.forward_interval_features(resized)
    e = [max_abs(g, w) / max(1.0, float(w.abs().max())) for g, w in zip(got, want)]
    rec(f"model_vit_fused_resize_{n}x{H}x{W}", out0=e[0], out1=e[1], out2=e[2])
    assert max(e) < 1e-4, e


def test_autocast_changes_nothing(dev):
    gold, meta, imgs, proj, dv = fixture("model_b2v2_64x96")
    net = cuda_model(model_state_dict(meta["wseed"]), dev)
    imgs, proj, dv = imgs.to(dev), _to(proj, dev), dv.to(dev)
    want = net(imgs, proj, dv, TMP)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        got = net(imgs, proj, dv, TMP)
    assert got["refined_depth"].dtype == torch.float32
    assert torch.equal(got["refined_depth"], want["refined_depth"])
    assert torch.equal(got["photometric_confidence"], want["photometric_confidence"])
    for s in range(1, 5):
        assert torch.equal(got[f"stage{s}"]["prob_volume"], want[f"stage{s}"]["prob_volume"])


def test_error_paths(dev):
    from mvsformerplusplus_b200 import DINOv2MVSNet
    net = cuda_model(model_state_dict(5), dev)
    imgs, proj, dv = make_inputs(dict(B=1, V=2, H=64, W=96, numdepth=48, iseed=1))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        net(imgs, proj, dv, TMP)
    with pytest.raises(ValueError, match="multiples of 32"):
        net(torch.zeros(1, 2, 3, 72, 96, device=dev), _to(proj, dev), dv.to(dev), TMP)
    with pytest.raises(NotImplementedError, match="eval"):
        net.train()(imgs.to(dev), _to(proj, dev), dv.to(dev), TMP)
    assert isinstance(net, DINOv2MVSNet)


def test_prefetching_runner_runs_the_model_on_image_batches(dev):
    """streaming.PrefetchingRunner with (imgs, proj_matrices, depth_values) batches returns what a direct forward on
    device-resident inputs returns, for alternating batches, with and without prefetch"""
    from mvsformerplusplus_b200.streaming import PrefetchingRunner
    net = cuda_model(model_state_dict(9), dev)
    batches = []
    for seed in (11, 12, 13):
        x, p, d = make_inputs(dict(B=1, V=3, H=64, W=96, numdepth=48, iseed=seed))
        batches.append((x.pin_memory(), {k: v.pin_memory() for k, v in p.items()}, d.pin_memory()))
    want = []
    for x, p, d in batches:
        out = net(x.to(dev), _to(p, dev), d.to(dev), TMP)
        want.append((out["refined_depth"].clone(), out["photometric_confidence"].clone()))
    runner = PrefetchingRunner(net, dev)
    assert runner.bytes_per_batch(batches[0]) == sum(t.numel() * 4 for t in runner._flat(batches[0]))
    order = [0, 1, 2, 0, 2, 1, 1]
    for i, b in enumerate(order):
        nxt = batches[order[i + 1]] if i + 1 < len(order) and i % 3 != 2 else None   # every third call: no prefetch
        out = runner.run(batches[b], next_batch=nxt, tmp=TMP)
        torch.cuda.synchronize()
        assert torch.equal(out["refined_depth"], want[b][0]), f"call {i} (batch {b})"
        assert torch.equal(out["photometric_confidence"], want[b][1])
