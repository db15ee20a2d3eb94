"""The training cost volume on the GPU: mvsf_warp_corr_aggregate_backward against fp64 autograd at the kernel's own
sample coordinates (tests/cost_volume_common.py), grazing geometry, the op's forward against the eval kernels bit for bit,
the reference's own training step (tests/golden/train_cost_volume_*.npz), install_training on a reference-shaped model,
memory, reproducibility and errors.  The backward's grid is one CTA per 8 warps of pixels, neither persistent nor strided,
so no case has to make it loop."""
import copy
import itertools

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from mvsformerplusplus_b200 import _lib
from mvsformerplusplus_b200.training import cost_volume, install_training
from oracle import train as OT
from tests import cost_volume_common as R
from tests import train_common as T
from tests.common import rec

pytestmark = pytest.mark.gpu

# |kernel - fp64| <= TOL * max|fp64| per feature-gradient tensor (reference view, source views); for dL/dw, which is a
# difference of two sums, TOL * max over pixels and views of sum_{g,d} |u| (|c_v| + |vm|).  About 3x the worst error
# measured on an H100 SXM (132 SMs, 700 W) over the cases of test_backward_against_fp64 and test_grazing_geometry
GRAD_REF_TOL = 2e-6    # measured 6.0e-7 (C = 64, V = 5)
GRAD_SRC_TOL = 6e-6    # measured 7.7e-7 .. 2.1e-6 over three runs (grazing: many taps share corners, atomics reorder)
GRAD_VIS_TOL = 2e-7    # measured 4.7e-8 (C = 16, V = 5)
# the op on the GPU against the reference's fp32 CPU step (fixture): the fixture's own distance to fp64 (2.0e-5) plus the
# op's; measured 1.9e-5
FIXTURE_GPU_TOL = 1e-4
# stand-in model through install_training against its fp64 restatement, relative to each tensor's max, about 3x the worst
# measured.  fp32 (cuDNN without TF32), eval(): 3.8e-4 (vis.3.bias, a sum over every pixel).  fp32, train(): 1.2e-2 - the
# train-mode BatchNorm of the visibility CNN normalises the entropy map by its batch statistics, which at this small size
# spread little, so the entropy's fp32 rounding reaches every gradient amplified; the outputs stay at 5e-6.  bf16
# autocast, where the stand-in's cost_reg runs in bf16: 5.5e-3 on the outputs; its gradients are only checked finite (bf16
# leaves them 10-25 % off fp64)
WIRING_TOL = {("fp32", "eval"): 1.2e-3, ("fp32", "train"): 4e-2, ("bf16", "eval"): 2e-2, ("bf16", "train"): 2e-2}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _case(dev, C, D, H, W, V, seed, th=0.12):
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(V, H, W, C, generator=g)
    pm = synth.make_proj_matrices(V, H, W, theta_step=th)["stage4"][0]
    base = O.init_inverse_range(synth.make_depth_values(192), D, H, W)[0]
    dd = (base * (1.0 + 0.02 * torch.rand(D, H, W, generator=g))).contiguous()
    vis = 0.05 + torch.rand(V - 1, H, W, generator=g)
    U = torch.randn(D, H, W, 8, generator=g)
    homs = torch.empty(V - 1, 12, device=dev)
    _lib.call("mvsf_compose_geometry", pm.to(dev), V, homs, torch.empty(9, device=dev))
    return f.to(dev), homs, dd.to(dev), vis.to(dev), U.to(dev)


def _kernel(f, homs, dd, vis, U):
    V, H, W, C = f.shape
    D = dd.shape[0]
    vol = torch.empty(D, H, W, 8, device=f.device)
    _lib.call("mvsf_warp_corr_aggregate", f, homs, dd, vis, vol, V, C, 8, D, H, W)
    gf = torch.full_like(f, float("nan"))
    gv = torch.full_like(vis, float("nan"))
    _lib.call("mvsf_warp_corr_aggregate_backward", f, homs, dd, vis, vol, U, gf, gv, V, C, 8, D, H, W)
    return vol, gf, gv


def _fp64(f, homs, dd, vis, U):
    """autograd in fp64 through the bilinear samples at the kernel's fp32 coordinates"""
    V, H, W, C = f.shape
    D = dd.shape[0]
    ix, iy, _ = R.restated_coords(homs, dd)
    feat = f.reshape(V, H * W, C).double().requires_grad_(True)
    w = vis.reshape(V - 1, H * W).double().requires_grad_(True)
    corr = torch.stack([torch.stack([(feat[0] * R.sample(feat[v + 1], ix[v, d], iy[v, d], H, W)).view(-1, 8, C // 8).mean(-1)
                                     for d in range(D)]) for v in range(V - 1)])
    vol = R.aggregate(corr, w)
    U64 = U.reshape(D, H * W, 8).double()
    vol.backward(U64)
    # dL/dw_v = sum u (c_v - vm) cancels (all of it when V = 2); its fp32 error scales with the terms, not the result
    with torch.no_grad():
        u = (U64 / (w.sum(0) + 1e-6)[None, :, None]).abs()
        vis_scale = float((u[None] * (corr.abs() + vol.abs()[None])).sum((1, 3)).max())
    return vol.detach(), feat.grad.view(V, H, W, C), w.grad.view(V - 1, H, W), vis_scale


def _errors(name, got, want):
    vol, gf, gv = got
    vol64, gf64, gv64, vis_scale = want
    e = dict(ref=T.rel(gf[0], gf64[0]), src=T.rel(gf[1:], gf64[1:]), vis=float((gv.double() - gv64).abs().max()) / vis_scale,
             volume=T.rel(vol.view(vol64.shape), vol64))
    rec(f"cost_volume_grad_{name}", **e, finite=bool(torch.isfinite(gf).all() and torch.isfinite(gv).all()))
    return e


SHIPPED = [(64, 32), (32, 16), (16, 8), (8, 4)]


@pytest.mark.parametrize("C,D,V,H,W", [(C, D, V, 36, 52) for (C, D), V in itertools.product(SHIPPED, (2, 3, 5))]
                         + [(8, 12, 3, 36, 52),        # D > 2 C / 4: the upstream gradient is reloaded per chunk
                            (64, 32, 5, 144, 192)])    # DTU stage 1 at full size (1152 x 1536 / 8)
def test_backward_against_fp64(dev, C, D, V, H, W):
    case = _case(dev, C, D, H, W, V, seed=C * 100 + D + V)
    got = _kernel(*case)
    e = _errors(f"C{C}_D{D}_V{V}_{H}x{W}", got, _fp64(*case))
    assert torch.isfinite(got[1]).all() and torch.isfinite(got[2]).all()
    assert e["ref"] < GRAD_REF_TOL and e["src"] < GRAD_SRC_TOL and e["vis"] < GRAD_VIS_TOL, e


def test_grazing_geometry(dev):
    """taps behind the source camera and +-Inf / NaN coordinates: the gradients are finite and match fp64"""
    H, W, C, D, V = 36, 52, 8, 4, 3
    g = torch.Generator().manual_seed(5)
    f = torch.randn(V, H, W, C, generator=g).to(dev)
    homs = R.compose_homs_fp64(R.grazing_projections(H, W)).to(dev)
    dd = R.grazing_depth(D, H, W, seed=1).to(dev)
    vis = (0.05 + torch.rand(V - 1, H, W, generator=g)).to(dev)
    U = torch.randn(D, H, W, 8, generator=g).to(dev)
    ix, iy, _ = R.restated_coords(homs, dd)
    nonfinite = int((~torch.isfinite(ix) | ~torch.isfinite(iy)).sum())
    assert nonfinite > 0
    got = _kernel(f, homs, dd, vis, U)
    assert torch.isfinite(got[0]).all()
    e = _errors("grazing", got, _fp64(f, homs, dd, vis, U))
    assert torch.isfinite(got[1]).all() and torch.isfinite(got[2]).all()
    assert e["ref"] < GRAD_REF_TOL and e["src"] < GRAD_SRC_TOL and e["vis"] < GRAD_VIS_TOL, e


def _fixed_vis(weights):
    """a vis callable returning weights[:, v] on its v-th call, as the op calls it"""
    it = iter(range(weights.shape[1]))
    return lambda e: weights[:, next(it)].unsqueeze(1)


@pytest.mark.parametrize("C,D", SHIPPED)
def test_forward_equals_eval_kernels(dev, C, D):
    """the op's volume is mvsf_warp_corr_aggregate's (two-gather plan) and mvsf_corr_aggregate's after
    mvsf_warp_corr_entropy_store (spill plan) bit for bit, for the same visibility weights"""
    from mvsformerplusplus_b200 import synth
    B, V, H, W = 2, 3, 36, 52
    g = torch.Generator().manual_seed(C + D)
    feats = torch.randn(B, V, C, H, W, generator=g).to(dev)
    pm = synth.make_proj_matrices(V, H, W, batch=B, theta_step=0.12)["stage4"].to(dev)
    from oracle import hotpath as O
    dv = O.init_inverse_range(synth.make_depth_values(192, batch=B), D, H, W).to(dev)
    weights = (0.05 + torch.rand(B, V - 1, H, W, generator=g)).to(dev)
    for budget in (0, 1 << 40):
        vol = cost_volume(feats, pm, dv, _fixed_vis(weights), spill_budget_bytes=budget)
        assert vol.shape == (B, 8, D, H, W)
        for b in range(B):
            fb = feats[b].permute(0, 2, 3, 1).contiguous()
            homs = torch.empty(V - 1, 12, device=dev)
            _lib.call("mvsf_compose_geometry", pm[b], V, homs, torch.empty(9, device=dev))
            want = torch.empty(D, H, W, 8, device=dev)
            if budget == 0:
                _lib.call("mvsf_warp_corr_aggregate", fb, homs, dv[b], weights[b], want, V, C, 8, D, H, W)
            else:
                corr = torch.empty(V - 1, D, H, W, 8, device=dev)
                _lib.call("mvsf_warp_corr_entropy_store", fb, homs, dv[b], torch.empty(V - 1, H, W, device=dev), corr,
                          V, C, 8, D, H, W)
                _lib.call("mvsf_corr_aggregate", corr, weights[b], want, V, 8, D, H, W)
            assert torch.equal(vol[b].permute(1, 2, 3, 0), want), (budget, b)


@pytest.mark.parametrize("name", T.CASES)
def test_reference_training_step(dev, name):
    g, meta, vis = T.fixture(name)
    vis = vis.to(dev)
    feats = g["features"].to(dev).requires_grad_(True)
    vol = cost_volume(feats, g["proj_matrices"].to(dev), g["depth_values"].to(dev), vis)
    vol.backward(g["volume_mean_grad"].to(dev))
    e = dict(volume=T.rel(vol.detach().cpu(), g["volume_mean"]), features_grad=T.rel(feats.grad.cpu(), g["features_grad"]))
    for k, p in vis.named_parameters():
        e[f"grad.{k}"] = T.rel(p.grad.cpu(), g[f"grad.vis.{k}"])
    for k, v in vis.state_dict().items():
        if "running" in k:
            e[k] = T.rel(v.cpu(), g[f"after.vis.{k}"])
    rec(f"train_fixture_{name}", **e)
    assert max(e.values()) < FIXTURE_GPU_TOL, e


# ---- install_training on a reference-shaped stand-in
class _CostReg(nn.Module):
    """a small regulariser with the reference's call signature cost_reg(volume_mean, position3d)"""

    def __init__(self, G):
        super().__init__()
        self.conv = nn.Conv3d(G, 4, 3, padding=1)
        self.prob = nn.Conv3d(4, 1, 1)

    def forward(self, x, position3d=None):
        return self.prob(F.relu(self.conv(x)))


class _Stage(nn.Module):
    """the attributes of models/cost_volume.py:StageNet that its forward reads"""

    def __init__(self, args, ndepth, stage_idx):
        super().__init__()
        self.args, self.ndepth, self.stage_idx = args, ndepth, stage_idx
        self.fusion_type, self.depth_type = "cnn", "ce"
        self.vis = T.make_vis()
        self.cost_reg = _CostReg(8)

    def forward(self, *a, **k):   # the reference's torch forward is not needed here: install_training replaces it
        raise AssertionError("install_training did not rebind forward")


class _StandIn(nn.Module):
    def __init__(self):
        super().__init__()
        self.args = {"base_ch": [8, 8, 8, 8], "ndepths": [32, 16, 8, 4]}
        self.fusions = nn.ModuleList([_Stage(self.args, 8, 2), _Stage(self.args, 4, 3)])


def _restated_stage(stage, features, proj, dv, tmp, training):
    """fp64 restatement of the rebound forward with the same modules"""
    vol = OT.cost_volume(features, proj, dv, stage.vis, G=8)
    pre = stage.cost_reg(vol).squeeze(1)
    prob = F.softmax(pre, dim=1)
    if training:
        depth = torch.gather(dv, 1, prob.argmax(1, keepdim=True)).squeeze(1)
    else:
        depth = torch.sum(F.softmax(pre * tmp, dim=1) * dv, 1)
    return dict(depth=depth, prob_volume=prob, prob_volume_pre=pre, photometric_confidence=prob.max(1)[0])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_install_training_wiring(dev, precision, mode):
    """forward, CE loss and backward through the rebound forward: outputs and every parameter gradient against the fp64
    restatement of the same modules; under bf16 autocast the cost volume still runs in fp32 (the volume cost_reg receives
    equals the fp32 run's bit for bit)"""
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    torch.manual_seed(3)
    model = _StandIn()
    ref = copy.deepcopy(model).double()
    install_training(model.to(dev))
    model.train(mode == "train")
    ref.train(mode == "train")
    B, V, H, W = 2, 3, 24, 32
    g = torch.Generator().manual_seed(17)
    errs = {}
    for i, (C, sc) in enumerate(((16, 2), (8, 1))):
        stage = model.fusions[i]
        D = stage.ndepth
        f = torch.randn(B, V, C, H, W, generator=g)
        pm = synth.make_proj_matrices(V, H * sc, W * sc, batch=B, theta_step=0.12)[f"stage{3 + i}"]
        dv = O.init_inverse_range(synth.make_depth_values(192, batch=B), D, H, W)
        target = torch.randint(0, D, (B, H, W), generator=g)
        volumes = []
        hook = stage.cost_reg.register_forward_pre_hook(lambda m, inp: volumes.append(inp[0].detach().clone()))
        fd = f.to(dev).requires_grad_(True)
        with torch.backends.cudnn.flags(allow_tf32=False):
            state = copy.deepcopy(stage.vis.state_dict())
            with torch.no_grad():   # the fp32 cost volume, for the autocast run's bit-for-bit check
                stage(fd, pm.to(dev), dv.to(dev), tmp=5.0)
            stage.vis.load_state_dict(state)   # undo that call's running-statistics update
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=precision == "bf16"):
                out = stage(fd, pm.to(dev), dv.to(dev), tmp=5.0)
            F.cross_entropy(out["prob_volume_pre"].float(), target.to(dev)).backward()
        hook.remove()
        assert torch.equal(volumes[0], volumes[1])
        f64 = f.double().requires_grad_(True)
        want = _restated_stage(ref.fusions[i], f64, pm.double(), dv.double(), 5.0, mode == "train")
        F.cross_entropy(want["prob_volume_pre"], target).backward()
        assert set(out) == {"depth", "prob_volume", "photometric_confidence", "depth_values", "prob_volume_pre"}
        assert not out["photometric_confidence"].requires_grad
        for k in ("prob_volume", "prob_volume_pre", "photometric_confidence"):
            errs[f"s{i}.{k}"] = T.rel(out[k].detach().float().cpu(), want[k].detach())
        if mode == "eval":
            errs[f"s{i}.depth"] = T.rel(out["depth"].detach().float().cpu(), want["depth"].detach())
        else:   # the argmax gather picks hypotheses; held where fp32 and fp64 agree on the argmax
            same = out["prob_volume"].argmax(1).cpu() == want["prob_volume"].argmax(1)
            assert float(same.float().mean()) > 0.95
            assert torch.equal(out["depth"].cpu()[same], want["depth"].float()[same])
        for k, v in stage.vis.state_dict().items():   # train(): both took one running-statistics step
            if "running" in k:
                errs[f"s{i}.vis.{k}"] = T.rel(v.cpu(), ref.fusions[i].vis.state_dict()[k])
        grads = [(f"s{i}.features", fd.grad, f64.grad)] + [
            (f"s{i}.{k}", p.grad, q.grad) for (k, p), (_, q) in zip(stage.named_parameters(), ref.fusions[i].named_parameters())]
        for k, a, b in grads:
            assert torch.isfinite(a).all(), k
            if precision == "fp32" and not k.endswith("prob.bias"):   # the softmax makes prob.bias's gradient 0
                errs[k + ".grad"] = T.rel(a.cpu(), b)
    rec(f"train_wiring_{precision}_{mode}", **errs)
    assert max(errs.values()) < WIRING_TOL[precision, mode], errs


def test_memory_bound(dev):
    """forward + backward of one training shape (B = 2, V = 5, stage 4 of 512 x 640, channels-last features as FMT gives
    them): the peak above the inputs stays below the outputs (volume, feature gradient, weights and their gradient) plus
    the op's working memory (one sample's upstream gradient copy, the entropy, 1 MB), and that working memory is well
    under the B C D H W warped volume the reference keeps per view (four tensors of that size per view)"""
    from mvsformerplusplus_b200 import synth
    from oracle import hotpath as O
    B, V, C, D, H, W = 2, 5, 8, 4, 512, 640
    g = torch.Generator().manual_seed(23)
    x = torch.randn(B, V, H, W, C, generator=g).to(dev).requires_grad_(True)
    pm = synth.make_proj_matrices(V, H, W, batch=B, theta_step=0.12)["stage4"].to(dev)
    dv = O.init_inverse_range(synth.make_depth_values(192, batch=B), D, H, W).to(dev)
    weights = (0.05 + torch.rand(B, V - 1, H, W, generator=g)).to(dev).requires_grad_(True)
    grad = torch.randn(B, 8, D, H, W, generator=g).to(dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    vol = cost_volume(x.permute(0, 1, 4, 2, 3), pm, dv, _fixed_vis(weights))
    vol.backward(grad)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    f4, HW = 4, H * W
    warped = B * C * D * HW * f4
    outputs = B * 8 * D * HW * f4 + B * V * C * HW * f4 + 2 * B * (V - 1) * HW * f4
    working = 8 * D * HW * f4 + B * (V - 1) * HW * f4 + (1 << 20)
    stand_in = (V - 1) * B * (V - 1) * HW * f4   # the select backward of _fixed_vis materialises each view's gradient
    rec("train_memory", peak_mb=peak / 2**20, bound_mb=(outputs + working + stand_in) / 2**20, working_mb=working / 2**20,
        warped_volume_mb=warped / 2**20)
    assert x.grad is not None and weights.grad is not None
    assert peak <= outputs + working + stand_in, (peak, outputs + working + stand_in)
    assert working < 0.75 * warped


def test_reproducible_and_errors(dev):
    C, D, V, H, W = 16, 8, 4, 36, 52
    case = _case(dev, C, D, H, W, V, seed=99)
    a, b = _kernel(*case), _kernel(*case)
    assert torch.equal(a[1][0], b[1][0]) and torch.equal(a[2], b[2])
    feats = torch.randn(1, V, C, H, W)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        cost_volume(feats, torch.zeros(1, V, 2, 4, 4), torch.ones(1, D, H, W), lambda e: e)
    f, homs, dd, vis, U = case
    vol, gf, gv = a
    for badC, badG in ((12, 4), (16, 4)):
        with pytest.raises(RuntimeError, match="G must be 8 and C in 8/16/32/64"):
            _lib.call("mvsf_warp_corr_aggregate_backward", f, homs, dd, vis, vol, U, gf, gv, V, badC, badG, D, H, W)
