"""The softmax attention kernels on inputs whose fp16 softmax weights are exact (tests/attention_exact_common.py),
against the fp64 weighted mean with those weights, to an fp32-class bar: mvsf_attention_forward (stage-1, 4 heads of 16,
split plan and merge included) and mvsf_vit_attention_forward (12 heads of 64, strided qkv rows, other images' keys as
decoys).  The error is relative to the scale of the terms of each row and head, max over the head's dims of
sum(w |v|) / sum(w), so that the small means of uniform rows are held to the same bar as the rest.  Outputs are NaN-filled and every case is computed twice, bit for
bit."""
import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import _lib
from tests import attention_exact_common as E
from tests import test_gpu_attention_split as SPLIT
from tests.common import rec

pytestmark = pytest.mark.gpu
# measured on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit): worst 1.9e-7 (stage-1), 4.8e-7 (ViT)
BAR = 1.5e-6


@pytest.fixture(scope="module")
def dev():
    from mvsformerplusplus_b200.build import build
    build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stage1(dev, sms, tag, N):
    plan = E.split_plan(N, sms)
    case = E.make_case(E.STAGE1, N, plan=plan, seed=N)
    E.premise(case)
    qd = torch.from_numpy(case.qkv).to(dev)
    ws = torch.empty((N + 128) * 224, device=dev)
    outs = []
    for _ in range(2):
        o = torch.full((N, 64), float("nan"), device=dev)
        _lib.launch_count(reset=True)
        _lib.call("mvsf_attention_forward", qd, o, ws, ws.numel() * 4, N, E.STAGE1_SCALE)
        assert _lib.launch_count() == (3 if plan[0] else 2)
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "two calls differ"
    e = E.error(outs[0].cpu().numpy(), case)
    rec(f"attention_exact_{tag}", N=N, sms=sms, split_items=plan[0], parts=plan[1], rel_terms=e)
    assert e < BAR, e
    return plan


@pytest.mark.parametrize("N", [1, 64, 128, 129, 385, 4000, 27648, 32640])
def test_attention_exact_weights(dev, sms, N):
    """one key; query blocks past the last one (1, 64, 129); a full tile (128); a last tile of one key (129); a K / V
    ring that wraps (385); the DTU and T&T stage-1 token counts, which split on 132 SMs"""
    _stage1(dev, sms, f"N{N}", N)


@pytest.mark.parametrize("case", sorted(SPLIT.CASES))
def test_attention_exact_weights_split_plan(dev, sms, case):
    """the N of test_gpu_attention_split for this device: two parts, ragged parts, a partial last tile, a plan capped by
    the workspace, and no leftover wave"""
    N = SPLIT.pick(sms, case)
    r, k = _stage1(dev, sms, f"split_{case}_N{N}", N)
    assert (r > 0) == (case != "no_leftover") and (k >= 2) == (r > 0)
    assert SPLIT.CASES[case][1](N, r, k, sms)


@pytest.mark.parametrize("N", [2, 13, 127, 128, 129, 1370, 1729, 2041])
@pytest.mark.parametrize("n", [1, 3, 5])
def test_vit_attention_exact_weights(dev, n, N):
    ldq, ldo = 2316, 776
    case = E.make_case(E.VIT, N, n=n, scale=E.VIT_SCALE, ldq=ldq, seed=n * 10000 + N)
    E.premise(case)
    qd = torch.from_numpy(case.qkv).to(dev)
    ws = torch.empty(n * 12 * ((N + 127) // 128) * 100352 // 4 + 64, device=dev)
    outs = []
    for _ in range(2):
        o = torch.full((n * N, ldo), float("nan"), device=dev)
        _lib.call("mvsf_vit_attention_forward", qd, ldq, o, ldo, ws, ws.numel() * 4, n, N)
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][:, :768], outs[1][:, :768]), "two calls differ"
    assert bool(torch.isnan(outs[0][:, 768:]).all()), "wrote past column 768"
    e = E.error(outs[0][:, :768].cpu().numpy(), case)
    rec(f"vit_attention_exact_n{n}_N{N}", rel_terms=e)
    assert e < BAR, e
