"""The fp16 hi + lo split that every tensor-core path feeds its fp32 operands through (common.cuh: split_f16x2, run on
whole blobs by split_hi_lo_f16_kernel), through mvsf_split_weights_f16: hi and lo must equal torch's independent
conversions x.half() and (x - x.half().float()).half() bit for bit.  The inputs are adversarial: signed zeros, fp16
subnormals, round-to-nearest-even ties, values at and just past the fp16 maximum 65504 (hi overflows to inf there, and
lo is then -inf), fp32 extremes (largest, smallest normal, smallest subnormal) and random normals over many scales."""
import numpy as np
import pytest
import torch

from mvsformerplusplus_b200 import _lib

pytestmark = pytest.mark.gpu


def _adversarial():
    f32 = np.finfo(np.float32)
    v = [0.0, -0.0, 65504.0, -65504.0, 65519.0, -65519.0, 65520.0, -65520.0, 65536.0, 65505.5, float(f32.max),
         -float(f32.max), float(f32.tiny), -float(f32.tiny), float(f32.smallest_subnormal),
         -float(f32.smallest_subnormal), 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 2.0 ** -14, 2.0 ** -24, 2.0 ** -25,
         3 * 2.0 ** -25, -(2.0 ** -24), 2.0 ** -14 - 2.0 ** -24, 1.0 / 3.0, -1e-8, 1e-30]
    sub = np.arange(1, 1024, dtype=np.float32) * np.float32(2.0 ** -24)   # every fp16 subnormal, and the midpoints
    return np.concatenate([np.array(v, dtype=np.float32), sub, sub + np.float32(2.0 ** -25), -sub])


def _inputs(n):
    g = np.random.default_rng(n)
    x = (g.standard_normal(n) * 10.0 ** g.uniform(-9, 5, n)).astype(np.float32)
    adv = _adversarial()
    k = min(n, adv.size)
    x[:k] = adv[:k]
    return torch.from_numpy(x)


@pytest.mark.parametrize("n", [8, 8 * 12345, 4_000_008])
def test_split_weights_f16_matches_torch_bit_for_bit(n):
    x = _inputs(n)
    xd = x.cuda()
    out = torch.full((2 * n,), float("nan"), device="cuda", dtype=torch.float16)
    _lib.call("mvsf_split_weights_f16", xd, out, n)
    torch.cuda.synchronize()
    got = out.cpu().view(torch.int16)
    hi = x.half()
    lo = (x - hi.float()).half()
    bad_hi = torch.nonzero(got[:n] != hi.view(torch.int16)).flatten()
    bad_lo = torch.nonzero(got[n:] != lo.view(torch.int16)).flatten()
    assert bad_hi.numel() == 0, f"hi differs at {bad_hi[:8].tolist()} (x = {x[bad_hi[:8]].tolist()})"
    assert bad_lo.numel() == 0, f"lo differs at {bad_lo[:8].tolist()} (x = {x[bad_lo[:8]].tolist()})"
