"""The stage-1 attention with the last wave's items split over key ranges (mvsf_attention_split_plan) against an fp64
softmax(QK^T * scale) V, on the inputs and at the bound of test_gpu_parity.test_attention_tensor_core_vs_fp64.  The N
are picked for the device's SM count so that the plan splits each item in two, into a number of parts that does not
divide the key tiles, with a partial last key tile, capped by the workspace, and (as a control) not at all."""
import ctypes
import math

import pytest
import torch

from mvsformerplusplus_b200 import _lib
from tests.common import max_abs, rec

pytestmark = pytest.mark.gpu

MIN_PART_TILES = 16


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def plan(N, sms):
    r, k = ctypes.c_int(), ctypes.c_int()
    _lib.call("mvsf_attention_split_plan", N, sms, ctypes.byref(r), ctypes.byref(k))
    return r.value, k.value


def items(N):
    return 4 * -(-N // 192)


CASES = {   # what the plan must do at N; the first N are the choices on 132 SMs (DTU, T&T, a capped plan, 4 full waves)
    "two_parts": ([27648], lambda N, r, k, sms: k == 2),
    "ragged_parts": ([32640], lambda N, r, k, sms: k > 2 and -(-N // 128) % k != 0),
    "partial_last_tile": ([20000], lambda N, r, k, sms: r > 0 and N % 128 != 0),
    "capped_by_workspace": ([20000], lambda N, r, k, sms: 2 <= k < min(sms // r, -(-N // 128) // MIN_PART_TILES)),
    "no_leftover": ([25344], lambda N, r, k, sms: items(N) % sms == 0),
}


def pick(sms, case):
    prefer, ok = CASES[case]
    for N in prefer + list(range(16000, 40000, 13)):
        if ok(N, *plan(N, sms), sms):
            return N
    pytest.skip(f"no N below 40 000 gives a {case} plan on {sms} SMs")


@pytest.mark.parametrize("case", sorted(CASES))
def test_split_attention_vs_fp64(sms, case):
    dev = torch.device("cuda:0")
    N = pick(sms, case)
    r, k = plan(N, sms)
    assert (r > 0) == (case != "no_leftover")
    g = torch.Generator().manual_seed(N)
    qd = (torch.randn(N, 192, generator=g) * 1.5).to(dev)
    scale = 16 ** -0.5 * math.log(N, 12185)
    ws = torch.empty((N + 128) * 224, device=dev)   # exactly the documented (N + 128) * 896 bytes
    outs = []
    for _ in range(2):
        o = torch.full((N, 64), float("nan"), device=dev)
        _lib.launch_count(reset=True)
        _lib.call("mvsf_attention_forward", qd, o, ws, ws.numel() * 4, N, float(scale))
        assert _lib.launch_count() == (3 if r else 2)   # operand tiling, attention, and the merge of the split items
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "two calls differ"
    q, kk, v = [qd[:, i * 64:(i + 1) * 64].double().view(N, 4, 16).transpose(0, 1) for i in range(3)]
    want = torch.empty(4, N, 16, dtype=torch.float64, device=dev)
    for s0 in range(0, N, 2048):
        want[:, s0:s0 + 2048] = torch.softmax(q[:, s0:s0 + 2048] @ kk.transpose(1, 2) * scale, -1) @ v
    want = want.transpose(0, 1).reshape(N, 64)
    e, sc = max_abs(outs[0], want), float(want.abs().max())
    # the split items are the last r of the grid's (head, 192-row group) items, in head-major order
    groups = -(-N // 192)
    rows = [(it // groups, (it % groups) * 192) for it in range(items(N) - r, items(N))]
    e_split = max((max_abs(outs[0][t0:t0 + 192, 16 * h:16 * h + 16], want[t0:t0 + 192, 16 * h:16 * h + 16])
                   for h, t0 in rows if t0 < N), default=0.0)
    rec(f"attention_split_{case}_N{N}", sms=sms, split_items=r, parts=k, tc_vs_f64=e, split_rows_vs_f64=e_split, scale=sc)
    assert e < 4e-4 * sc
