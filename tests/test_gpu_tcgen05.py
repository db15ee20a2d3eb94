"""Tensor-core linear layer (linear_tc.cu, wgmma) against an fp64 GEMM evaluated with torch on the GPU (test-side ground
truth).  The module keeps its original name (the layer first ran on tcgen05) so that its test ids stay stable.
Run in its own process: a mis-programmed tensor-core pipeline traps the CUDA context."""
import ctypes
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def P(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("M,N,K,gelu", [(128, 64, 64, 0), (300, 64, 64, 0), (1000, 256, 64, 1), (513, 64, 256, 0),
                                         (27648, 192, 64, 0), (27648, 64, 256, 1), (130, 16, 128, 0),
                                         (110592, 64, 64, 0), (110592, 256, 64, 1)])   # 6 tiles per persistent CTA
def test_linear_tc_vs_fp64(M, N, K, gelu):
    from mvsformerplusplus_b200 import _lib
    L = _lib.lib()
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 1.5).to(dev)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = (0.1 * torch.randn(N, generator=g)).to(dev)
    C = torch.full((M, N), float("nan"), device=dev)
    ws = torch.empty(((M + N) * 2 * K * 2 + 1024) // 4 + 64, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.mvsf_linear_tc_forward(P(A), P(W), P(b), P(C), P(ws), ctypes.c_size_t(ws.numel() * 4), M, N, K, gelu, st),
               "linear_tc_forward")
    torch.cuda.synchronize()
    want = A.double() @ W.double().t() + b.double()
    if gelu:
        want = torch.nn.functional.gelu(want)
    err = float((C.double() - want).abs().max())
    f32 = A @ W.t() + b
    if gelu:
        f32 = torch.nn.functional.gelu(f32)
    err32 = float((f32.double() - want).abs().max())
    from tests.common import REPORT_DIR
    os.makedirs(REPORT_DIR, exist_ok=True)
    with open(os.path.join(REPORT_DIR, "linear_tc_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(M=M, N=N, K=K, gelu=gelu, tc_vs_f64=err, torch_f32_vs_f64=err32, scale=float(want.abs().max()))) + "\n")
    assert err < 5e-6 * max(1.0, float(want.abs().max()))
