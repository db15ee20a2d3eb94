"""Tensor-core linear layer (linear_tc.cu, wgmma) against an fp64 GEMM evaluated with torch on the GPU (test-side ground
truth).  The module keeps its original name (the layer first ran on tcgen05) so that its test ids stay stable.
Run in its own process: a mis-programmed tensor-core pipeline traps the CUDA context."""
import json
import os

import pytest
import torch

from mvsformerplusplus_b200 import _lib

pytestmark = pytest.mark.gpu


BIAS, GELU, ELU1, RES, RES_LN, LN = range(6)
EPI_NAMES = ["bias", "gelu", "elu1", "res", "res_ln", "ln"]
# The cases use the (N, epilogue) pairs the library builds (kTcPairs in linear_tc.cu).  Bias-only products whose weights
# fit no N that BIAS is built for (K = 256) run as ELU1 with elu_cols = 0: the same arithmetic.
LINEAR_CASES = [(128, 192, 64, BIAS), (300, 192, 64, BIAS), (1000, 256, 64, GELU), (513, 64, 256, ELU1),
                (27648, 192, 64, BIAS), (27648, 256, 64, GELU), (130, 192, 128, BIAS), (110592, 192, 64, BIAS),
                (110592, 256, 64, GELU)]   # 110 592 rows: 6 tiles per persistent CTA


@pytest.mark.parametrize("M,N,K,epi", LINEAR_CASES, ids=[f"{EPI_NAMES[e]}-M{M}-N{N}-K{K}" for M, N, K, e in LINEAR_CASES])
def test_linear_tc_vs_fp64(M, N, K, epi):
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 1.5).to(dev)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = (0.1 * torch.randn(N, generator=g)).to(dev)
    C = torch.full((M, N), float("nan"), device=dev)
    ws = torch.empty(((M + N) * 2 * K * 2 + 1024) // 4 + 64, device=dev)
    _lib.call("mvsf_linear_tc_epilogue", epi, A, K, W, b, None, 0, None, None, None, 1e-5, 0, C, N, None, 0, None, 0, ws,
              ws.numel() * 4, M, N, K)
    torch.cuda.synchronize()
    gelu = epi == GELU
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
        f.write(json.dumps(dict(M=M, N=N, K=K, epi=epi, tc_vs_f64=err, torch_f32_vs_f64=err32, scale=float(want.abs().max()))) + "\n")
    assert err < 5e-6 * max(1.0, float(want.abs().max()))


# ---- every fused epilogue through mvsf_linear_tc_epilogue, the way FMT (fmt.cu) and the transformer regulariser
#      (costreg_tr.cu) call them: strided outputs in NaN-filled buffers with spare rows and columns, the fp16 hi|lo
#      output C2 that feeds the next GEMM, and M chosen so that tiles are partial, a MMA warpgroup has no valid row or
#      only one, and a persistent CTA runs a second tile ("wave": M = SMs * 128 + 1).
# |out - fp64| <= EPI_TOL * max(1, max|fp64|), for C, Cpre and hi + lo of C2.  Measured on an H100: at most 1.5e-6; a
# dropped lo operand product or a lost lo half of C2 costs >= 1.8e-4
EPI_TOL = 5e-6
EPI_CASES = [
    # epi, N, K, M, bias, outputs, elu_cols / ln_eps
    (BIAS, 192, 64, 1, True, "C", None),
    (ELU1, 64, 256, "wave", False, "C+C2", 0),   # elu_cols = 0: the BIAS arithmetic
    (BIAS, 192, 128, 65, False, "C+C2", None),
    (BIAS, 192, 64, 110592, True, "C", None),
    (BIAS, 192, 128, 127, True, "C2", None),
    (BIAS, 192, 64, "wave", False, "C", None),
    (BIAS, 192, 128, 1000, False, "C+C2", None),
    (BIAS, 192, 64, 129, True, "C", None),
    (BIAS, 256, 64, 65, False, "C", None),
    (BIAS, 256, 64, "wave", True, "C+C2", None),
    (ELU1, 64, 64, 65, False, "C+C2", 9),
    (ELU1, 64, 256, 1, False, "C", 64),
    (ELU1, 64, 128, 1000, True, "C+C2", 37),
    (ELU1, 128, 64, 110592, False, "C", 64),   # FMT's cross-attention K/V GEMM (run_cross_kv)
    (ELU1, 128, 64, "wave", False, "C", 64),
    (ELU1, 192, 64, 129, False, "C", 128),     # FMT's self-attention QKV GEMM
    (ELU1, 192, 128, "wave", True, "C+C2", 128),
    (ELU1, 192, 64, 127, True, "C", 37),
    (RES, 64, 64, 1000, True, "C", None),
    (RES, 64, 256, "wave", True, "C+C2", None),
    (RES, 64, 128, 65, False, "C", None),
    (RES_LN, 64, 64, 110592, True, "Cpre=res+C2", 1e-5),   # FMT: x += gamma * proj(..), xn2 = split(norm2(x))
    (RES_LN, 64, 256, "wave", True, "Cpre=res+C2", 1e-5),
    (RES_LN, 64, 128, 1, True, "Cpre=res+C2", 1e-6),
    (RES_LN, 64, 64, 1000, True, "C+C2", 1e-5),            # transformer: post-norm block output and its split
    (RES_LN, 64, 64, 127, False, "C+C2", 1e-6),
    (LN, 64, 64, 129, True, "C", 1e-6),
    (LN, 64, 256, "wave", True, "C+Cpre+C2", 1e-5),
    (LN, 64, 128, 65, False, "C2", 1e-6),
]


def _epi_id(c):
    epi, N, K, M, bias, outs, extra = c
    name = EPI_NAMES[epi]
    return f"{name}-N{N}-K{K}-M{M}-{'b' if bias else 'nob'}-{outs}" + ("" if extra is None else f"-{extra}")


def _nan_buffer(rows, cols, dtype, dev):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device=dev)


def _check_spare_nan(buf, M, N, what):
    """the valid block [:M, :N] is finite, every other element of the buffer still holds its NaN"""
    assert bool(torch.isfinite(buf[:M, :N].float()).all()), f"{what}: non-finite value in the output"
    spare = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    spare[:M, :N] = False
    assert bool(torch.isnan(buf[spare].float()).all()), f"{what}: write outside the output"


@pytest.mark.parametrize("epi,N,K,M,bias,outs,extra", EPI_CASES, ids=[_epi_id(c) for c in EPI_CASES])
def test_linear_tc_epilogue_vs_fp64(epi, N, K, M, bias, outs, extra):
    from tests.common import rec
    dev = torch.device("cuda:0")
    name = "linear_tc_epi_" + _epi_id((epi, N, K, M, bias, outs, extra))
    outs = set(outs.split("+"))
    if M == "wave":
        M = torch.cuda.get_device_properties(0).multi_processor_count * 128 + 1
    g = torch.Generator().manual_seed(7 * M + 3 * N + K + epi)
    lda, ldc, ldc2, ldres, spare = K + 8, N + 8, 2 * N + 16, 72, 3
    A = _nan_buffer(M, lda, torch.float32, dev)   # NaN in the spare columns: the split must not read them
    A[:, :K] = (torch.randn(M, K, generator=g) * 1.5).to(dev)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = (0.1 * torch.randn(N, generator=g)).to(dev) if bias else None
    gamma = (0.5 * torch.randn(N, generator=g)).to(dev)
    ln_w = (1.0 + 0.2 * torch.randn(N, generator=g)).to(dev)
    ln_b = (0.1 * torch.randn(N, generator=g)).to(dev)
    res = None
    if epi in (RES, RES_LN):
        res = _nan_buffer(M + spare, ldres, torch.float32, dev)
        res[:M, :N] = torch.randn(M, N, generator=g).to(dev)
    res64 = res[:M, :N].double() if res is not None else None   # before the call: Cpre may overwrite res

    C = _nan_buffer(M + spare, ldc, torch.float32, dev) if "C" in outs else None
    C2 = _nan_buffer(M + spare, ldc2, torch.float16, dev) if "C2" in outs else None
    if "Cpre=res" in outs:
        Cpre, ldcpre = res, ldres
    elif "Cpre" in outs:
        Cpre, ldcpre = _nan_buffer(M + spare, 72, torch.float32, dev), 72
    else:
        Cpre, ldcpre = None, 0
    ws = torch.empty(((M + N) * 2 * K * 2 + 1024) // 4 + 64, device=dev)
    eps = extra if epi in (RES_LN, LN) else 1e-5
    elu_cols = extra if epi == ELU1 else 0
    _lib.call("mvsf_linear_tc_epilogue", epi, A, lda, W, b, res, ldres, gamma, ln_w, ln_b, float(eps), elu_cols, C, ldc,
              Cpre, ldcpre, C2, ldc2, ws, ws.numel() * 4, M, N, K)
    torch.cuda.synchronize()

    t = A[:, :K].double() @ W.double().t()
    if b is not None:
        t = t + b.double()
    if epi == ELU1:
        t = torch.cat([torch.nn.functional.elu(t[:, :elu_cols]) + 1.0, t[:, elu_cols:]], 1)
    if epi in (RES, RES_LN):
        t = res64 + gamma.double() * t
    pre = t
    if epi in (RES_LN, LN):
        t = torch.nn.functional.layer_norm(t, (N,), ln_w.double(), ln_b.double(), eps)
    scale = max(1.0, float(t.abs().max()))
    errs = {}   # output -> (max abs error vs fp64, max(1, max|fp64|))
    if C is not None:
        errs["C"] = (float((C[:M, :N].double() - t).abs().max()), scale)
    if C2 is not None:
        hi, lo = C2[:M, :N], C2[:M, N:2 * N]
        errs["C2"] = (float((hi.double() + lo.double() - t).abs().max()), scale)
    if Cpre is not None:
        errs["Cpre"] = (float((Cpre[:M, :N].double() - pre).abs().max()), max(1.0, float(pre.abs().max())))
    rec(name, M=M, **{k: e for k, (e, _) in errs.items()}, **{k + "_scale": s for k, (_, s) in errs.items()})
    for k, buf in (("C", C), ("C2", C2), ("Cpre", Cpre)):
        if buf is not None:
            _check_spare_nan(buf, M, 2 * N if k == "C2" else N, k)
    if C is not None and C2 is not None:   # the split of C itself, bit for bit
        c = C[:M, :N]
        want_hi = c.half()
        want_lo = (c - want_hi.float()).half()
        assert torch.equal(hi.view(torch.int16), want_hi.view(torch.int16)), "C2 hi != fp16(C)"
        assert torch.equal(lo.view(torch.int16), want_lo.view(torch.int16)), "C2 lo != fp16(C - hi)"
    for k, (e, s) in errs.items():
        assert e < EPI_TOL * s, f"{k}: max error {e:.3e} vs fp64, limit {EPI_TOL * s:.3e}"
