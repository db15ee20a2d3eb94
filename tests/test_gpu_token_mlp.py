"""The fused token MLP (linear_tc.cu: token_mlp_kernel, through mvsf_token_mlp_forward) that FMT blocks and the
transformer-regulariser layers run: bit for bit against the three single GEMMs it replaces (proj, FFN1, FFN2 through
mvsf_linear_tc_epilogue), and against an fp64 reference at the bar of test_linear_tc_epilogue_vs_fp64.  Every form:
pre-norm block, last pre-norm block, post-norm layer.  M covers one row, partial and whole 128-row tiles, a persistent
CTA running a second tile (SMs * 128 + 1) and the FMT source-view batch at DTU (110 592 rows).  The MLP runs in place
(C aliases res), as both callers run it.  Run in its own process: a mis-programmed tensor-core pipeline traps the CUDA
context."""
import pytest
import torch

from mvsformerplusplus_b200 import _lib
from tests.test_gpu_tcgen05 import EPI_TOL, GELU, RES, RES_LN

pytestmark = pytest.mark.gpu

PRE, PRE_LAST, POST = 0, 1, 2
SPARE = 3   # rows past M in every output buffer, NaN-filled: the kernel must not write them


def _inputs(M, form, dev):
    g = torch.Generator().manual_seed(11 * M + form)
    r = lambda *s, scale=1.0, shift=0.0: (shift + scale * torch.randn(*s, generator=g)).to(dev)
    return dict(A=r(M, 64, scale=1.5), res=r(M, 64), proj_w=r(64, 64, scale=64 ** -0.5), proj_b=r(64, scale=0.1),
                gamma1=r(64, scale=0.5), mid_w=r(64, scale=0.2, shift=1.0), mid_b=r(64, scale=0.1),
                f1_w=r(256, 64, scale=64 ** -0.5), f1_b=r(256, scale=0.1), f2_w=r(64, 256, scale=256 ** -0.5),
                f2_b=r(64, scale=0.1), gamma2=r(64, scale=0.5), out_w=r(64, scale=0.2, shift=1.0), out_b=r(64, scale=0.1))


def _nan(rows, cols, dtype, dev):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device=dev)


def _fused(form, M, t, dev):
    C = _nan(M + SPARE, 64, torch.float32, dev)
    C[:M] = t["res"]
    C2 = _nan(M + SPARE, 128, torch.float16, dev) if form != PRE_LAST else None
    ws = torch.empty((M * 128 + 73728) // 2 + 64, device=dev)
    _lib.call("mvsf_token_mlp_forward", form, t["A"], C, t["proj_w"], t["proj_b"], t["gamma1"], t["mid_w"], t["mid_b"], 1e-5,
              t["f1_w"], t["f1_b"], t["f2_w"], t["f2_b"], t["gamma2"], t["out_w"], t["out_b"], 1e-6, C, C2, ws,
              ws.numel() * 4, M)
    return C, C2


def _three_gemms(form, M, t, dev):
    """proj, FFN1 and FFN2 as the single GEMMs with fused epilogues: fp32 intermediates re-split inside each call round
    exactly as the fp16 hi|lo outputs the callers used to chain"""
    ws = torch.empty((M + 256) * 2 * 256 * 2 // 4 + 64, device=dev)

    def gemm(epi, A, K, W, bias, res, gamma, ln_w, ln_b, eps, C, Cpre, C2, N):
        _lib.call("mvsf_linear_tc_epilogue", epi, A, K, W, bias, res, 64, gamma, ln_w, ln_b, float(eps), 0, C, N, Cpre, 64,
                  C2, 128, ws, ws.numel() * 4, M, N, K)

    x = t["res"].clone()
    mid = torch.empty(M, 64, device=dev)   # LN_mid(...): the FFN input (and, post-norm, FFN2's residual)
    hid = torch.empty(M, 256, device=dev)
    C = torch.empty(M, 64, device=dev)
    C2 = torch.empty(M, 128, dtype=torch.float16, device=dev) if form != PRE_LAST else None
    gemm(RES_LN, t["A"], 64, t["proj_w"], t["proj_b"], x, t["gamma1"], t["mid_w"], t["mid_b"], 1e-5, mid,
         x if form != POST else None, None, 64)
    gemm(GELU, mid, 64, t["f1_w"], t["f1_b"], None, None, None, None, 1e-5, hid, None, None, 256)
    r = mid if form == POST else x
    if form == PRE:
        gemm(RES_LN, hid, 256, t["f2_w"], t["f2_b"], r, t["gamma2"], t["out_w"], t["out_b"], 1e-6, None, C, C2, 64)
    elif form == PRE_LAST:
        gemm(RES, hid, 256, t["f2_w"], t["f2_b"], r, t["gamma2"], None, None, 1e-6, C, None, None, 64)
    else:
        gemm(RES_LN, hid, 256, t["f2_w"], t["f2_b"], r, t["gamma2"], t["out_w"], t["out_b"], 1e-6, C, None, C2, 64)
    return C, C2


def _fp64(form, t):
    d = {k: v.double() for k, v in t.items()}
    ln = lambda z, w, b, eps: torch.nn.functional.layer_norm(z, (64,), w, b, eps)
    ffn = lambda z: torch.nn.functional.gelu(z @ d["f1_w"].t() + d["f1_b"]) @ d["f2_w"].t() + d["f2_b"]
    x = d["res"] + d["gamma1"] * (d["A"] @ d["proj_w"].t() + d["proj_b"])
    if form == POST:
        y = ln(x, d["mid_w"], d["mid_b"], 1e-5)
        out = ln(y + d["gamma2"] * ffn(y), d["out_w"], d["out_b"], 1e-6)
        return out, out
    x = x + d["gamma2"] * ffn(ln(x, d["mid_w"], d["mid_b"], 1e-5))
    return x, (ln(x, d["out_w"], d["out_b"], 1e-6) if form == PRE else None)


def _m(M):
    return torch.cuda.get_device_properties(0).multi_processor_count * 128 + 1 if M == "wave" else M


FORMS = {"pre": PRE, "pre_last": PRE_LAST, "post": POST}
MS = [1, 127, 128, 129, "wave", 110592]


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("form", list(FORMS))
def test_token_mlp_bitwise_vs_three_gemms(form, M):
    dev = torch.device("cuda:0")
    form, M = FORMS[form], _m(M)
    t = _inputs(M, form, dev)
    C, C2 = _fused(form, M, t, dev)
    C3, C23 = _three_gemms(form, M, t, dev)
    torch.cuda.synchronize()
    assert bool(torch.isnan(C[M:]).all()), "C: write past row M"
    assert torch.equal(C[:M].view(torch.int32), C3.view(torch.int32)), \
        f"C differs from the three GEMMs at {int((C[:M] != C3).any(1).sum())} rows, max {float((C[:M] - C3).abs().max()):.3e}"
    if C2 is not None:
        assert bool(torch.isnan(C2[M:].float()).all()), "C2: write past row M"
        assert torch.equal(C2[:M].view(torch.int16), C23.view(torch.int16)), "C2 differs from the three GEMMs"


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("form", list(FORMS))
def test_token_mlp_vs_fp64(form, M):
    from tests.common import rec
    dev = torch.device("cuda:0")
    name, form, M = f"token_mlp_{form}_M{M}", FORMS[form], _m(M)
    t = _inputs(M, form, dev)
    C, C2 = _fused(form, M, t, dev)
    torch.cuda.synchronize()
    want_c, want_c2 = _fp64(form, t)
    errs = {"C": (float((C[:M].double() - want_c).abs().max()), max(1.0, float(want_c.abs().max())))}
    if C2 is not None:
        hi, lo = C2[:M, :64].double(), C2[:M, 64:].double()
        errs["C2"] = (float((hi + lo - want_c2).abs().max()), max(1.0, float(want_c2.abs().max())))
    rec(name, M=M, **{k: e for k, (e, _) in errs.items()}, **{k + "_scale": s for k, (_, s) in errs.items()})
    for k, (e, s) in errs.items():
        assert e < EPI_TOL * s, f"{k}: max error {e:.3e} vs fp64, limit {EPI_TOL * s:.3e}"
