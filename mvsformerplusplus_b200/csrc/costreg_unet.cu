// R2-R4: 3-D conv U-Net cost regularisers (models/module.py:367-408 CostRegNet, :453-504 CostRegNet3D).
// Activations are NDHWC fp32; BatchNorm (eval) is folded into the packed weights [27][Cin][Cout] + bias[Cout];
// ReLU, the U-Net skip additions (added AFTER the ReLU: `conv4 + self.conv7(x)`, module.py:403-405) and, for
// CostRegNet3D, the final 1x1x1 `prob` conv are fused into the producing kernel's epilogue.
//
// The 3x3x3 layers run on the tensor cores (conv3d_tc.cu: implicit GEMM, fp16 hi|lo activations); this file holds the
// layer schedule of the two U-Nets, the install-time weight re-packing and CostRegNet's final 3x3x3 `prob` conv (8 -> 1).
#include "common.cuh"
#include "conv3d_tc.cuh"

namespace mvsf {

// CostRegNet `prob`: Conv3d(8,1,3,padding=1,bias=False) (module.py:392).  in [D][H][W][8], w [27][8] -> out [D][H][W]
__global__ void prob3_kernel(const float* __restrict__ in, const float* __restrict__ w, float* __restrict__ out, int D,
                             int H, int W) {
  __shared__ float ws[27 * 8];
  for (int i = threadIdx.x; i < 27 * 8; i += blockDim.x) ws[i] = __ldg(w + i);
  __syncthreads();
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, d = blockIdx.z;
  if (x >= W) return;
  float acc = 0.f;
  for (int kd = 0; kd < 3; ++kd) {
    int zd = d + kd - 1;
    if (zd < 0 || zd >= D) continue;
    for (int kh = 0; kh < 3; ++kh) {
      int yh = y + kh - 1;
      if (yh < 0 || yh >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        int xw = x + kw - 1;
        if (xw < 0 || xw >= W) continue;
        const float* p = in + (((size_t)zd * H + yh) * W + xw) * 8;
        float4 a = ldg4(p), b = ldg4(p + 4);
        const float* wp = ws + ((kd * 3 + kh) * 3 + kw) * 8;
        acc = fmaf(a.x, wp[0], acc); acc = fmaf(a.y, wp[1], acc); acc = fmaf(a.z, wp[2], acc); acc = fmaf(a.w, wp[3], acc);
        acc = fmaf(b.x, wp[4], acc); acc = fmaf(b.y, wp[5], acc); acc = fmaf(b.z, wp[6], acc); acc = fmaf(b.w, wp[7], acc);
      }
    }
  }
  out[((size_t)d * H + y) * W + x] = acc;
}

// ---------------------------------------------------------------------------------------------------- host
// ------------------------------------------------------------------------------------ tensor-core path (conv3d_tc.cu)
constexpr int kLayerCh[9][2] = {{8, 16}, {16, 16}, {16, 32}, {32, 32}, {32, 64}, {64, 64}, {64, 32}, {32, 16}, {16, 8}};
static const int kLayerMode[9] = {CONV_S2, CONV_S1, CONV_S2, CONV_S1, CONV_S2, CONV_S1, DECONV_S2, DECONV_S2, DECONV_S2};

// Two fp32 parts (packing.pack_costreg_unet), each counted from 0.  Conv part (the input of mvsf_costreg_unet_pack_tc):
// per layer w [27][Cin][Cout].  Small part, the wts argument: per layer bias[Cout], then the prob conv: [27][8]
// (kind 0) or w[8], b[1] (kind 1), padded to a multiple of 4.
constexpr size_t unet_floats(bool conv) {
  size_t n = 0;
  for (int l = 0; l < 9; ++l) n += conv ? (size_t)27 * kLayerCh[l][0] * kLayerCh[l][1] : kLayerCh[l][1];
  return n;
}
constexpr size_t NCONV = unet_floats(true), NSMALL[2] = {unet_floats(false) + 27 * 8, unet_floats(false) + 8 + 1 + 3};
static_assert(NCONV == 290304 && NSMALL[0] == 496 && NSMALL[1] == 292,
              "packing.COSTREG_UNET_CONV_WTS / COSTREG_UNET_SMALL_WTS");

static size_t tc_total_halves() {
  size_t n = 0;
  for (int l = 0; l < 9; ++l) n += conv3d_tc_packed_halves(kLayerMode[l], kLayerCh[l][0], kLayerCh[l][1]);
  return n;
}

static int unet_forward_tc(int kind, const float* vol, const float* wts, const __half* wtc, float* logits, void* ws, int D,
                           int H, int W, cudaStream_t s) {
  const int SD = kind == 0 ? 2 : 1;
  const int D1 = (D - 1) / SD + 1, H1 = H / 2, W1 = W / 2;
  const int D2 = (D1 - 1) / SD + 1, H2 = H1 / 2, W2 = W1 / 2;
  const int D3 = (D2 - 1) / SD + 1, H3 = H2 / 2, W3 = W2 / 2;
  const size_t n0 = (size_t)D * H * W * 8;
  const size_t n1 = (size_t)D1 * H1 * W1 * 16, n2 = (size_t)D2 * H2 * W2 * 32, n3 = (size_t)D3 * H3 * W3 * 64;
  // every activation buffer is [hi (n halves) | lo (n halves)]
  __half* v0 = reinterpret_cast<__half*>(ws);
  __half* t1 = v0 + 2 * n0;   __half* c2 = t1 + 2 * n1;
  __half* t3 = c2 + 2 * n1;   __half* c4 = t3 + 2 * n2;
  __half* t5 = c4 + 2 * n2;   __half* c6 = t5 + 2 * n3;
  float* x11 = reinterpret_cast<float*>(c6 + 2 * n3);   // kind 0 only: [D][H][W][8] fp32
  const float* bias[9];
  const __half* w16[9];
  {
    const float* p = wts;
    const __half* q = wtc;
    for (int l = 0; l < 9; ++l) {
      bias[l] = p; w16[l] = q;
      p += kLayerCh[l][1];
      q += conv3d_tc_packed_halves(kLayerMode[l], kLayerCh[l][0], kLayerCh[l][1]);
    }
  }
  const float* wp = bias[8] + 8;
  int rc;
  if ((rc = launch_split_f16(vol, n0, v0, 2 * n0, 1, n0, s))) return rc;
  auto conv = [&](int l, const __half* in, size_t nin, __half* out, size_t nout, const __half* skip, size_t nskip,
                  int ID, int IH, int IW) {
    ConvTcArgs a{};
    a.in_hi = in; a.in_lo = in + nin;
    a.wtc = w16[l]; a.bias = bias[l];
    a.skip_hi = skip; a.skip_lo = skip ? skip + nskip : nullptr;
    a.out_hi = out; a.out_lo = out + nout;
    a.CIN = kLayerCh[l][0]; a.COUT = kLayerCh[l][1]; a.SD = SD; a.ID = ID; a.IH = IH; a.IW = IW;
    a.KG = conv3d_tc_kg(kLayerMode[l], a.CIN);
    a.col = conv3d_tc_col(kLayerMode[l], SD, a.COUT);
    return launch_conv3d_tc(a, kLayerMode[l], OUT_SPLIT, s);
  };
  if ((rc = conv(0, v0, n0, t1, n1, nullptr, 0, D, H, W))) return rc;
  if ((rc = conv(1, t1, n1, c2, n1, nullptr, 0, D1, H1, W1))) return rc;
  if ((rc = conv(2, c2, n1, t3, n2, nullptr, 0, D1, H1, W1))) return rc;
  if ((rc = conv(3, t3, n2, c4, n2, nullptr, 0, D2, H2, W2))) return rc;
  if ((rc = conv(4, c4, n2, t5, n3, nullptr, 0, D2, H2, W2))) return rc;
  if ((rc = conv(5, t5, n3, c6, n3, nullptr, 0, D3, H3, W3))) return rc;
  // x = conv4 + conv7(x) -> t3 ; x = conv2 + conv9(x) -> t1 ; x = conv0 + conv11(x)
  if ((rc = conv(6, c6, n3, t3, n2, c4, n2, D3, H3, W3))) return rc;
  if ((rc = conv(7, t3, n2, t1, n1, c2, n1, D2, H2, W2))) return rc;
  {
    ConvTcArgs a{};
    a.in_hi = t1; a.in_lo = t1 + n1;
    a.wtc = w16[8]; a.bias = bias[8];
    a.skip32 = vol;
    a.CIN = 16; a.COUT = 8; a.SD = SD; a.ID = D1; a.IH = H1; a.IW = W1; a.KG = conv3d_tc_kg(DECONV_S2, 16);
    if (kind == 1) {
      a.out32 = logits; a.probw = wp;
      if ((rc = launch_conv3d_tc(a, DECONV_S2, OUT_PROB, s))) return rc;
    } else {
      a.out32 = x11;
      if ((rc = launch_conv3d_tc(a, DECONV_S2, OUT_F32, s))) return rc;
      dim3 grid(cdiv(W, 128), H, D);
      prob3_kernel<<<grid, 128, 0, s>>>(x11, wp, logits, D, H, W);
      MVSF_LAUNCH_CHECK("prob3");
    }
  }
  return MVSF_OK;
}

}  // namespace mvsf

using namespace mvsf;

extern "C" {

int mvsf_costreg_unet_workspace_bytes(int kind, int C, int D, int H, int W, size_t* bytes) {
  MVSF_REQUIRE(bytes && (kind == 0 || kind == 1) && C == 8, "costreg_unet: kind in {0,1}, C == 8");
  MVSF_REQUIRE(H % 8 == 0 && W % 8 == 0 && D >= 1 && (kind == 1 || D % 8 == 0),
               "costreg_unet: H, W (and D for CostRegNet) must be multiples of 8");
  const int SD = kind == 0 ? 2 : 1;
  size_t D1 = (D - 1) / SD + 1, D2 = (D1 - 1) / SD + 1, D3 = (D2 - 1) / SD + 1;
  size_t n1 = D1 * (H / 2) * (W / 2) * 16, n2 = D2 * (H / 4) * (W / 4) * 32, n3 = D3 * (H / 8) * (W / 8) * 64;
  // fp16 hi|lo activation buffers (4 bytes per element, like fp32): input split + two per level; kind 0: fp32 x11
  size_t n = (size_t)D * H * W * 8 + 2 * (n1 + n2 + n3) + (kind == 0 ? (size_t)D * H * W * 8 : 0);
  *bytes = n * sizeof(float);
  return MVSF_OK;
}

int mvsf_costreg_unet_tc_bytes(size_t* bytes) {
  MVSF_REQUIRE(bytes, "costreg_unet_tc_bytes: null pointer");
  *bytes = tc_total_halves() * sizeof(__half);
  return MVSF_OK;
}

int mvsf_costreg_unet_pack_tc(int kind, const float* conv, void* wts_tc, size_t wts_tc_bytes, mvsf_stream_t stream) {
  MVSF_REQUIRE(conv && wts_tc && ((uintptr_t)wts_tc & 15) == 0 && (kind == 0 || kind == 1), "costreg_unet_pack_tc: null or unaligned pointer, or bad kind");
  if (wts_tc_bytes < tc_total_halves() * sizeof(__half))
    return fail(MVSF_ERR_WORKSPACE, "costreg_unet_pack_tc: buffer %zu < %zu bytes", wts_tc_bytes, tc_total_halves() * sizeof(__half));
  const float* p = conv;
  __half* q = reinterpret_cast<__half*>(wts_tc);
  for (int l = 0; l < 9; ++l) {
    int rc = conv3d_tc_pack(p, q, kLayerMode[l], kind == 0 ? 2 : 1, kLayerCh[l][0], kLayerCh[l][1], (cudaStream_t)stream);
    if (rc) return rc;
    p += (size_t)27 * kLayerCh[l][0] * kLayerCh[l][1];
    q += conv3d_tc_packed_halves(kLayerMode[l], kLayerCh[l][0], kLayerCh[l][1]);
  }
  return MVSF_OK;
}

int mvsf_costreg_unet_forward(int kind, const float* volume, const float* wts, const void* wts_tc, float* logits,
                              void* workspace, size_t workspace_bytes, int C, int D, int H, int W, mvsf_stream_t stream) {
  MVSF_REQUIRE(volume && wts && logits && workspace, "costreg_unet: null pointer");
  size_t need = 0;
  int rc = mvsf_costreg_unet_workspace_bytes(kind, C, D, H, W, &need);
  if (rc) return rc;
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "costreg_unet: workspace %zu < %zu bytes", workspace_bytes, need);
  MVSF_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)wts & 15) == 0 && ((uintptr_t)volume & 15) == 0,
               "costreg_unet: pointers must be 16-byte aligned");
  MVSF_REQUIRE(wts_tc && ((uintptr_t)wts_tc & 15) == 0, "costreg_unet: wts_tc (mvsf_costreg_unet_pack_tc) is required, 16-byte aligned");
  return unet_forward_tc(kind, volume, wts, reinterpret_cast<const __half*>(wts_tc), logits, workspace, D, H, W,
                         (cudaStream_t)stream);
}
}
