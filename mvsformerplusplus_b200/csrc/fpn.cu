// FPN feature pyramid: models/module.py:208-239 FPNEncoder and :242-270 FPNDecoder (eval, feat_chs [8,16,32,64], BN folded).
// Every 3x3 / 5x5 convolution is one launch of the implicit-GEMM template conv2d_tc_kernel (conv2d_tc.cuh) with a source
// and a destination of this file.
// Sources: an NHWC fp32 tensor (encoder layers), conv00 computed in SIMT from the [N][3][H][W] image (fused conv00 + conv01:
// conv00's output never reaches HBM), and the decoder's intra_k = up2(intra_{k-1}) + inner_k(lateral_k) (align_corners=True
// bilinear + 1x1 conv with bias; the tile interior of intra_1 / intra_2 is also stored for the next level, the
// full-resolution intra_3 is not).  Epilogue: folded bias (+ BN), then the destination's LeakyReLU(0.1) -> NHWC fp32
// (encoder) or Swish -> NCHW fp32 (decoder).  out0 (1x1 at 1/8 resolution) is a small SIMT kernel.
#include "conv2d_tc.cuh"
#include "linear_tc.cuh"

namespace mvsf {
namespace fpn {
using namespace c2d;

// ---- sources (phase 1)
// input NHWC fp32 [N][IH][IW][CI]
template <class L>
struct NhwcSrc {
  const float* in;
  int IH, IW;
  static constexpr uint32_t EXTRA = 0;
  __device__ void fill(unsigned char* smem, int n, int y0, int x0, int tid) const {
    constexpr int NPIX = L::PR * L::PC;
#pragma unroll 2   // two pixel octets' loads in flight per thread
    for (int i = tid; i < L::NP * NPIX * L::NO; i += 256) {
      const int o = i % L::NO, rest = i / L::NO;
      const int pix = rest % NPIX, par = rest / NPIX;
      const int r = pix / L::PC, c = pix - r * L::PC;
      const int iy = L::S * (y0 + r) - L::PAD + par / L::S, ix = L::S * (x0 + c) - L::PAD + par % L::S;
      float v[8];
      if (iy >= 0 && iy < IH && ix >= 0 && ix < IW) {
        const float* p = in + (((size_t)n * IH + iy) * IW + ix) * L::CI + o * 8;
        const float4 a = ldg4(p), b = ldg4(p + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.f;
      }
      __half* h = reinterpret_cast<__half*>(smem + L::plane(par, o, 0) + (uint32_t)pix * 16u);
      split_store8(h, h + L::PLANE / 2, v);   // lo plane = + PLANE bytes
    }
  }
};

// conv00 (3 -> 8, 7x7, pad 3, folded BN, LeakyReLU) in SIMT from the image x [N][3][H][W]; w = [49 taps][3 ci][8 co], b[8]
template <class L>
struct Conv00Src {
  const float* x;
  const float* w;
  int H, W;
  static constexpr int IR = L::PR + 6, IC = L::PC + 6, NW = 49 * 3 * 8 + 8;
  static constexpr uint32_t EXTRA = (3 * IR * IC + NW) * 4;
  static_assert(L::CI == 8 && L::S == 1, "conv00 feeds an 8-channel stride-1 layer");
  __device__ void fill(unsigned char* smem, int n, int y0, int x0, int tid) const {
    float* in_s = reinterpret_cast<float*>(smem + L::SMEM);
    float* ws = in_s + 3 * IR * IC;
    for (int i = tid; i < NW; i += 256) ws[i] = __ldg(w + i);
    const float* xn = x + (size_t)n * 3 * H * W;
    for (int i = tid; i < 3 * IR * IC; i += 256) {
      const int ch = i / (IR * IC), rem = i - ch * (IR * IC);
      const int r = rem / IC, c = rem - r * IC;
      const int gy = y0 - L::PAD - 3 + r, gx = x0 - L::PAD - 3 + c;
      in_s[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(xn + ((size_t)ch * H + gy) * W + gx) : 0.f;
    }
    __syncthreads();
    for (int pix = tid; pix < L::PR * L::PC; pix += 256) {
      const int r = pix / L::PC, c = pix - r * L::PC;
      const int gy = y0 - L::PAD + r, gx = x0 - L::PAD + c;
      float acc[8];
#pragma unroll
      for (int oc = 0; oc < 8; ++oc) acc[oc] = ws[NW - 8 + oc];
      for (int ch = 0; ch < 3; ++ch)
#pragma unroll
        for (int ky = 0; ky < 7; ++ky)
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) {
            const float v = in_s[(ch * IR + r + ky) * IC + c + kx];
            const float* wp = ws + ((ky * 7 + kx) * 3 + ch) * 8;
#pragma unroll
            for (int oc = 0; oc < 8; ++oc) acc[oc] = fmaf(v, wp[oc], acc[oc]);
          }
      const bool inside = gy >= 0 && gy < H && gx >= 0 && gx < W;
#pragma unroll
      for (int oc = 0; oc < 8; ++oc) acc[oc] = inside ? (acc[oc] > 0.f ? acc[oc] : 0.1f * acc[oc]) : 0.f;
      __half* h = reinterpret_cast<__half*>(smem + L::plane(0, 0, 0) + (uint32_t)pix * 16u);
      split_store8(h, h + L::PLANE / 2, acc);
    }
  }
};

// intra = F.interpolate(prev, scale_factor=2, bilinear, align_corners=True) + inner(lat):  prev [N][h][w][64],
// lat [N][2h][2w][CL], w = inner [CL ci][64 co] then b[64]; intra_out (or NULL) receives the tile interior, NHWC fp32
template <class L, int CL>
struct IntraSrc {
  const float* prev;
  const float* lat;
  const float* w;
  float* intra_out;
  int h, wd;
  static constexpr uint32_t EXTRA = (CL * 64 + 64) * 4;
  static_assert(L::CI == 64 && L::S == 1 && L::KS == 3, "decoder level: 3x3 conv of the 64-channel intra feature");
  __device__ void fill(unsigned char* smem, int n, int y0, int x0, int tid) const {
    float* ws = reinterpret_cast<float*>(smem + L::SMEM);
    for (int i = tid; i < CL * 64 + 64; i += 256) ws[i] = __ldg(w + i);
    __syncthreads();
    const int H = 2 * h, W = 2 * wd;
    // ATen area_pixel_compute_scale / source_index, align_corners=True: src = dst * (in - 1) / (out - 1)
    const float scy = (float)(h - 1) / (float)(H - 1), scx = (float)(wd - 1) / (float)(W - 1);
    const float* pv = prev + (size_t)n * h * wd * 64;
    for (int i = tid; i < L::PR * L::PC * 8; i += 256) {
      const int o = i & 7, pix = i >> 3;
      const int r = pix / L::PC, c = pix - r * L::PC;
      const int y = y0 - 1 + r, x = x0 - 1 + c;
      float v[8];
      if (y >= 0 && y < H && x >= 0 && x < W) {
        const float sy = scy * (float)y, sx = scx * (float)x;
        const int ya = (int)sy, yb = ya + (ya < h - 1 ? 1 : 0), xa = (int)sx, xb = xa + (xa < wd - 1 ? 1 : 0);
        const float ly1 = sy - (float)ya, ly0 = 1.f - ly1, lx1 = sx - (float)xa, lx0 = 1.f - lx1;
        const float* p00 = pv + ((size_t)ya * wd + xa) * 64 + o * 8;
        const float* p01 = pv + ((size_t)ya * wd + xb) * 64 + o * 8;
        const float* p10 = pv + ((size_t)yb * wd + xa) * 64 + o * 8;
        const float* p11 = pv + ((size_t)yb * wd + xb) * 64 + o * 8;
#pragma unroll
        for (int q4 = 0; q4 < 2; ++q4) {
          const float4 v00 = ldg4(p00 + q4 * 4), v01 = ldg4(p01 + q4 * 4), v10 = ldg4(p10 + q4 * 4), v11 = ldg4(p11 + q4 * 4);
          const float a00[4] = {v00.x, v00.y, v00.z, v00.w}, a01[4] = {v01.x, v01.y, v01.z, v01.w};
          const float a10[4] = {v10.x, v10.y, v10.z, v10.w}, a11[4] = {v11.x, v11.y, v11.z, v11.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float up = ly0 * (lx0 * a00[e] + lx1 * a01[e]) + ly1 * (lx0 * a10[e] + lx1 * a11[e]);
            v[q4 * 4 + e] = up + ws[CL * 64 + o * 8 + q4 * 4 + e];
          }
        }
        const float* lp = lat + (((size_t)n * H + y) * W + x) * CL;
#pragma unroll 4
        for (int ci = 0; ci < CL; ++ci) {
          const float l = __ldg(lp + ci);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = fmaf(l, ws[ci * 64 + o * 8 + e], v[e]);
        }
        if (intra_out != nullptr && r >= 1 && r <= L::TR && c >= 1 && c <= 32) {
          float* op = intra_out + (((size_t)n * H + y) * W + x) * 64 + o * 8;
          *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(op + 4) = make_float4(v[4], v[5], v[6], v[7]);
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.f;
      }
      __half* hp = reinterpret_cast<__half*>(smem + L::plane(0, o, 0) + (uint32_t)pix * 16u);
      split_store8(hp, hp + L::PLANE / 2, v);
    }
  }
};

// ---- destinations (phase 3): two consecutive channels ch, ch + 1 of one output pixel, folded bias b[CO] already added
template <int CO>
struct NhwcLeaky {   // encoder: LeakyReLU(0.1), [N][OH][OW][CO]
  float* out;
  static constexpr bool BIAS = true;
  __device__ void store(int n, int OH, int OW, int y, int x, int ch, float a, float b) const {
    a = a > 0.f ? a : 0.1f * a;
    b = b > 0.f ? b : 0.1f * b;
    *reinterpret_cast<float2*>(out + (((size_t)n * OH + y) * OW + x) * CO + ch) = make_float2(a, b);
  }
};
template <int CO>
struct NhwcLeakyAddVit {   // last encoder layer of the model: LeakyReLU(0.1), then + vit[n % V] (conv31 + vit_feat)
  float* out;
  const float* vit;   // [V][OH][OW][CO]
  int V;
  static constexpr bool BIAS = true;
  __device__ void store(int n, int OH, int OW, int y, int x, int ch, float a, float b) const {
    a = a > 0.f ? a : __fmul_rn(0.1f, a);   // rounded on its own, as the reference's two separate ops round it
    b = b > 0.f ? b : __fmul_rn(0.1f, b);
    const float2 v = *reinterpret_cast<const float2*>(vit + (((size_t)(n % V) * OH + y) * OW + x) * CO + ch);
    *reinterpret_cast<float2*>(out + (((size_t)n * OH + y) * OW + x) * CO + ch) = make_float2(__fadd_rn(a, v.x),
                                                                                              __fadd_rn(b, v.y));
  }
};
__device__ __forceinline__ float swish(float v) { return v / (1.0f + expf(-v)); }
template <int CO>
struct NchwSwish {   // decoder: Swish, [N][CO][OH][OW]
  float* out;
  static constexpr bool BIAS = true;
  __device__ void store(int n, int OH, int OW, int y, int x, int ch, float a, float b) const {
    float* p = out + (((size_t)n * CO + ch) * OH + y) * OW + x;
    p[0] = swish(a);
    p[(size_t)OH * OW] = swish(b);
  }
};

// out0 = Swish(BN(conv1x1(conv31) + b)):  c31 [N][h][w][64] -> out [N][64][h][w];  w = [64 ci][64 co] then b[64]
__global__ void __launch_bounds__(128) fpn_out0_kernel(const float* __restrict__ c31, const float* __restrict__ w,
                                                        float* __restrict__ out, int HW, int npix) {
  __shared__ float ws[64 * 64 + 64];
  for (int i = threadIdx.x; i < 64 * 64 + 64; i += 128) ws[i] = __ldg(w + i);
  __syncthreads();
  const int p = blockIdx.x * 128 + threadIdx.x;
  if (p >= npix) return;
  const int n = p / HW, px = p - n * HW;
  float xv[64];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float4 t = ldg4(c31 + (size_t)p * 64 + 4 * i);
    xv[4 * i] = t.x; xv[4 * i + 1] = t.y; xv[4 * i + 2] = t.z; xv[4 * i + 3] = t.w;
  }
#pragma unroll 4
  for (int co = 0; co < 64; ++co) {
    float s = ws[64 * 64 + co];
#pragma unroll
    for (int ci = 0; ci < 64; ++ci) s = fmaf(xv[ci], ws[ci * 64 + co], s);
    out[((size_t)n * 64 + co) * HW + px] = swish(s);
  }
}

// ---- layer table.  Each module's weights come in two fp32 parts (packing.pack_fpn_encoder / pack_fpn_decoder), each
// counted from 0: the conv part holds the weights w [KS*KS][CI][CO] of the tensor-core convolutions (the input of
// mvsf_fpn_pack_tc); the small part, the wts argument, holds what the kernels read in fp32.
struct LayerDesc { int ci, co, ks, ns; };
// encoder conv part: conv01 ... conv31 w; small part: conv00 w [49][3][8] b[8] (SIMT), then b[CO] of conv01 ... conv31
constexpr LayerDesc kEnc[11] = {{3, 8, 7, 0},    {8, 8, 5, 8},    {8, 16, 5, 16},  {16, 16, 3, 16},
                                {16, 16, 3, 16}, {16, 32, 5, 32}, {32, 32, 3, 32}, {32, 32, 3, 32},
                                {32, 64, 3, 32}, {64, 64, 3, 32}, {64, 64, 3, 32}};
// decoder conv part: out_k [9][64][C_k], k = 1..3; small part: out0 [64][64] b[64], then per level k = 1..3:
// inner_k [CL][64] b[64], out_k b[C_k]
constexpr LayerDesc kDec[3] = {{64, 32, 3, 32}, {64, 16, 3, 16}, {64, 8, 3, 8}};
constexpr int kLat[3] = {32, 16, 8};

template <int I> using EncL = Conv<kEnc[I].ci, kEnc[I].co, kEnc[I].ks, (I == 2 || I == 5 || I == 8) ? 2 : 1,
                                   (I >= 8) ? 8 : 16, kEnc[I].ns>;
template <int K> using DecL = Conv<64, kDec[K].co, 3, 1, K == 0 ? 8 : 16, kDec[K].ns>;

constexpr size_t conv_floats(const LayerDesc& d) { return (size_t)d.ks * d.ks * d.ci * d.co; }
constexpr size_t layer_tc_bytes(const LayerDesc& d) { return conv2d_tc_bytes(d.ci, d.co, d.ks); }
constexpr size_t enc_conv_off(int i) { size_t o = 0; for (int j = 1; j < i; ++j) o += conv_floats(kEnc[j]); return o; }
constexpr size_t enc_bias_off(int i) {   // small-part offset of b of encoder layer i
  size_t o = conv_floats(kEnc[0]);
  for (int j = 0; j < i; ++j) o += kEnc[j].co;
  return o;
}
static size_t enc_tc_off(int i) { size_t o = 0; for (int j = 1; j < i; ++j) o += layer_tc_bytes(kEnc[j]); return o; }
constexpr size_t dec_conv_off(int k) { size_t o = 0; for (int j = 0; j < k; ++j) o += conv_floats(kDec[j]); return o; }
constexpr size_t dec_inner_off(int k) {   // small-part offset of inner_{k+1}
  size_t o = 64 * 64 + 64;
  for (int j = 0; j < k; ++j) o += (size_t)kLat[j] * 64 + 64 + kDec[j].co;
  return o;
}
constexpr size_t dec_bias_off(int k) { return dec_inner_off(k) + (size_t)kLat[k] * 64 + 64; }   // b of out_{k+1}
static_assert(enc_conv_off(11) == 132800 && enc_bias_off(11) == 1528 && dec_conv_off(3) == 32256 &&
                  dec_inner_off(3) == 7992,
              "packing.FPN_ENCODER_CONV_WTS / FPN_ENCODER_SMALL_WTS / FPN_DECODER_CONV_WTS / FPN_DECODER_SMALL_WTS");
static size_t dec_tc_off(int k) { size_t o = 0; for (int j = 0; j < k; ++j) o += layer_tc_bytes(kDec[j]); return o; }
static size_t enc_tc_total() { return enc_tc_off(11); }
static size_t dec_tc_total() { return dec_tc_off(3); }

// encoder layer I (>= 2) reading an NHWC map of the previous layer's size
template <int I>
static int enc_layer(const float* in, float* out, const float* wts, const unsigned char* wtc, int N, int IH, int IW,
                     cudaStream_t s) {
  using L = EncL<I>;
  const int OH = IH / L::S, OW = IW / L::S;
  return launch_conv<L>(NhwcSrc<L>{in, IH, IW}, NhwcLeaky<L::CO>{out}, wtc + enc_tc_off(I), wts + enc_bias_off(I), N,
                        OH, OW, s);
}

template <int K>
static int dec_level(const float* prev, const float* lat, const float* wts, const unsigned char* wtc, float* intra_out,
                     float* out, int N, int h, int w, cudaStream_t s) {
  using L = DecL<K>;
  return launch_conv<L>(IntraSrc<L, kLat[K]>{prev, lat, wts + dec_inner_off(K), intra_out, h, w},
                        NchwSwish<L::CO>{out}, wtc + dec_tc_off(K), wts + dec_bias_off(K), N, 2 * h, 2 * w, s);
}

// conv31: the last encoder layer, optionally with the model's + vit_feat in its epilogue
static int enc_last(const float* in, float* out, const float* vit, int V, const float* wts, const unsigned char* wtc,
                    int N, int IH, int IW, cudaStream_t s) {
  if (vit == nullptr) return enc_layer<10>(in, out, wts, wtc, N, IH, IW, s);
  using L = EncL<10>;
  return launch_conv<L>(NhwcSrc<L>{in, IH, IW}, NhwcLeakyAddVit<L::CO>{out, vit, V}, wtc + enc_tc_off(10),
                        wts + enc_bias_off(10), N, IH, IW, s);
}

static bool shape_ok(int N, int H, int W) {
  return N > 0 && N <= 65535 && H >= 8 && W >= 8 && H % 8 == 0 && W % 8 == 0 && (long long)H * W < (1ll << 28);
}

}  // namespace fpn
}  // namespace mvsf

using namespace mvsf;
using namespace mvsf::fpn;

extern "C" int mvsf_fpn_tc_bytes(int part, size_t* bytes) {
  MVSF_REQUIRE(bytes && (part == 0 || part == 1), "fpn_tc_bytes: part must be 0 (encoder) or 1 (decoder)");
  *bytes = part == 0 ? enc_tc_total() : dec_tc_total();
  return MVSF_OK;
}

extern "C" int mvsf_fpn_pack_tc(int part, const float* conv, void* wts_tc, size_t wts_tc_bytes, mvsf_stream_t stream) {
  MVSF_REQUIRE(conv && wts_tc && (part == 0 || part == 1), "fpn_pack_tc: bad arguments");
  MVSF_REQUIRE(wts_tc_bytes >= (part == 0 ? enc_tc_total() : dec_tc_total()), "fpn_pack_tc: wts_tc too small");
  unsigned char* out = static_cast<unsigned char*>(wts_tc);
  const int n = part == 0 ? 10 : 3;
  for (int j = 0; j < n; ++j) {
    const LayerDesc& d = part == 0 ? kEnc[j + 1] : kDec[j];
    const float* w = conv + (part == 0 ? enc_conv_off(j + 1) : dec_conv_off(j));
    unsigned char* o = out + (part == 0 ? enc_tc_off(j + 1) : dec_tc_off(j));
    const int rc = pack_conv2d_tc(w, o, d.ci, d.co, d.ks, d.ns, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return MVSF_OK;
}

extern "C" int mvsf_fpn_encoder_workspace_bytes(int N, int H, int W, size_t* bytes) {
  MVSF_REQUIRE(bytes, "fpn_encoder_workspace_bytes: null pointer");
  MVSF_REQUIRE(shape_ok(N, H, W), "fpn encoder: H and W must be positive multiples of 8 (got N=%d H=%d W=%d)", N, H, W);
  *bytes = 2 * (size_t)N * H * W * 16;   // two ping-pong maps of the largest intermediate, [N][H/2][W/2][16] fp32
  return MVSF_OK;
}

static int encoder_forward(const float* x, const float* vit, int V, const float* wts, const void* wts_tc, float* c01,
                           float* c11, float* c21, float* c31, void* workspace, size_t workspace_bytes, int N, int H,
                           int W, mvsf_stream_t stream) {
  size_t need = 0;
  if (mvsf_fpn_encoder_workspace_bytes(N, H, W, &need) != MVSF_OK) return MVSF_ERR_INVALID;
  MVSF_REQUIRE(x && wts && wts_tc && c01 && c11 && c21 && c31 && workspace, "fpn_encoder_forward: null pointer");
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "fpn_encoder_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned char* wtc = static_cast<const unsigned char*>(wts_tc);
  float* t0 = static_cast<float*>(workspace);
  float* t1 = t0 + (size_t)N * H * W * 4;
  using L1 = EncL<1>;
  int rc = launch_conv<L1>(Conv00Src<L1>{x, wts, H, W}, NhwcLeaky<8>{c01}, wtc + enc_tc_off(1), wts + enc_bias_off(1),
                           N, H, W, s);
  if (rc) return rc;
  if ((rc = enc_layer<2>(c01, t0, wts, wtc, N, H, W, s))) return rc;
  if ((rc = enc_layer<3>(t0, t1, wts, wtc, N, H / 2, W / 2, s))) return rc;
  if ((rc = enc_layer<4>(t1, c11, wts, wtc, N, H / 2, W / 2, s))) return rc;
  if ((rc = enc_layer<5>(c11, t0, wts, wtc, N, H / 2, W / 2, s))) return rc;
  if ((rc = enc_layer<6>(t0, t1, wts, wtc, N, H / 4, W / 4, s))) return rc;
  if ((rc = enc_layer<7>(t1, c21, wts, wtc, N, H / 4, W / 4, s))) return rc;
  if ((rc = enc_layer<8>(c21, t0, wts, wtc, N, H / 4, W / 4, s))) return rc;
  if ((rc = enc_layer<9>(t0, t1, wts, wtc, N, H / 8, W / 8, s))) return rc;
  return enc_last(t1, c31, vit, V, wts, wtc, N, H / 8, W / 8, s);
}

extern "C" int mvsf_fpn_encoder_forward(const float* x, const float* wts, const void* wts_tc, float* c01, float* c11,
                                        float* c21, float* c31, void* workspace, size_t workspace_bytes, int N, int H,
                                        int W, mvsf_stream_t stream) {
  return encoder_forward(x, nullptr, 1, wts, wts_tc, c01, c11, c21, c31, workspace, workspace_bytes, N, H, W, stream);
}

extern "C" int mvsf_fpn_encoder_vit_forward(const float* x, const float* vit_feat, int V, const float* wts,
                                            const void* wts_tc, float* c01, float* c11, float* c21, float* c31,
                                            void* workspace, size_t workspace_bytes, int N, int H, int W,
                                            mvsf_stream_t stream) {
  MVSF_REQUIRE(vit_feat && ((uintptr_t)vit_feat & 7) == 0 && V >= 1, "fpn_encoder_vit_forward: need an 8-byte aligned "
               "vit_feat and V >= 1 (got V=%d)", V);
  return encoder_forward(x, vit_feat, V, wts, wts_tc, c01, c11, c21, c31, workspace, workspace_bytes, N, H, W, stream);
}

extern "C" int mvsf_fpn_decoder_workspace_bytes(int N, int H, int W, size_t* bytes) {
  MVSF_REQUIRE(bytes, "fpn_decoder_workspace_bytes: null pointer");
  MVSF_REQUIRE(shape_ok(N, H, W), "fpn decoder: H and W must be positive multiples of 8 (got N=%d H=%d W=%d)", N, H, W);
  *bytes = (size_t)N * ((size_t)(H / 4) * (W / 4) + (size_t)(H / 2) * (W / 2)) * 64 * 4;   // intra_1, intra_2
  return MVSF_OK;
}

extern "C" int mvsf_fpn_decoder_forward(const float* c01, const float* c11, const float* c21, const float* c31,
                                        const float* wts, const void* wts_tc, float* o0, float* o1, float* o2, float* o3,
                                        void* workspace, size_t workspace_bytes, int N, int H, int W,
                                        mvsf_stream_t stream) {
  size_t need = 0;
  if (mvsf_fpn_decoder_workspace_bytes(N, H, W, &need) != MVSF_OK) return MVSF_ERR_INVALID;
  MVSF_REQUIRE(c01 && c11 && c21 && c31 && wts && wts_tc && o0 && o1 && o2 && o3 && workspace,
               "fpn_decoder_forward: null pointer");
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "fpn_decoder_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned char* wtc = static_cast<const unsigned char*>(wts_tc);
  float* intra1 = static_cast<float*>(workspace);
  float* intra2 = intra1 + (size_t)N * (H / 4) * (W / 4) * 64;
  const int npix = N * (H / 8) * (W / 8);
  fpn_out0_kernel<<<cdiv(npix, 128), 128, 0, s>>>(c31, wts, o0, (H / 8) * (W / 8), npix);
  MVSF_LAUNCH_CHECK("fpn_out0");
  int rc;
  if ((rc = dec_level<0>(c31, c21, wts, wtc, intra1, o1, N, H / 8, W / 8, s))) return rc;
  if ((rc = dec_level<1>(intra1, c11, wts, wtc, intra2, o2, N, H / 4, W / 4, s))) return rc;
  return dec_level<2>(intra2, c01, wts, wtc, nullptr, o3, N, H / 2, W / 2, s);
}
