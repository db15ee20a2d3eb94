// F1-F4: FMT_with_pathway.forward (models/FMT.py:164-206): cross-view feature transformer on the 1/8-resolution
// features (FMT.forward :81-137, CrossBlock block.py:336-346 pre-norm with pre_norm_query=False, linear attention
// attention.py:261-291, LayerScale, Mlp) followed by the top-down pathway
//   stage_{k+1} = smooth_k( bilinear_up(dim_reduction_k(stage_k)) + lateral_{k+1} )      (FMT.py:154-162,195-197).
// Tokens "(h w) c" of the reference are exactly channels-last pixels, so the stage-1 output is produced directly in
// the [V][H][W][64] layout the warp kernels consume.  All source views are processed as one batch; the K/V
// summaries of the two cross layers depend only on the reference view and are computed once.
#include "conv2d_tc.cuh"
#include "linattn.cuh"
#include "linear_tc.cuh"

namespace mvsf {

// ---- GEMM weights (the gemm part of packing.pack_fmt), fp32 [N][K] rows; wts16 holds their hi / lo splits with the
// same indexing.  Per CrossBlock: qkv_w[192][64] proj_w[64][64] f1_w[256][64] f2_w[64][256]
constexpr int B_QKV = 0, B_PW = 192 * 64, B_F1W = B_PW + 64 * 64, B_F2W = B_F1W + 256 * 64, G_BLK = B_F2W + 64 * 256,
              NG = 4 * G_BLK;
// ---- small fp32 parameters (the small part of packing.pack_fmt, the wts argument).  Per CrossBlock: n1_w[64] n1_b[64]
// proj_b[64] g1[64] n2_w[64] n2_b[64] f1_b[256] f2_b[64] g2[64]
constexpr int B_N1W = 0, B_N1B = 64, B_PB = 128, B_G1 = B_PB + 64, B_N2W = B_G1 + 64, B_N2B = B_N2W + 64,
              B_F1B = B_N2B + 64, B_F2B = B_F1B + 256, B_G2 = B_F2B + 64, B_SIZE = B_G2 + 64;
// after 4 blocks: dr1[32][64] dr2[16][32] dr3[8][16] sm1[9][32][32] sm2[9][16][16] sm3[9][8][8]   ([tap][ci][co])
constexpr int P_DR1 = 4 * B_SIZE, P_DR2 = P_DR1 + 32 * 64, P_DR3 = P_DR2 + 16 * 32, P_SM1 = P_DR3 + 8 * 16,
              P_SM2 = P_SM1 + 9 * 32 * 32, P_SM3 = P_SM2 + 9 * 16 * 16, NS = P_SM3 + 9 * 8 * 8;
static_assert(NG == 196608 && NS == 17856, "packing.FMT_GEMM_WTS / FMT_SMALL_WTS");
// float2 loads of the biases and LayerScales, float4 loads of the dim_reduction weights
static_assert(B_SIZE % 4 == 0 && B_PB % 4 == 0 && B_G1 % 4 == 0 && B_F1B % 4 == 0 && B_F2B % 4 == 0 && B_G2 % 4 == 0 &&
                  P_DR1 % 4 == 0 && P_DR2 % 4 == 0 && P_DR3 % 4 == 0,
              "vector-loaded small parameters start at a multiple of 4 floats");
using FmtAttn = LinAttn<4, 16>;
constexpr int KVSZ = FmtAttn::KVSZ;  // KV[h][m][d] + ksum[h][d]

// f [V][64][L] (NCHW) + pe [L][64] -> tok [V][L][64]
__global__ void tokens_add_pe_kernel(const float* __restrict__ f, const float* __restrict__ pe, float* __restrict__ tok,
                                     int L) {
  __shared__ float tile[32][33];
  const int v = blockIdx.z;
  const float* s = f + (size_t)v * 64 * L;
  float* d = tok + (size_t)v * 64 * L;
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    if (p < L) tile[i][threadIdx.x] = s[(size_t)c * L + p];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < L) d[(size_t)p * 64 + c] = tile[threadIdx.x][i] + __ldg(pe + (size_t)p * 64 + c);
  }
}

struct FmtWs {
  __half *xn2, *att2;          // fp16 hi|lo split activations: [M][128], [M][128]
  float *qkv, *ref0, *kvpart, *kvfin, *kvc;
  const __half *wh, *wl;       // fp16 hi / lo parts of the GEMM weights
};

// one CrossBlock over `M` tokens (nviews views of L tokens each) stored at x (in place); bw: the block's small
// parameters, boff: the offset of its GEMM weights in ws.wh / ws.wl.
// self attention: kv_src == nullptr ; cross attention: kvc = precomputed K/V summary of the reference view.
// LayerNorms are fused into the epilogue of the GEMM that produces their input: proj emits x (residual stream) and
// split(norm2(x)), FFN2 emits x and split(norm1 of the NEXT block) when `next_bw` is given; `ln1_ready` says the previous
// block already left split(norm1(x)) in ws.xn2.
static int run_block(float* x, int nviews, int L, const float* bw, size_t boff, const float* kvc, const FmtWs& ws,
                     cudaStream_t s, bool ln1_ready = false, const float* next_bw = nullptr) {
  const int M = nviews * L;
  int rc;
  if (!ln1_ready) {
    layernorm_split_kernel<64><<<cdiv(M, 8), 256, 0, s>>>(x, bw + B_N1W, bw + B_N1B, ws.xn2, M, 1e-5f);
    MVSF_LAUNCH_CHECK("fmt_ln1");
  }
  const float* kvsum;
  size_t kv_stride;
  int ldq;
  TcLinArgs a{};
  a.Ah = ws.xn2; a.Al = ws.xn2 + 64; a.lda = 128; a.Bh = ws.wh + boff + B_QKV; a.Bl = ws.wl + boff + B_QKV; a.ldb = 64;
  a.M = M; a.K = 64; a.C = ws.qkv;
  if (!kvc) {
    a.N = 192; a.ldc = 192; a.elu_cols = 128;
    if ((rc = launch_linear_tc(a, LIN_ELU1, s))) return rc;
    if ((rc = launch_kv_summary<4, 16>(ws.qkv, 192, 64, 128, L, nviews, ws.kvpart, ws.kvfin, s))) return rc;
    kvsum = ws.kvfin; kv_stride = KVSZ; ldq = 192;
  } else {
    a.N = 64; a.ldc = 64; a.elu_cols = 64;
    if ((rc = launch_linear_tc(a, LIN_ELU1, s))) return rc;
    kvsum = kvc; kv_stride = 0; ldq = 64;
  }
  if (L % 128 == 0 || nviews == 1) {
    linattn_apply_kernel<4, 16><<<dim3(cdiv(M, 128), 4), 128, 0, s>>>(ws.qkv, ldq, kvsum, kv_stride, ws.att2, L, M);
    MVSF_LAUNCH_CHECK("fmt_linattn_apply");
  } else {
    for (int v = 0; v < nviews; ++v) {  // views do not align with 128-token blocks: one launch per view
      linattn_apply_kernel<4, 16><<<dim3(cdiv(L, 128), 4), 128, 0, s>>>(ws.qkv + (size_t)v * L * ldq, ldq,
                                                                 kvsum + (size_t)v * kv_stride, 0,
                                                                 ws.att2 + (size_t)v * L * 128, L, L);
      MVSF_LAUNCH_CHECK("fmt_linattn_apply");
    }
  }
  // x += gamma1 * proj(...); x += gamma2 * ffn(norm2(x)); xn2 = split(norm1_next(x))
  TokenMlpArgs p{};
  p.A = ws.att2; p.res = x; p.C = x; p.C2 = next_bw ? ws.xn2 : nullptr; p.M = M;
  p.pw_h = ws.wh + boff + B_PW; p.pw_l = ws.wl + boff + B_PW; p.f1w_h = ws.wh + boff + B_F1W; p.f1w_l = ws.wl + boff + B_F1W;
  p.f2w_h = ws.wh + boff + B_F2W; p.f2w_l = ws.wl + boff + B_F2W;
  p.proj_b = bw + B_PB; p.gamma1 = bw + B_G1; p.f1_b = bw + B_F1B; p.f2_b = bw + B_F2B; p.gamma2 = bw + B_G2;
  p.mid_w = bw + B_N2W; p.mid_b = bw + B_N2B; p.mid_eps = 1e-5f;
  if (next_bw) { p.out_w = next_bw + B_N1W; p.out_b = next_bw + B_N1B; p.out_eps = 1e-5f; }
  return launch_token_mlp(p, next_bw ? MLP_PRE_NORM : MLP_PRE_NORM_LAST, s);
}

// K/V summary of a cross layer: key = value = norm1_layer(ref_feature)   (block.py:341-343, FMT.py:121-125)
static int run_cross_kv(const float* ref_tok, int L, const float* bw, size_t boff, float* kvc_out, const FmtWs& ws,
                        cudaStream_t s) {
  int rc;
  layernorm_split_kernel<64><<<cdiv(L, 8), 256, 0, s>>>(ref_tok, bw + B_N1W, bw + B_N1B, ws.xn2, L, 1e-5f);
  MVSF_LAUNCH_CHECK("fmt_ln_key");
  TcLinArgs a{};
  a.Ah = ws.xn2; a.Al = ws.xn2 + 64; a.lda = 128;
  a.Bh = ws.wh + boff + B_QKV + 64 * 64; a.Bl = ws.wl + boff + B_QKV + 64 * 64; a.ldb = 64;
  a.M = L; a.N = 128; a.K = 64; a.C = ws.qkv; a.ldc = 128; a.elu_cols = 64;
  if ((rc = launch_linear_tc(a, LIN_ELU1, s))) return rc;
  return launch_kv_summary<4, 16>(ws.qkv, 128, 0, 64, L, 1, ws.kvpart, kvc_out, s);
}

// 1x1 dim_reduction_k of the pathway (FMT.py:186-189, a bias-free conv = per-pixel CIN -> COUT linear map), channels-last.
// One pixel per thread: the CIN inputs sit in registers, the [COUT][CIN] weights in shared memory (every lane reads the
// same weight: broadcast), HBM traffic = CIN + COUT floats per pixel.  (The generic SIMT GEMM tile this replaces ran at
// 39 / 76 / 185 us for the three levels, ~7x its memory time.)
template <int CIN, int COUT>
__global__ void __launch_bounds__(128)
reduce1x1_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int M) {
  __shared__ __align__(16) float ws[COUT * CIN];
  for (int i = threadIdx.x; i < COUT * CIN / 4; i += 128) reinterpret_cast<float4*>(ws)[i] = ldg4(w + 4 * i);
  __syncthreads();
  const int m = blockIdx.x * 128 + threadIdx.x;
  if (m >= M) return;
  float4 xv[CIN / 4];
#pragma unroll
  for (int k = 0; k < CIN / 4; ++k) xv[k] = ldg4(x + (size_t)m * CIN + 4 * k);
  float* yo = y + (size_t)m * COUT;
#pragma unroll
  for (int n4 = 0; n4 < COUT / 4; ++n4) {
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4* wr = reinterpret_cast<const float4*>(ws + (n4 * 4 + j) * CIN);
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < CIN / 4; ++k) {
        const float4 wv = wr[k];
        acc = fmaf(xv[k].x, wv.x, acc); acc = fmaf(xv[k].y, wv.y, acc);
        acc = fmaf(xv[k].z, wv.z, acc); acc = fmaf(xv[k].w, wv.w, acc);
      }
      o[j] = acc;
    }
    *reinterpret_cast<float4*>(yo + n4 * 4) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// Phase 1 of smooth_k on the conv2d_tc template: pre = lateral + bilinear_up2(red) on the halo of the tile, written as the
// planes of the single parity; red [V][h][w][C] (NHWC), lat [V][C][2h][2w] (NCHW).  The upsampled + added tensor never
// goes to HBM.
template <class L>
struct PathwaySrc {
  const float* red;
  const float* lat;
  int h, w;
  static constexpr uint32_t EXTRA = 0;
  static_assert(L::CI == L::CO && L::KS == 3 && L::S == 1, "pathway smooth conv: C -> C, 3x3, stride 1");
  __device__ void fill(unsigned char* smem, int v, int y0, int x0, int tid) const {
    constexpr int C = L::CI, PR = L::PR, PC = L::PC;
    const int H = 2 * h, W = 2 * w;
    const float* lv = lat + (size_t)v * C * H * W;
    const float* rv = red + (size_t)v * h * w * C;
    for (int i = tid; i < L::NO * PR * PC; i += 256) {
      const int o = i / (PR * PC), pix = i - o * (PR * PC);
      const int r = pix / PC, c = pix - r * PC;
      const int y = y0 - 1 + r, x = x0 - 1 + c;
      float pre[8];
      if (y >= 0 && y < H && x >= 0 && x < W) {
        // ATen area_pixel_compute_source_index(scale=0.5, align_corners=False): src = 0.5*(dst+0.5)-0.5, clamped at 0
        const float sy = fmaxf(0.5f * ((float)y + 0.5f) - 0.5f, 0.0f);
        const int ya = (int)sy, yb = ya + ((ya < h - 1) ? 1 : 0);
        const float ly1 = sy - (float)ya, ly0 = 1.0f - ly1;
        const float sx = fmaxf(0.5f * ((float)x + 0.5f) - 0.5f, 0.0f);
        const int xa = (int)sx, xb = xa + ((xa < w - 1) ? 1 : 0);
        const float lx1 = sx - (float)xa, lx0 = 1.0f - lx1;
        const float* p00 = rv + ((size_t)ya * w + xa) * C + o * 8;
        const float* p01 = rv + ((size_t)ya * w + xb) * C + o * 8;
        const float* p10 = rv + ((size_t)yb * w + xa) * C + o * 8;
        const float* p11 = rv + ((size_t)yb * w + xb) * C + o * 8;
#pragma unroll
        for (int q4 = 0; q4 < 2; ++q4) {
          const float4 v00 = ldg4(p00 + q4 * 4), v01 = ldg4(p01 + q4 * 4), v10 = ldg4(p10 + q4 * 4), v11 = ldg4(p11 + q4 * 4);
          const float a00[4] = {v00.x, v00.y, v00.z, v00.w}, a01[4] = {v01.x, v01.y, v01.z, v01.w};
          const float a10[4] = {v10.x, v10.y, v10.z, v10.w}, a11[4] = {v11.x, v11.y, v11.z, v11.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float up = ly0 * (lx0 * a00[e] + lx1 * a01[e]) + ly1 * (lx0 * a10[e] + lx1 * a11[e]);
            pre[q4 * 4 + e] = up + __ldg(lv + ((size_t)(o * 8 + q4 * 4 + e) * H + y) * W + x);
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) pre[e] = 0.f;
      }
      __half* p = reinterpret_cast<__half*>(smem + L::plane(0, o, 0) + (uint32_t)pix * 16u);
      split_store8(p, p + L::PLANE / 2, pre);   // hi plane of octet o, then its lo plane (+ PLANE bytes)
    }
  }
};

template <int C>
struct NhwcOut {   // smooth_k has no bias and no activation: [V][H][W][C]
  float* out;
  static constexpr bool BIAS = false;
  __device__ void store(int v, int H, int W, int y, int x, int ch, float a, float b) const {
    *reinterpret_cast<float2*>(out + (((size_t)v * H + y) * W + x) * C + ch) = make_float2(a, b);
  }
};

// smooth-conv weight tiles (sm_tc) come from c2d::pack_conv2d_tc
template <int CIN, int COUT>
static int run_pathway_level(const float* prev, const float* lat, const float* dr_w, const void* sm_tc, float* red,
                             float* out, int V, int h, int w, cudaStream_t s) {
  const int M = V * h * w;
  reduce1x1_kernel<CIN, COUT><<<cdiv(M, 128), 128, 0, s>>>(prev, dr_w, red, M);
  MVSF_LAUNCH_CHECK("fmt_reduce1x1");
  using L = c2d::Conv<COUT, COUT, 3, 1, 16, COUT>;
  return c2d::launch_conv<L>(PathwaySrc<L>{red, lat, h, w}, NhwcOut<COUT>{out}, sm_tc, nullptr, V, 2 * h, 2 * w, s);
}

// packed smooth_1..3 weight tiles at the end of the workspace
constexpr size_t SM_TC1 = c2d::conv2d_tc_bytes(32, 32, 3), SM_TC2 = c2d::conv2d_tc_bytes(16, 16, 3),
                 SM_TC = SM_TC1 + SM_TC2 + c2d::conv2d_tc_bytes(8, 8, 3);

}  // namespace mvsf

using namespace mvsf;

extern "C" {

int mvsf_fmt_workspace_bytes(int V, int H1, int W1, size_t* bytes) {
  MVSF_REQUIRE(bytes && V >= 2 && H1 > 0 && W1 > 0, "fmt: bad arguments");
  size_t L = (size_t)H1 * W1, VL = (size_t)V * L;
  size_t nblk = (L + KV_CHUNK - 1) / KV_CHUNK;
  size_t n = 320 * VL + 64 * L + (size_t)V * nblk * KVSZ + (size_t)(V + 2) * KVSZ + 64;
  *bytes = n * sizeof(float) + SM_TC;
  return MVSF_OK;
}

int mvsf_fmt_forward(const float* f1, const float* f2, const float* f3, const float* f4, const float* pe,
                     const float* wts, const void* wts16, size_t n_wts, float* o1, float* o2, float* o3, float* o4,
                     void* workspace, size_t workspace_bytes, int V, int H1, int W1, mvsf_stream_t stream) {
  MVSF_REQUIRE(f1 && f2 && f3 && f4 && pe && wts && wts16 && o1 && o2 && o3 && o4 && workspace, "fmt: null pointer");
  MVSF_REQUIRE(n_wts == (size_t)NG && ((uintptr_t)wts16 & 15) == 0, "fmt: bad fp16 weight blob");
  size_t need = 0;
  int rc = mvsf_fmt_workspace_bytes(V, H1, W1, &need);
  if (rc) return rc;
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "fmt: workspace %zu < %zu bytes", workspace_bytes, need);
  MVSF_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)wts & 15) == 0, "fmt: pointers must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int L = H1 * W1;
  const size_t VL = (size_t)V * L;
  float* base = (float*)workspace;
  FmtWs ws;
  ws.xn2 = reinterpret_cast<__half*>(base);                  // [V*L][128] halves (= 64 floats / token)
  ws.qkv = base + 64 * VL;                                   // [V*L][192]
  ws.att2 = reinterpret_cast<__half*>(ws.qkv + 192 * VL);    // [V*L][128] halves  (320 VL floats in total; the pathway reuses the first 128 VL)
  ws.wh = reinterpret_cast<const __half*>(wts16);
  ws.wl = ws.wh + n_wts;
  ws.ref0 = base + 320 * VL;          // [L][64]
  const size_t nblk = (L + KV_CHUNK - 1) / KV_CHUNK;
  ws.kvpart = ws.ref0 + 64 * (size_t)L;
  ws.kvfin = ws.kvpart + (size_t)V * nblk * KVSZ;
  ws.kvc = ws.kvfin + (size_t)V * KVSZ;   // [2][KVSZ]

  MVSF_REQUIRE(V <= 65535, "fmt: too many views");
  tokens_add_pe_kernel<<<dim3(cdiv(L, 32), 2, V), dim3(32, 8), 0, s>>>(f1, pe, o1, L);
  MVSF_LAUNCH_CHECK("fmt_tokens_add_pe");

  const float* b0 = wts; const float* b1 = wts + B_SIZE; const float* b2 = wts + 2 * B_SIZE; const float* b3 = wts + 3 * B_SIZE;
  // reference view: the two self layers (FMT.py:96-107); keep the output of the first one for cross layer 1
  if ((rc = run_block(o1, 1, L, b0, 0, nullptr, ws, s, false, b2))) return rc;
  MVSF_CUDA_OK(cudaMemcpyAsync(ws.ref0, o1, (size_t)L * 64 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if ((rc = run_block(o1, 1, L, b2, 2 * (size_t)G_BLK, nullptr, ws, s, true, nullptr))) return rc;
  if ((rc = run_cross_kv(ws.ref0, L, b1, (size_t)G_BLK, ws.kvc, ws, s))) return rc;
  if ((rc = run_cross_kv(o1, L, b3, 3 * (size_t)G_BLK, ws.kvc + KVSZ, ws, s))) return rc;
  // source views as one batch: self, cross(ref_list[0]), self, cross(ref_list[1])   (FMT.py:119-135)
  float* xs = o1 + (size_t)L * 64;
  if ((rc = run_block(xs, V - 1, L, b0, 0, nullptr, ws, s, false, b1))) return rc;
  if ((rc = run_block(xs, V - 1, L, b1, (size_t)G_BLK, ws.kvc, ws, s, true, b2))) return rc;
  if ((rc = run_block(xs, V - 1, L, b2, 2 * (size_t)G_BLK, nullptr, ws, s, true, b3))) return rc;
  if ((rc = run_block(xs, V - 1, L, b3, 3 * (size_t)G_BLK, ws.kvc + KVSZ, ws, s, true, nullptr))) return rc;

  // top-down pathway (FMT.py:195-197), all views batched
  unsigned char* sm_tc = static_cast<unsigned char*>(workspace) + need - SM_TC;
  if ((rc = c2d::pack_conv2d_tc(wts + P_SM1, sm_tc, 32, 32, 3, 32, s))) return rc;
  if ((rc = c2d::pack_conv2d_tc(wts + P_SM2, sm_tc + SM_TC1, 16, 16, 3, 16, s))) return rc;
  if ((rc = c2d::pack_conv2d_tc(wts + P_SM3, sm_tc + SM_TC1 + SM_TC2, 8, 8, 3, 8, s))) return rc;
  float* red = base;                  // <= 128 VL floats
  if ((rc = run_pathway_level<64, 32>(o1, f2, wts + P_DR1, sm_tc, red, o2, V, H1, W1, s))) return rc;
  if ((rc = run_pathway_level<32, 16>(o2, f3, wts + P_DR2, sm_tc + SM_TC1, red, o3, V, 2 * H1, 2 * W1, s))) return rc;
  if ((rc = run_pathway_level<16, 8>(o3, f4, wts + P_DR3, sm_tc + SM_TC1 + SM_TC2, red, o4, V, 4 * H1, 4 * W1, s))) return rc;
  return MVSF_OK;
}
}
