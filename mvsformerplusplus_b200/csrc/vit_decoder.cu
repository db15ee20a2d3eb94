// V1: CrossVITDecoder.forward (models/module.py:273-364), shipped config: d_model 768, 12 heads of 64, linear attention
// (attention.py:261-291), ffn "ffn" (768 -> 3072 exact-erf GELU -> 768), LayerScale, pre-norm CrossBlocks
// (block.py:336-346) with pre_norm_query = True (the K / V of a cross block are the raw reference tokens), combine
// norms LN_eps1e-6(prev * s + x_i), then the conv head proj (3x3, 768 -> 256) / upsampler0 / upsampler1 (ConvTranspose2d
// k4 s2 p1) with BN folded and SiLU.
//   * every linear and every convolution is the streamed-weight wgmma GEMM of linear_tc.cu: token rows for the linears,
//     implicit-GEMM rows for the 3x3 conv (9 taps x 768 channels) and for each parity class of the transposed convs in
//     gather form (2 x 2 taps, the epilogue stores to pixel (2y + py, 2x + px));
//   * per sample, the reference view runs self0, combine, self1, combine; the K / V summaries of cross layer i depend only
//     on r_i and are computed once; the V - 1 source views then run as one batch of tokens;
//   * tokens stay fp32 in the residual stream; GEMM inputs are fp16 hi|lo splits written by the producing kernel.
#include "linattn.cuh"
#include "linear_tc.cuh"

namespace mvsf {
namespace vitdec {

constexpr int D = 768, HID = 3072, NBLK = 5;   // blocks: self0, self1, cross0, cross1, cross2
using Attn = LinAttn<12, 64>;
constexpr int KVSZ = Attn::KVSZ;

// ---- GEMM weights (the gemm part of packing.pack_vit_decoder), fp32 [N][K] rows; the tc blob holds their hi / lo
// splits with the same indexing
constexpr size_t G_QKV = 0, G_PROJ = (size_t)3 * D * D, G_FC1 = (size_t)4 * D * D, G_FC2 = G_FC1 + (size_t)HID * D,
                 G_BLK = G_FC2 + (size_t)D * HID;
constexpr size_t G_CONV = NBLK * G_BLK;                       // [256][9 taps * 768]     tap = ky * 3 + kx
constexpr size_t G_UP0 = G_CONV + (size_t)256 * 9 * D;        // [4 classes][128][4 taps * 256]
constexpr size_t G_UP1 = G_UP0 + (size_t)4 * 128 * 4 * 256;   // [4 classes][64][4 taps * 128]
constexpr size_t NG = G_UP1 + (size_t)4 * 64 * 4 * 128;
// ---- small fp32 parameters (the small part of packing.pack_vit_decoder, the wts argument): per block norm1 w, b,
// proj bias, ls1, norm2 w, b, fc1 bias [3072], fc2 bias, ls2
constexpr size_t S_N1W = 0, S_N1B = D, S_PB = 2 * D, S_LS1 = 3 * D, S_N2W = 4 * D, S_N2B = 5 * D, S_F1B = 6 * D,
                 S_F2B = S_F1B + HID, S_LS2 = S_F2B + D, S_BLK = S_LS2 + D;
constexpr size_t P_NORM = NBLK * S_BLK,   // norm_layers[0] w, b, norm_layers[1] w, b
                 P_PREV = P_NORM + 4 * D, // prev_values[0], [1], 6 floats of padding
                 P_CB = P_PREV + 8,       // folded conv biases: proj [256], up0 [128], up1 [64]
                 N_WTS = P_CB + 448;
static_assert(NG == 37814272 && N_WTS == 49608, "packing.VIT_DECODER_GEMM_WTS / VIT_DECODER_SMALL_WTS");

// x <- LN_a(prev * x + xi)  (module.py:337-339,350-352: combine + norm_layers, eps 1e-6);  y2 <- split(LN_b(x)) when ln_b
// weights are given (norm1 of the next block, eps 1e-5)
__global__ void __launch_bounds__(256)
combine_kernel(float* __restrict__ x, const float* __restrict__ xi, const float* __restrict__ prev,
               const float* __restrict__ aw, const float* __restrict__ ab, const float* __restrict__ bw,
               const float* __restrict__ bb, __half* __restrict__ y2, int M) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float p = __ldg(prev);
  RowVec<D> r, a;
  r.load(x + (size_t)row * D, lane);
  a.load(xi + (size_t)row * D, lane);
#pragma unroll
  for (int e = 0; e < RowVec<D>::E; ++e) r.v[e] = __fadd_rn(__fmul_rn(p, r.v[e]), a.v[e]);
  r.layernorm(aw, ab, 1e-6f, lane);
  r.store(x + (size_t)row * D, lane);
  if (bw) {
    r.layernorm(bw, bb, 1e-5f, lane);
    r.store_split(y2 + (size_t)row * 2 * D, lane);
  }
}

struct Ws {
  __half *xn2, *att2, *hid2;   // [Mx][2D], [Mx][2D], [Mx][2 HID] halves
  float *qkv, *kvp, *kvf, *kvc; // qkv >= max(L * 3D, Ms * D) floats; kvc [3][KVSZ]
  const float* w;               // small fp32 parameters
  const __half *wh, *wl;        // tc blob: hi / lo parts of the GEMM weights
};

static TcsArgs gemm(const Ws& ws, const __half* A, int lda, int K, size_t woff, int N, int M) {
  return tcs_rows(A, lda, K, ws.wh + woff, ws.wl + woff, N, M);
}

// K / V summary of a cross layer from the raw reference tokens r [L][D] (pre_norm_query: no norm1)
static int cross_kv(const float* r, int L, int blk, float* kvc_out, const Ws& ws, cudaStream_t s) {
  int rc;
  if ((rc = launch_split_f16(r, D, ws.att2, 2 * D, L, D, s))) return rc;
  TcsArgs a = gemm(ws, ws.att2, 2 * D, D, blk * G_BLK + G_QKV + (size_t)D * D, 2 * D, L);   // rows k_proj; v_proj
  a.elu_cols = D; a.C = ws.qkv; a.ldc = 2 * D;
  if ((rc = launch_linear_tcs(a, LIN_ELU1, s))) return rc;
  return launch_kv_summary<12, 64>(ws.qkv, 2 * D, 0, D, L, 1, ws.kvp, kvc_out, s);
}

// one CrossBlock over M tokens at x (in place): self attention when kvc == nullptr (M == L), else cross attention
// against the summary kvc.  ln1_ready: ws.xn2 already holds split(norm1(x)).
static int run_block(float* x, int M, int L, int blk, const float* kvc, bool ln1_ready, const Ws& ws, cudaStream_t s) {
  const float* sp = ws.w + blk * S_BLK;
  int rc;
  if (!ln1_ready) {
    layernorm_split_kernel<D><<<cdiv(M, 8), 256, 0, s>>>(x, sp + S_N1W, sp + S_N1B, ws.xn2, M, 1e-5f);
    MVSF_LAUNCH_CHECK("vit_decoder_ln1");
  }
  const size_t wb = blk * G_BLK;
  int ldq;
  if (!kvc) {
    TcsArgs a = gemm(ws, ws.xn2, 2 * D, D, wb + G_QKV, 3 * D, M);
    a.elu_cols = 2 * D; a.C = ws.qkv; a.ldc = 3 * D;
    if ((rc = launch_linear_tcs(a, LIN_ELU1, s))) return rc;
    if ((rc = launch_kv_summary<12, 64>(ws.qkv, 3 * D, D, 2 * D, L, 1, ws.kvp, ws.kvf, s))) return rc;
    kvc = ws.kvf; ldq = 3 * D;
  } else {
    TcsArgs a = gemm(ws, ws.xn2, 2 * D, D, wb + G_QKV, D, M);
    a.elu_cols = D; a.C = ws.qkv; a.ldc = D;
    if ((rc = launch_linear_tcs(a, LIN_ELU1, s))) return rc;
    ldq = D;
  }
  linattn_apply_kernel<12, 64><<<dim3(cdiv(M, 128), 12), 128, 0, s>>>(ws.qkv, ldq, kvc, 0, ws.att2, M, M);
  MVSF_LAUNCH_CHECK("vit_decoder_linattn_apply");
  TcsArgs p = gemm(ws, ws.att2, 2 * D, D, wb + G_PROJ, D, M);   // x += ls1 * proj(attn)
  p.bias = sp + S_PB; p.res = x; p.ldres = D; p.gamma = sp + S_LS1; p.C = x; p.ldc = D;
  if ((rc = launch_linear_tcs(p, LIN_RES, s))) return rc;
  layernorm_split_kernel<D><<<cdiv(M, 8), 256, 0, s>>>(x, sp + S_N2W, sp + S_N2B, ws.xn2, M, 1e-5f);
  MVSF_LAUNCH_CHECK("vit_decoder_ln2");
  TcsArgs f1 = gemm(ws, ws.xn2, 2 * D, D, wb + G_FC1, HID, M);
  f1.bias = sp + S_F1B; f1.C2 = ws.hid2; f1.ldc2 = 2 * HID;
  if ((rc = launch_linear_tcs(f1, LIN_GELU, s))) return rc;
  TcsArgs f2 = gemm(ws, ws.hid2, 2 * HID, HID, wb + G_FC2, D, M);   // x += ls2 * fc2(gelu(fc1(norm2(x))))
  f2.bias = sp + S_F2B; f2.res = x; f2.ldres = D; f2.gamma = sp + S_LS2; f2.C = x; f2.ldc = D;
  return launch_linear_tcs(f2, LIN_RES, s);
}

static int combine(float* x, const float* xi, int M, int i, int next_blk, const Ws& ws, cudaStream_t s) {
  const float* nl = ws.w + P_NORM + 2 * i * D;
  const float* nb = next_blk >= 0 ? ws.w + next_blk * S_BLK : nullptr;
  combine_kernel<<<cdiv(M, 8), 256, 0, s>>>(x, xi, ws.w + P_PREV + i, nl, nl + D, nb ? nb + S_N1W : nullptr,
                                            nb ? nb + S_N1B : nullptr, ws.xn2, M);
  MVSF_LAUNCH_CHECK("vit_decoder_combine");
  return MVSF_OK;
}

// ConvTranspose2d(k4, s2, p1) in gather form: output row 2y + py reads input rows y (ky = 1 + py) and y - 1 + 2 py
// (ky = 3 - 3 py); same for columns.  Class taps t = 2 ty + tx.
static unsigned long long deconv_taps(int py, int px) {
  unsigned long long taps = 0;
  for (int t = 0; t < 4; ++t) {
    const int dy = (t >> 1) ? (py ? 1 : -1) : 0, dx = (t & 1) ? (px ? 1 : -1) : 0;
    taps |= (unsigned long long)((dy + 1) | ((dx + 1) << 2)) << (4 * t);
  }
  return taps;
}

static bool shape_ok(int B, int V, int h, int w) {
  return B >= 1 && V >= 2 && h >= 1 && w >= 1 && h < 2048 && w < 2048 && (long long)B * V * h * w * 16 < (1ll << 31);
}

struct Layout {
  size_t T, xn2, att2, hid2, qkv, kvp, kvf, kvc, p0, p1, p2, total;   // float offsets
};
static Layout layout(int B, int V, int h, int w) {
  const size_t L = (size_t)h * w, Ms = (size_t)(V - 1) * L, Mx = Ms > L ? Ms : L, BVL = (size_t)B * V * L;
  const size_t nblk = (L + KV_CHUNK - 1) / KV_CHUNK;
  size_t o = 0;
  auto take = [&](size_t n) { const size_t r = o; o += align_up(n, 64); return r; };
  Layout l;
  l.T = take(BVL * D);
  l.xn2 = take(Mx * D);
  l.att2 = take(Mx * D);
  l.hid2 = take(Mx * HID);
  l.qkv = take(L * 3 * D > Ms * D ? L * 3 * D : Ms * D);
  l.kvp = take(nblk * KVSZ);
  l.kvf = take(KVSZ);
  l.kvc = take(3 * (size_t)KVSZ);
  l.p0 = take(BVL * D);
  l.p1 = take(BVL * 256);
  l.p2 = take(BVL * 4 * 128);
  l.total = o;
  return l;
}

}  // namespace vitdec
}  // namespace mvsf

using namespace mvsf;
using namespace mvsf::vitdec;

extern "C" int mvsf_vit_decoder_workspace_bytes(int B, int V, int h, int w, size_t* bytes) {
  MVSF_REQUIRE(bytes, "vit_decoder_workspace_bytes: null pointer");
  MVSF_REQUIRE(shape_ok(B, V, h, w), "vit_decoder: need B >= 1, V >= 2, 1 <= h, w < 2048 (got B=%d V=%d h=%d w=%d)", B,
               V, h, w);
  *bytes = layout(B, V, h, w).total * sizeof(float);
  return MVSF_OK;
}

extern "C" int mvsf_vit_decoder_forward(const float* x0, const float* x1, const float* x2, const float* wts,
                                        const void* wts_tc, float* out, void* workspace, size_t workspace_bytes, int B,
                                        int V, int h, int w, mvsf_stream_t stream) {
  size_t need = 0;
  if (mvsf_vit_decoder_workspace_bytes(B, V, h, w, &need) != MVSF_OK) return MVSF_ERR_INVALID;
  MVSF_REQUIRE(x0 && x1 && x2 && wts && wts_tc && out && workspace, "vit_decoder_forward: null pointer");
  MVSF_REQUIRE(((uintptr_t)x0 & 15) == 0 && ((uintptr_t)x1 & 15) == 0 && ((uintptr_t)x2 & 15) == 0 &&
                   ((uintptr_t)wts & 15) == 0 && ((uintptr_t)wts_tc & 15) == 0 && ((uintptr_t)out & 15) == 0 &&
                   ((uintptr_t)workspace & 15) == 0,
               "vit_decoder_forward: pointers must be 16-byte aligned");
  if (workspace_bytes < need)
    return fail(MVSF_ERR_WORKSPACE, "vit_decoder_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  const Layout l = layout(B, V, h, w);
  float* base = static_cast<float*>(workspace);
  Ws ws;
  ws.xn2 = reinterpret_cast<__half*>(base + l.xn2);
  ws.att2 = reinterpret_cast<__half*>(base + l.att2);
  ws.hid2 = reinterpret_cast<__half*>(base + l.hid2);
  ws.qkv = base + l.qkv; ws.kvp = base + l.kvp; ws.kvf = base + l.kvf; ws.kvc = base + l.kvc;
  ws.w = wts;
  ws.wh = static_cast<const __half*>(wts_tc);
  ws.wl = ws.wh + NG;
  float* T = base + l.T;   // token map [B][V][L][D]: r2 in view 0, the cross-attended source views after it
  const int L = h * w, Ms = (V - 1) * L;
  const size_t VLD = (size_t)V * L * D, LD = (size_t)L * D;
  int rc;
  for (int b = 0; b < B; ++b) {
    const float* xr[3] = {x0 + b * VLD, x1 + b * VLD, x2 + b * VLD};
    float* X = T + b * VLD;
    // reference view (module.py:322-333): r0 = x0; r_i = norm_layers[i-1](p * SelfBlock_{i-1}(r_{i-1}) + x_i)
    MVSF_CUDA_OK(cudaMemcpyAsync(X, xr[0], LD * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if ((rc = cross_kv(xr[0], L, 2, ws.kvc, ws, s))) return rc;
    if ((rc = run_block(X, L, L, 0, nullptr, false, ws, s))) return rc;
    if ((rc = combine(X, xr[1], L, 0, 1, ws, s))) return rc;
    if ((rc = cross_kv(X, L, 3, ws.kvc + KVSZ, ws, s))) return rc;
    if ((rc = run_block(X, L, L, 1, nullptr, true, ws, s))) return rc;
    if ((rc = combine(X, xr[2], L, 1, -1, ws, s))) return rc;
    if ((rc = cross_kv(X, L, 4, ws.kvc + 2 * KVSZ, ws, s))) return rc;
    // source views as one batch (module.py:334-346): Cross0(x0), then Cross_i(norm_layers[i-1](p * s + x_i))
    float* Xs = X + LD;
    MVSF_CUDA_OK(cudaMemcpyAsync(Xs, xr[0] + LD, (size_t)Ms * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if ((rc = run_block(Xs, Ms, L, 2, ws.kvc, false, ws, s))) return rc;
    if ((rc = combine(Xs, xr[1] + LD, Ms, 0, 3, ws, s))) return rc;
    if ((rc = run_block(Xs, Ms, L, 3, ws.kvc + KVSZ, true, ws, s))) return rc;
    if ((rc = combine(Xs, xr[2] + LD, Ms, 1, 4, ws, s))) return rc;
    if ((rc = run_block(Xs, Ms, L, 4, ws.kvc + 2 * KVSZ, true, ws, s))) return rc;
  }
  // conv head over all B*V token maps (module.py:359-362), NHWC
  const int imgs = B * V;
  __half* P0 = reinterpret_cast<__half*>(base + l.p0);
  __half* P1 = reinterpret_cast<__half*>(base + l.p1);
  __half* P2 = reinterpret_cast<__half*>(base + l.p2);
  if ((rc = launch_split_f16(T, D, P0, 2 * D, imgs * L, D, s))) return rc;
  const float* cb = wts + P_CB;
  {
    TcsArgs a{};
    a.Ah = P0; a.Al = P0 + D; a.lda = 2 * D;
    a.Bh = ws.wh + G_CONV; a.Bl = ws.wl + G_CONV; a.ldb = 9 * D;
    a.M = imgs * L; a.N = 256; a.K = 9 * D;
    a.H = h; a.W = w; a.cin = D; a.ntaps = 9; a.sy = a.sx = 1;
    for (int t = 0; t < 9; ++t) a.taps |= (unsigned long long)((t / 3) | ((t % 3) << 2)) << (4 * t);
    a.bias = cb; a.C2 = P1; a.ldc2 = 512;
    if ((rc = launch_linear_tcs(a, LIN_SILU, s))) return rc;
  }
  for (int cls = 0; cls < 4; ++cls) {   // upsampler0: [imgs][h][w][256] -> [imgs][2h][2w][128]
    TcsArgs a{};
    a.Ah = P1; a.Al = P1 + 256; a.lda = 512;
    a.Bh = ws.wh + G_UP0 + (size_t)cls * 128 * 1024; a.Bl = ws.wl + G_UP0 + (size_t)cls * 128 * 1024; a.ldb = 1024;
    a.M = imgs * L; a.N = 128; a.K = 1024;
    a.H = h; a.W = w; a.cin = 256; a.ntaps = 4; a.taps = deconv_taps(cls >> 1, cls & 1);
    a.sy = a.sx = 2; a.py = cls >> 1; a.px = cls & 1;
    a.bias = cb + 256; a.C2 = P2; a.ldc2 = 256;
    if ((rc = launch_linear_tcs(a, LIN_SILU, s))) return rc;
  }
  for (int cls = 0; cls < 4; ++cls) {   // upsampler1: [imgs][2h][2w][128] -> out [imgs][4h][4w][64]
    TcsArgs a{};
    a.Ah = P2; a.Al = P2 + 128; a.lda = 256;
    a.Bh = ws.wh + G_UP1 + (size_t)cls * 64 * 512; a.Bl = ws.wl + G_UP1 + (size_t)cls * 64 * 512; a.ldb = 512;
    a.M = imgs * 4 * L; a.N = 64; a.K = 512;
    a.H = 2 * h; a.W = 2 * w; a.cin = 128; a.ntaps = 4; a.taps = deconv_taps(cls >> 1, cls & 1);
    a.sy = a.sx = 2; a.py = cls >> 1; a.px = cls & 1;
    a.bias = cb + 384; a.C = out; a.ldc = 64;
    if ((rc = launch_linear_tcs(a, LIN_SILU, s))) return rc;
  }
  return MVSF_OK;
}
