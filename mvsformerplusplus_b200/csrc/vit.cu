// V2: DinoVisionTransformer.forward_interval_features (models/dino/dinov2.py:249-266), shipped configuration: ViT-B/14
// (embed 768, 12 blocks, 12 heads of 64, mlp 3072 exact-erf GELU, LayerScale, LayerNorm eps 1e-6, qkv / proj / ffn
// biases, softmax scale 1/8), cross_interval_layers = 3: the raw outputs of blocks 3 and 7 and norm(x) after block 11,
// each without the cls token.
//   * patch embedding (patch_embed.py:76-78): SIMT im2col to fp16 hi|lo rows (K = 3 * 14 * 14 = 588, zero-padded to
//     640), then the streamed-weight GEMM of linear_tc.cu with bias, straight into the residual stream;
//   * tokens (dinov2.py:202-211): x[cls] = cls + pos[0], x[patch p] = patch[p] + pos[1 + p]; the same row kernel writes
//     block 0's norm1 split.  pos is the interpolated pos_embed of the patch grid, computed once per grid at pack time;
//   * blocks (block.py:85-120): norm1 split, qkv GEMM (bias), softmax attention (vit_attention.cuh), proj GEMM with the
//     LayerScale residual, norm2 split, fc1 GEMM with GELU to hi|lo, fc2 GEMM with the LayerScale residual;
//   * final norm (dinov2.py:263) of the patch rows into the third output.
// Token rows: the patch tokens of all images first (image-major), then the n cls rows (vfa::token_row with cls_last):
// attention gathers each image's tokens through that map, everything else is row-wise.  So the patch rows of the
// residual stream ARE the [n, gh * gw, 768] interval output, contiguous: blocks 0-3 run in out0, block 4's proj
// epilogue writes its residual sum into out1 (out0 keeps the block-3 output), and block 8's into a workspace stream.
#include "linattn.cuh"
#include "linear_tc.cuh"
#include "vit_attention.cuh"

namespace mvsf {
namespace vit {

constexpr int D = 768, HID = 3072, NBLK = 12, PATCH = 14, KP = 588, KPAD = 640;
// ---- GEMM weights (the gemm part of packing.pack_vit), fp32 [N][K] rows; the tc blob holds their hi / lo splits with
// the same indexing
constexpr size_t G_PATCH = 0, G_BLK0 = (size_t)D * KPAD;   // patch_embed.proj [768][640] (k = c * 196 + ky * 14 + kx)
constexpr size_t G_QKV = 0, G_PROJ = (size_t)3 * D * D, G_FC1 = (size_t)4 * D * D, G_FC2 = G_FC1 + (size_t)HID * D,
                 G_BLK = G_FC2 + (size_t)D * HID;
constexpr size_t NG = G_BLK0 + NBLK * G_BLK;
// ---- small fp32 parameters (the small part of packing.pack_vit, the wts argument): per block norm1 w, b,
// qkv bias [2304], proj bias, ls1, norm2 w, b, fc1 bias [3072], fc2 bias, ls2; then patch bias, cls token, norm w, b
constexpr size_t S_N1W = 0, S_N1B = D, S_QKVB = 2 * D, S_PB = 5 * D, S_LS1 = 6 * D, S_N2W = 7 * D, S_N2B = 8 * D,
                 S_F1B = 9 * D, S_F2B = 13 * D, S_LS2 = 14 * D, S_BLK = 15 * D;
constexpr size_t P_PATCHB = NBLK * S_BLK, P_CLS = P_PATCHB + D, P_NW = P_CLS + D, P_NB = P_NW + D, NS = P_NB + D;
static_assert(NG == 85426176 && NS == 141312, "packing.VIT_GEMM_WTS / VIT_SMALL_WTS");
constexpr float LN_EPS = 1e-6f;

// im2col of the 14 x 14 / stride-14 patch conv: row b * P + py * gw + px = [hi(640) | lo(640)], k = c * 196 + ky * 14 + kx
// (proj.weight.reshape(768, 588) order), k >= 588 zero.  One thread per (row, 8 consecutive k).
__global__ void patch_im2col_kernel(const float* __restrict__ img, __half* __restrict__ rows, int n, int gh, int gw) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int P = gh * gw, oct = (int)(i % (KPAD / 8));
  const long long row = i / (KPAD / 8);
  if (row >= (long long)n * P) return;
  const int b = (int)(row / P), p = (int)(row % P), py = p / gw, px = p % gw;
  const int H = gh * PATCH, W = gw * PATCH;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = oct * 8 + e;
    if (k < KP) {
      const int c = k / 196, r = k % 196, ky = r / PATCH, kx = r % PATCH;
      v[e] = __ldg(img + (((size_t)b * 3 + c) * H + py * PATCH + ky) * W + px * PATCH + kx);
    } else {
      v[e] = 0.f;
    }
  }
  __half* dst = rows + (size_t)row * 2 * KPAD + oct * 8;
  split_store8(dst, dst + KPAD, v);
}

// ATen upsample_bicubic2d (UpSample.h get_cubic_upsample_coefficients, A = -0.75)
__device__ __forceinline__ void cubic_coeffs(float t, float c[4]) {
  constexpr float A = -0.75f;
  const float x1 = t + 1.f, x2 = 1.f - t, x3 = x2 + 1.f;
  c[0] = ((A * x1 - 5.f * A) * x1 + 8.f * A) * x1 - 4.f * A;
  c[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
  c[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  c[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}

// patch_im2col_kernel on the image resized from H x W to 14 gh x 14 gw the way F.interpolate(mode="bicubic",
// align_corners=False) does it (ATen upsample_bicubic2d: scale in / out, source index scale (dst + 0.5) - 0.5, the four
// taps clamped to the border, each row interpolated along x first, then the four rows along y).  The resized image never
// reaches memory: each im2col element is evaluated from its 16 source pixels.
__global__ void patch_im2col_bicubic_kernel(const float* __restrict__ img, __half* __restrict__ rows, int n, int gh,
                                            int gw, int H, int W) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int P = gh * gw, oct = (int)(i % (KPAD / 8));
  const long long row = i / (KPAD / 8);
  if (row >= (long long)n * P) return;
  const int b = (int)(row / P), p = (int)(row % P), py = p / gw, px = p % gw;
  const float sy = (float)H / (float)(gh * PATCH), sx = (float)W / (float)(gw * PATCH);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = oct * 8 + e;
    v[e] = 0.f;
    if (k < KP) {
      const int c = k / 196, r = k % 196, ky = r / PATCH, kx = r % PATCH;
      const float ry = sy * ((float)(py * PATCH + ky) + 0.5f) - 0.5f, rx = sx * ((float)(px * PATCH + kx) + 0.5f) - 0.5f;
      const float fy = floorf(ry), fx = floorf(rx);
      const int iy = (int)fy, ix = (int)fx;
      float cy[4], cx[4];
      cubic_coeffs(ry - fy, cy);
      cubic_coeffs(rx - fx, cx);
      int xs[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) xs[t] = min(max(ix - 1 + t, 0), W - 1);
      const float* plane = img + ((size_t)b * 3 + c) * H * W;
      float acc = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float* src = plane + (size_t)min(max(iy - 1 + t, 0), H - 1) * W;
        const float rowv = __ldg(src + xs[0]) * cx[0] + __ldg(src + xs[1]) * cx[1] + __ldg(src + xs[2]) * cx[2] +
                           __ldg(src + xs[3]) * cx[3];
        acc = t == 0 ? rowv * cy[0] : acc + rowv * cy[t];
      }
      v[e] = acc;
    }
  }
  __half* dst = rows + (size_t)row * 2 * KPAD + oct * 8;
  split_store8(dst, dst + KPAD, v);
}

// x rows [0, n P): patch embedding (conv output with bias) += pos[1 + p]; rows n P + b: cls + pos[0]
// (prepare_tokens_with_masks: cat(cls, patches) + pos).  Then xn2 <- split(norm1_0(x)).  One warp per row.
__global__ void __launch_bounds__(256)
tokens_kernel(float* __restrict__ x, const float* __restrict__ pos, const float* __restrict__ cls,
              const float* __restrict__ lw, const float* __restrict__ lb, __half* __restrict__ xn2, int n, int P) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n * (P + 1)) return;
  RowVec<D> r, pe;
  if (row < n * P) {
    r.load(x + (size_t)row * D, lane);
    pe.load(pos + (size_t)(1 + row % P) * D, lane);
  } else {
    r.load(cls, lane);
    pe.load(pos, lane);
  }
#pragma unroll
  for (int e = 0; e < RowVec<D>::E; ++e) r.v[e] = __fadd_rn(r.v[e], pe.v[e]);
  r.store(x + (size_t)row * D, lane);
  r.layernorm(lw, lb, LN_EPS, lane);
  r.store_split(xn2 + (size_t)row * 2 * D, lane);
}

// out[row] = norm(x[row]) for the patch rows (dinov2.py:263-264)
__global__ void __launch_bounds__(256)
final_norm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                  float* __restrict__ out, int M) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  RowVec<D> r;
  r.load(x + (size_t)row * D, lane);
  r.layernorm(w, b, LN_EPS, lane);
  r.store(out + (size_t)row * D, lane);
}

static bool shape_ok(int n, int gh, int gw) {
  return n >= 1 && gh >= 1 && gw >= 1 && n <= 65535 && gh <= 1024 && gw <= 1024 &&
         (long long)n * (gh * gw + 1) <= (1ll << 21);
}

static int attention(const float* qkv, int ldq, float* out, int ldo, __half* out2, __half* tiled, int n, int N,
                     bool cls_last, cudaStream_t s) {
  const int nt = cdiv(N, 128);
  const long long threads = (long long)n * nt * 128 * 3 * vfa::NH * 8;
  vit_qkv_tile_kernel<<<cdiv(threads, 256), 256, 0, s>>>(qkv, ldq, tiled, n, N, nt, cls_last,
                                                         0.125f * 1.4426950408889634f);
  MVSF_LAUNCH_CHECK("vit_qkv_tile");
  static DeviceOnce once;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(vit_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vfa::Layout::SMEM));
    once.done(dev);
  }
  cudaEvent_t kt = ktimer_enabled() ? ktimer_begin("vit_attention", s) : nullptr;
  vit_attention_kernel<<<dim3(cdiv(N, 128), vfa::NH, n), vfa::Layout::THREADS, vfa::Layout::SMEM, s>>>(tiled, out, ldo, out2,
                                                                                                         n, N, nt, cls_last);
  if (kt) ktimer_end(kt, s);
  MVSF_LAUNCH_CHECK("vit_attention");
  return MVSF_OK;
}

struct Layout {
  size_t act2, hid2, qkv, tiled, x3, total;   // float offsets
};
static Layout layout(int n, int gh, int gw) {
  const size_t N = (size_t)gh * gw + 1, M = (size_t)n * N;
  size_t o = 0;
  auto take = [&](size_t k) { const size_t r = o; o += align_up(k, 64); return r; };
  Layout l;
  l.act2 = take(M * D);       // [M][2D] halves: norm1 / norm2 splits and the attention output split
  l.hid2 = take(M * HID);     // [M][2 HID] halves: fc1 output split; the patch im2col rows before block 0
  l.qkv = take(M * 3 * D);
  l.tiled = take(vfa::tiled_halves(n, cdiv(N, 128)) / 2);
  l.x3 = take(M * D);         // residual stream of blocks 8-11
  l.total = o;
  return l;
}

}  // namespace vit
}  // namespace mvsf

using namespace mvsf;
using namespace mvsf::vit;

extern "C" int mvsf_vit_workspace_bytes(int n, int gh, int gw, size_t* bytes) {
  MVSF_REQUIRE(bytes, "vit_workspace_bytes: null pointer");
  MVSF_REQUIRE(shape_ok(n, gh, gw), "vit: need 1 <= n <= 65535, 1 <= gh, gw <= 1024, n (gh gw + 1) <= 2^21 (got n=%d gh=%d gw=%d)",
               n, gh, gw);
  *bytes = layout(n, gh, gw).total * sizeof(float);
  return MVSF_OK;
}

extern "C" int mvsf_vit_attention_forward(const float* qkv, int ldq, float* out, int ldo, void* workspace,
                                          size_t workspace_bytes, int n, int N, mvsf_stream_t stream) {
  MVSF_REQUIRE(n >= 1 && n <= 65535 && N >= 1 && (long long)n * N <= (1ll << 21),
               "vit_attention: need 1 <= n <= 65535, N >= 1, n N <= 2^21 (got n=%d N=%d)", n, N);
  MVSF_REQUIRE(qkv && out && workspace, "vit_attention: null pointer");
  MVSF_REQUIRE(ldq >= 3 * D && ldq % 4 == 0 && ldo >= D && ldo % 4 == 0 && ((uintptr_t)qkv & 15) == 0 &&
                   ((uintptr_t)out & 15) == 0 && ((uintptr_t)workspace & 15) == 0,
               "vit_attention: need ldq >= 2304, ldo >= 768 (multiples of 4) and 16-byte aligned pointers");
  const size_t need = vfa::tiled_halves(n, cdiv(N, 128)) * sizeof(__half);
  if (workspace_bytes < need)
    return fail(MVSF_ERR_WORKSPACE, "vit_attention: workspace %zu < %zu bytes", workspace_bytes, need);
  return vit::attention(qkv, ldq, out, ldo, nullptr, static_cast<__half*>(workspace), n, N, false, (cudaStream_t)stream);
}

// the forward of both entry points: img [n][3][H][W], resized to 14 gh x 14 gw inside the patch im2col when `resize`
static int vit_forward(const float* img, int H, int W, bool resize, const float* pos, const float* wts,
                       const void* wts_tc, float* out0, float* out1, float* out2, void* workspace, size_t workspace_bytes,
                       int n, int gh, int gw, mvsf_stream_t stream) {
  size_t need = 0;
  if (mvsf_vit_workspace_bytes(n, gh, gw, &need) != MVSF_OK) return MVSF_ERR_INVALID;
  MVSF_REQUIRE(img && pos && wts && wts_tc && out0 && out1 && out2 && workspace, "vit_forward: null pointer");
  MVSF_REQUIRE(((uintptr_t)img & 15) == 0 && ((uintptr_t)pos & 15) == 0 && ((uintptr_t)wts & 15) == 0 &&
                   ((uintptr_t)wts_tc & 15) == 0 && ((uintptr_t)out0 & 15) == 0 && ((uintptr_t)out1 & 15) == 0 &&
                   ((uintptr_t)out2 & 15) == 0 && ((uintptr_t)workspace & 15) == 0,
               "vit_forward: pointers must be 16-byte aligned");
  if (workspace_bytes < need)
    return fail(MVSF_ERR_WORKSPACE, "vit_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  const Layout l = layout(n, gh, gw);
  float* base = static_cast<float*>(workspace);
  __half* act2 = reinterpret_cast<__half*>(base + l.act2);
  __half* hid2 = reinterpret_cast<__half*>(base + l.hid2);
  float* qkv = base + l.qkv;
  __half* tiled = reinterpret_cast<__half*>(base + l.tiled);
  const __half* wh = static_cast<const __half*>(wts_tc);
  const __half* wl = wh + NG;
  const int P = gh * gw, N = P + 1, M = n * N;
  int rc;
  // patch embedding straight into the patch rows of the stream, then the tokens and block 0's norm1
  const long long im2col_threads = (long long)n * P * (KPAD / 8);
  if (resize) {
    patch_im2col_bicubic_kernel<<<cdiv(im2col_threads, 256), 256, 0, s>>>(img, hid2, n, gh, gw, H, W);
    MVSF_LAUNCH_CHECK("vit_patch_im2col_bicubic");
  } else {
    patch_im2col_kernel<<<cdiv(im2col_threads, 256), 256, 0, s>>>(img, hid2, n, gh, gw);
    MVSF_LAUNCH_CHECK("vit_patch_im2col");
  }
  {
    TcsArgs a = tcs_rows(hid2, 2 * KPAD, KPAD, wh + G_PATCH, wl + G_PATCH, D, n * P);
    a.bias = wts + P_PATCHB; a.C = out0; a.ldc = D;
    if ((rc = launch_linear_tcs(a, LIN_BIAS, s))) return rc;
  }
  tokens_kernel<<<cdiv(M, 8), 256, 0, s>>>(out0, pos, wts + P_CLS, wts + S_N1W, wts + S_N1B, act2, n, P);
  MVSF_LAUNCH_CHECK("vit_tokens");
  float* x = out0;
  for (int blk = 0; blk < NBLK; ++blk) {
    const float* sp = wts + blk * S_BLK;
    const size_t wb = G_BLK0 + blk * G_BLK;
    if (blk > 0) {
      layernorm_split_kernel<D><<<cdiv(M, 8), 256, 0, s>>>(x, sp + S_N1W, sp + S_N1B, act2, M, LN_EPS);
      MVSF_LAUNCH_CHECK("vit_ln1");
    }
    TcsArgs q = tcs_rows(act2, 2 * D, D, wh + wb + G_QKV, wl + wb + G_QKV, 3 * D, M);
    q.bias = sp + S_QKVB; q.C = qkv; q.ldc = 3 * D;
    if ((rc = launch_linear_tcs(q, LIN_BIAS, s))) return rc;
    if ((rc = vit::attention(qkv, 3 * D, nullptr, 0, act2, tiled, n, N, true, s))) return rc;
    // x += ls1 * proj(attn).  Blocks 4 and 8 write the sum into a fresh stream: the old one keeps the interval output
    float* xo = blk == 4 ? out1 : blk == 8 ? base + l.x3 : x;
    TcsArgs p = tcs_rows(act2, 2 * D, D, wh + wb + G_PROJ, wl + wb + G_PROJ, D, M);
    p.bias = sp + S_PB; p.res = x; p.ldres = D; p.gamma = sp + S_LS1; p.C = xo; p.ldc = D;
    if ((rc = launch_linear_tcs(p, LIN_RES, s))) return rc;
    x = xo;
    layernorm_split_kernel<D><<<cdiv(M, 8), 256, 0, s>>>(x, sp + S_N2W, sp + S_N2B, act2, M, LN_EPS);
    MVSF_LAUNCH_CHECK("vit_ln2");
    TcsArgs f1 = tcs_rows(act2, 2 * D, D, wh + wb + G_FC1, wl + wb + G_FC1, HID, M);
    f1.bias = sp + S_F1B; f1.C2 = hid2; f1.ldc2 = 2 * HID;
    if ((rc = launch_linear_tcs(f1, LIN_GELU, s))) return rc;
    TcsArgs f2 = tcs_rows(hid2, 2 * HID, HID, wh + wb + G_FC2, wl + wb + G_FC2, D, M);   // x += ls2 * fc2(gelu(...))
    f2.bias = sp + S_F2B; f2.res = x; f2.ldres = D; f2.gamma = sp + S_LS2; f2.C = x; f2.ldc = D;
    if ((rc = launch_linear_tcs(f2, LIN_RES, s))) return rc;
  }
  final_norm_kernel<<<cdiv(n * P, 8), 256, 0, s>>>(x, wts + P_NW, wts + P_NB, out2, n * P);
  MVSF_LAUNCH_CHECK("vit_final_norm");
  return MVSF_OK;
}

extern "C" int mvsf_vit_forward(const float* img, const float* pos, const float* wts, const void* wts_tc, float* out0,
                                float* out1, float* out2, void* workspace, size_t workspace_bytes, int n, int gh, int gw,
                                mvsf_stream_t stream) {
  return vit_forward(img, PATCH * gh, PATCH * gw, false, pos, wts, wts_tc, out0, out1, out2, workspace, workspace_bytes, n,
                     gh, gw, stream);
}

extern "C" int mvsf_vit_forward_image(const float* img, int H, int W, const float* pos, const float* wts,
                                      const void* wts_tc, float* out0, float* out1, float* out2, void* workspace,
                                      size_t workspace_bytes, int n, int gh, int gw, mvsf_stream_t stream) {
  MVSF_REQUIRE(H >= 1 && W >= 1 && (long long)H * W < (1ll << 30),
               "vit_forward_image: need 1 <= H, W and H W < 2^30 (got H=%d W=%d)", H, W);
  return vit_forward(img, H, W, true, pos, wts, wts_tc, out0, out1, out2, workspace, workspace_bytes, n, gh, gw, stream);
}
