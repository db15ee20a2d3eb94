// Softmax attention of the DINOv2 ViT-B blocks (models/dino/layers/attention.py:77-101: 12 heads of 64, non-causal,
// scale head_dim ** -0.5 = 1/8) on wgmma: the layout policy of softmax_attention.cuh for head dim 64.  Included by vit.cu.
//
// One CTA works on 128 query rows of one (image, head): two consumer warpgroups, K and V^T tiles of 128 keys (pre-tiled
// by vit_qkv_tile_kernel) through rings of NKV = 2 stages.  Per 128-key tile: S = three m64n128 products per 16 head
// dims; P against the V^T tile's rows [V_hi (64) | 1 | 0 (7)] (N = 72), then P against the V_lo rows (N = 64) into the
// same accumulator.
// Shared memory: a stage holds K hi + lo (32 KB) and the V^T tile (34 KB), so two stages and two consumer warpgroups
// (164 KB with the Q blocks) fit one SM; a third stage would not.  Per thread the loop keeps 64 scores, 36 P*V
// accumulators, 32 running outputs and 32 packed P registers: the producer gives its registers to the consumers
// (setmaxnreg 40 / 232).  At hd 64 a key tile costs 64 exponentials per row against 6 x 128 x 64 + 2 x 136 x 128
// multiply-adds, so unlike the hd-16 kernel the loop is bound by the tensor core, not the exp unit.
#pragma once
#include <cuda_fp16.h>

#include "linear_tc.cuh"
#include "softmax_attention.cuh"
#include "wgmma.cuh"

namespace mvsf {
namespace vfa {
using namespace gmma;
constexpr int NH = 12, HD = 64;
constexpr uint32_t LBO_K = 2048, LBO_Q = 1024;          // k-chunk (8 head dims) strides: K 128 rows, Q block 64 rows
constexpr uint32_t K_TILE = 8 * LBO_K;                   // 16 KB: one 128-key x 64-dim fp16 tile (hi or lo)
constexpr uint32_t Q_TILE = 8 * LBO_Q;                   // 8 KB: one 64-query block (hi or lo)
constexpr int VROWS = 136;                               // V^T rows: V_hi dims 0-63 | ones | 7 zero rows | V_lo dims 0-63
constexpr uint32_t LBO_V = VROWS * 16, V_TILE = 16 * LBO_V, V_LO = 9 * 128;   // 16 key chunks; V_lo starts at row 72
// halves of one (image, head) in each plane of the tiled buffer
__host__ __device__ constexpr size_t q_plane(int nqb) { return (size_t)nqb * (Q_TILE / 2); }
__host__ __device__ constexpr size_t k_plane(int nt) { return (size_t)nt * (K_TILE / 2); }
__host__ __device__ constexpr size_t v_plane(int nt) { return (size_t)nt * (V_TILE / 2); }
// tiled buffer: Q hi, Q lo, K hi, K lo, V^T planes, each [image][head][...]
__host__ __device__ constexpr size_t tiled_halves(int n, int nt) {
  return (size_t)n * NH * (2 * q_plane(2 * nt) + 2 * k_plane(nt) + v_plane(nt));
}

// row of token t of image b in the token-row buffers: the natural order b * N + t, or (cls_last) the patch tokens of
// all images first and the n cls rows after them, so that the patch rows of the residual stream are the contiguous
// [n, N - 1, 768] interval output
__host__ __device__ __forceinline__ size_t token_row(int b, int t, int n, int N, bool cls_last) {
  if (!cls_last) return (size_t)b * N + t;
  return t ? (size_t)b * (N - 1) + t - 1 : (size_t)n * (N - 1) + b;
}
}  // namespace vfa

// qkv rows (nn.Linear output [.., 2304] = [q | k | v] x 12 heads x 64) -> the tiled fp16 hi / lo operands.  Q is
// pre-scaled by qscale = 1/8 * log2(e) (the kernel uses exp2).  One thread per (image, token, q/k/v, head, 8 dims); rows
// >= N are zero, and so is the ones row of V for keys >= N.
__global__ void vit_qkv_tile_kernel(const float* __restrict__ qkv, int ldq, __half* __restrict__ tiled, int n, int N,
                                    int nt, bool cls_last, float qscale) {
  using namespace vfa;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (b, token, which, head, octet)
  const long long total = (long long)n * nt * 128 * 3 * NH * 8;
  if (i >= total) return;
  const int oct = (int)(i & 7), head = (int)((i >> 3) % NH), which = (int)((i / (8 * NH)) % 3);
  const long long bt = i / (8 * NH * 3);
  const int t = (int)(bt % (nt * 128)), b = (int)(bt / (nt * 128));
  float v[8];
  if (t < N) {
    const float* src = qkv + token_row(b, t, n, N, cls_last) * ldq + which * (NH * HD) + head * HD + oct * 8;
    const float4 a = ldg4(src), c = ldg4(src + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
    if (which == 0) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= qscale;
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  }
  const size_t bh = (size_t)b * NH + head, qp = q_plane(2 * nt), kp = k_plane(nt);
  const size_t planes = (size_t)n * NH;
  if (which == 0) {
    __half* ph = tiled + bh * qp + (size_t)(t >> 6) * (Q_TILE / 2) + oct * (LBO_Q / 2) + (t & 63) * 8;
    split_store8(ph, ph + planes * qp, v);
  } else if (which == 1) {
    __half* ph = tiled + 2 * planes * qp + bh * kp + (size_t)(t >> 7) * (K_TILE / 2) + oct * (LBO_K / 2) + (t & 127) * 8;
    split_store8(ph, ph + planes * kp, v);
  } else {
    __half* pv = tiled + 2 * planes * (qp + kp) + bh * v_plane(nt) + (size_t)(t >> 7) * (V_TILE / 2) +
                 ((t & 127) >> 3) * (LBO_V / 2) + (t & 7);
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      __half hi, lo;
      split_f16(v[d], hi, lo);
      pv[(oct * 8 + d) * 8] = hi;
      pv[(72 + oct * 8 + d) * 8] = lo;
    }
    if (oct == 0) pv[64 * 8] = __float2half_rn(t < N ? 1.0f : 0.0f);
    if (oct == 1) {
#pragma unroll
      for (int z = 65; z < 72; ++z) pv[z * 8] = __float2half_rn(0.f);
    }
  }
}

namespace vfa {
// layout policy of attn::softmax_attention over the planes of vit_qkv_tile_kernel
struct Layout {
  static constexpr int NWG = 2, NKV = 2, REGS_PRODUCER = 40, REGS_CONSUMER = 232, HD = vfa::HD, NH = vfa::NH, O_REGS = 36;
  static constexpr uint32_t K_TILE = vfa::K_TILE, V_TILE = vfa::V_TILE, Q_BLOCK = 2 * Q_TILE;
  static constexpr uint32_t OFF_K = 0, OFF_V = OFF_K + NKV * 2 * K_TILE, OFF_Q = OFF_V + NKV * V_TILE,
                            OFF_BAR = OFF_Q + NWG * Q_BLOCK, SMEM = OFF_BAR + 8 + 32 * NKV;
  static constexpr int THREADS = 128 * (NWG + 1);
  static constexpr bool SPLIT = false;   // grid (query tiles, heads, images), every CTA over all keys

  const __half* qbase;   // this (image, head) in the Q hi, K hi and V^T planes
  const __half* kbase;
  const __half* vbase;
  size_t planes, qp, kp;   // (image, head) pairs per plane, halves of one pair in a Q and a K plane
  int img, n, N;
  bool cls_last;

  using QOperand = uint32_t;   // the warpgroup's Q block in shared memory
  static __device__ __forceinline__ QOperand q_operand(uint32_t q) { return q; }
  // S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi over the 64 head dims (the small products first), issued and committed
  static __device__ __forceinline__ void issue_scores(float (&S)[64], uint32_t q, uint32_t kt) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      mma_ss<128>(S, make_desc(q + Q_TILE + 2 * i * LBO_Q, LBO_Q, 128), make_desc(kt + 2 * i * LBO_K, LBO_K, 128),
                  i > 0 ? 1u : 0u);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      mma_ss<128>(S, make_desc(q + 2 * i * LBO_Q, LBO_Q, 128), make_desc(kt + K_TILE + 2 * i * LBO_K, LBO_K, 128), 1u);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      mma_ss<128>(S, make_desc(q + 2 * i * LBO_Q, LBO_Q, 128), make_desc(kt + 2 * i * LBO_K, LBO_K, 128), 1u);
    wg_commit();
  }
  // O columns [P V_hi (64) | sum of P (1) | 0 (7)] + [P V_lo (64)] on the first 64
  static __device__ __forceinline__ void issue_pv(float (&O)[36], const uint32_t (&ph)[8][4], uint32_t vt) {
#pragma unroll
    for (int i = 0; i < 8; ++i) mma_rs_n72(O, ph[i], make_desc(vt + 2 * i * LBO_V, LBO_V, 128), i > 0 ? 1u : 0u);
#pragma unroll
    for (int i = 0; i < 8; ++i) mma_rs_n64(O, ph[i], make_desc(vt + 2 * i * LBO_V + V_LO, LBO_V, 128), 1u);
    wg_commit();
  }
  // running output and normaliser of the thread's two rows <- tile (O, corr)
  static __device__ __forceinline__ void fold_tile(float (&o)[2][16], float (&l)[2], const float (&O)[36], const float (&corr)[2],
                                                   int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int b = 0; b < 8; ++b)
#pragma unroll
        for (int e = 0; e < 2; ++e) o[h][2 * b + e] = fmaf(o[h][2 * b + e], corr[h], O[4 * b + 2 * h + e]);
      const float lt = __shfl_sync(0xffffffffu, O[32 + 2 * h], lane & ~3);   // column 64 sits in the quad's first thread
      l[h] = fmaf(l[h], corr[h], lt);
    }
  }
  static __device__ __forceinline__ int q_blocks(int N, int nt) { return (N + 63) / 64; }
  // 64-row Q block b: hi, lo (8 KB each)
  __device__ __forceinline__ void load_q(uint32_t dst, int b, uint32_t bar) const {
    for (int p = 0; p < 2; ++p) bulk_load(dst + p * Q_TILE, qbase + p * planes * qp + (size_t)b * (Q_TILE / 2), Q_TILE, bar);
  }
  __device__ __forceinline__ const __half* k_tile(int t, int p) const { return kbase + p * planes * kp + (size_t)t * (K_TILE / 2); }
  __device__ __forceinline__ const __half* v_tile(int t) const { return vbase + (size_t)t * (V_TILE / 2); }
  __device__ __forceinline__ size_t row(int t) const { return token_row(img, t, n, N, cls_last); }
};
}  // namespace vfa

// grid (query tiles of 128, heads, images).  out: fp32 rows (row stride ldo) and / or out2: fp16 hi|lo rows
// [hi(768) | lo(768)]; rows follow vfa::token_row.
__global__ void __launch_bounds__(vfa::Layout::THREADS, 1)
vit_attention_kernel(const __half* __restrict__ tiled, float* __restrict__ out, int ldo, __half* __restrict__ out2, int n,
                     int N, int nt, bool cls_last) {
  using namespace vfa;
  const int head = blockIdx.y, img = blockIdx.z;
  const size_t bh = (size_t)img * NH + head, planes = (size_t)n * NH;
  const size_t qp = q_plane(2 * nt), kp = k_plane(nt);
  const Layout lay{tiled + bh * qp, tiled + 2 * planes * qp + bh * kp, tiled + 2 * planes * (qp + kp) + bh * v_plane(nt),
                   planes, qp, kp, img, n, N, cls_last};
  attn::softmax_attention(lay, out, ldo, out2, N, nt);
}

}  // namespace mvsf
