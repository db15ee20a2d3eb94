// Softmax attention of the stage-1 transformer regulariser (models/module.py:507-600 -> attention.py:141-170) on wgmma:
// the layout policy of softmax_attention.cuh for 4 heads of 16.  Included by costreg_tr.cu.
//
// One CTA works on NWG x 64 query rows of one head (192 with the shipped three warpgroups).  The producer streams K / V^T
// tiles (pre-tiled by qkv_tile_kernel, 4 KB and 10 KB) through two mbarrier rings of 3 stages.  Per 128-key tile: S =
// three m64n128k16 products; P*V against [V_lo | V_hi | 1 | 0] (N = 40): the V_lo and V_hi column halves are added while
// folding the tile.
// The exp unit (MUFU.EX2, 64 per row and key tile) bounds the loop.  While a warpgroup waits for its scores or reduces
// its row maxima it feeds no exps, so three warpgroups (three softmax warps per SM sub-partition instead of two) keep the
// unit busier; each row still sees the same products in the same order, so the results are bit-identical to two.  A
// 416-thread CTA (three warpgroups + one producer warp) would cap every thread at 128 registers (four of its warps share
// one sub-partition's 16 384), below the loop's ~150: the producer is a whole warpgroup that gives its registers away
// (setmaxnreg 32 / 160).  On an H100 SXM at a 400 W limit: 1.63-1.73 ms per launch at N = 27 648 (two warpgroups
// 1.83-1.92), 2.44-2.48 ms at N = 32 640 (2.59-2.64).
// One CTA per SM runs in waves, and time follows the waves, not the work: on an H100 SXM (132 SMs, 700 W) N = 27 648
// (576 items: 4 full waves + 48) takes 1.33x the time of N = 25 344 (528: exactly 4 waves) for 1.19x the work.  So the
// items of a partial last wave are split over key ranges (fa::split_plan) that run on the otherwise idle SMs, and
// attention_merge_kernel merges their partials: DTU 48 items x 2 parts, T&T (680 items) 20 x 6.  Same card, merge
// included: 1.23-1.26 ms per call at N = 27 648 (1.37-1.39 without the split), 1.67-1.69 ms at N = 32 640 (1.91-1.96).
#pragma once
#include <cuda_fp16.h>

#include <algorithm>

#include "linear_tc.cuh"
#include "softmax_attention.cuh"
#include "wgmma.cuh"

namespace mvsf {

// tiled layout: planes Qh, Ql, Kh, Kl of 4 heads x ntiles x 2048 halves (tile = [2 k-chunks][128 rows][8]) and one V plane
// of 4 heads x ntiles x 5120 halves: V^T tile = [16 k-chunks of 8 keys][40 rows][8 keys] with rows 0-15 = dims of V_lo,
// 16-31 = dims of V_hi, row 32 = ones (its product with P is the softmax normaliser of the tile), rows 33-39 = zero.
// Rows / keys >= N of Q, K, V are zero.
__global__ void qkv_tile_kernel(const float* __restrict__ qkv, __half* __restrict__ tiled, int N, int ntiles, float qscale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (token, which, head, octet of 8 dims)
  const int total = ntiles * 128 * 3 * 4 * 2;
  if (i >= total) return;
  const int oct = i & 1, h = (i >> 1) & 3, which = (i >> 3) % 3, tok = i / 24;
  const size_t plane = (size_t)4 * ntiles * 2048;
  const int tile = tok >> 7, r = tok & 127;
  float v[8];
  if (tok < N) {
    const float4 a = ldg4(qkv + (size_t)tok * 192 + which * 64 + h * 16 + oct * 8);
    const float4 b = ldg4(qkv + (size_t)tok * 192 + which * 64 + h * 16 + oct * 8 + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    if (which == 0) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= qscale;
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  }
  if (which < 2) {
    __half* ph = tiled + (size_t)(which * 2) * plane + ((size_t)h * ntiles + tile) * 2048;
    __half* pl = ph + plane;
    split_store8(ph + oct * 1024 + r * 8, pl + oct * 1024 + r * 8, v);
  } else {
    __half* pv = tiled + (size_t)4 * plane + ((size_t)h * ntiles + tile) * 5120;
    const int kc = r >> 3, e = r & 7;
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      __half hi, lo;
      split_f16(v[d], hi, lo);
      pv[kc * 320 + (oct * 8 + d) * 8 + e] = lo;
      pv[kc * 320 + (16 + oct * 8 + d) * 8 + e] = hi;
    }
    if (oct == 0) {
      pv[kc * 320 + 32 * 8 + e] = __float2half_rn(1.0f);
    } else {
#pragma unroll
      for (int z = 33; z < 40; ++z) pv[kc * 320 + z * 8 + e] = __float2half_rn(0.f);
    }
  }
}

namespace fa {
using namespace gmma;
// layout policy of attn::softmax_attention over the planes of qkv_tile_kernel
template <int NWG_>
struct Layout {
  static constexpr int NWG = NWG_, NKV = 3, REGS_PRODUCER = 32, REGS_CONSUMER = 160, HD = 16, NH = 4, O_REGS = 20;
  // k-chunk strides: K 128 rows; the Q block of one warpgroup 64 rows; V^T 40 rows = V_lo dims | V_hi dims | ones row + 7 zero rows
  static constexpr uint32_t LBO_QK = 2048, LBO_Q = 1024, LBO_V = 640;
  // one canonical 128 x 16 K tile (hi or lo); the Q block of a warpgroup (hi, lo: 64 rows each); the V^T tile (10 KB)
  static constexpr uint32_t K_TILE = 4096, Q_BLOCK = 4096, V_TILE = 16 * LBO_V;
  static constexpr uint32_t OFF_K = 0, OFF_V = OFF_K + NKV * 2 * K_TILE, OFF_Q = OFF_V + NKV * V_TILE,
                            OFF_BAR = OFF_Q + NWG * Q_BLOCK, SMEM = OFF_BAR + 8 + 32 * NKV;
  static constexpr int THREADS = 128 * (NWG + 1);   // NWG consumer warpgroups + the producer warpgroup
  // an item is one head's group of ROWS query rows; the partial of a key range of it: per row o (HD), m, l
  static constexpr bool SPLIT = true;
  static constexpr int ROWS = 64 * NWG, PART_FLOATS = ROWS * (HD + 2);

  const __half* tiled;
  const __half* base;         // this head in the Q and K planes: + plane index * plane + tile * 2048
  size_t plane, head_tiles;   // head_tiles = head * ntiles
  int head, group, t0, t1;    // the CTA's item and key tiles [t0, t1)
  float* part;                // null for a whole item, else the partial slot of the key range

  // descriptors of the warpgroup's Q block at q (hi, lo)
  struct QOperand { uint64_t hi, lo; };
  static __device__ __forceinline__ QOperand q_operand(uint32_t q) {
    return {make_desc(q, LBO_Q, 128), make_desc(q + Q_BLOCK / 2, LBO_Q, 128)};
  }
  // S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi of the K tile at kt (issued and committed, not waited for)
  static __device__ __forceinline__ void issue_scores(float (&S)[64], const QOperand& q, uint32_t kt) {
    const uint64_t k_hi = make_desc(kt, LBO_QK, 128), k_lo = make_desc(kt + K_TILE, LBO_QK, 128);
    mma_ss<128>(S, q.lo, k_hi, 0u);
    mma_ss<128>(S, q.hi, k_lo, 1u);
    mma_ss<128>(S, q.hi, k_hi, 1u);
    wg_commit();
  }
  // O columns: [P V_lo (16) | P V_hi (16) | sum of P (1) | 0 (7)]
  static __device__ __forceinline__ void issue_pv(float (&O)[20], const uint32_t (&ph)[8][4], uint32_t vt) {
#pragma unroll
    for (int i = 0; i < 8; ++i) mma_rs_n40(O, ph[i], make_desc(vt + 2 * i * LBO_V, LBO_V, 128), i > 0 ? 1u : 0u);
    wg_commit();
  }
  // running output and normaliser of the thread's two rows <- tile (O, corr)
  static __device__ __forceinline__ void fold_tile(float (&o)[2][4], float (&l)[2], const float (&O)[20], const float (&corr)[2],
                                                   int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int e = 0; e < 2; ++e) o[h][2 * b + e] = fmaf(o[h][2 * b + e], corr[h], O[4 * b + 2 * h + e] + O[4 * (b + 2) + 2 * h + e]);
      const float lt = __shfl_sync(0xffffffffu, O[16 + 2 * h], lane & ~3);   // column 32 sits in the quad's first thread
      l[h] = fmaf(l[h], corr[h], lt);
    }
  }
  static __device__ __forceinline__ int q_blocks(int N, int ntiles) { return 2 * ntiles; }
  // 64-row Q block b = half b & 1 of 128-row tile b >> 1, as four 1 KB copies (hi, lo x two k-chunks)
  __device__ __forceinline__ void load_q(uint32_t dst, int b, uint32_t bar) const {
    for (int p = 0; p < 2; ++p)
      for (int kc = 0; kc < 2; ++kc)
        bulk_load(dst + p * (Q_BLOCK / 2) + kc * LBO_Q, base + p * plane + (size_t)(b >> 1) * 2048 + kc * 1024 + (b & 1) * 512,
                  LBO_Q, bar);
  }
  __device__ __forceinline__ const __half* k_tile(int t, int p) const { return base + (2 + p) * plane + (size_t)t * 2048; }
  __device__ __forceinline__ const __half* v_tile(int t) const { return tiled + 4 * plane + (head_tiles + t) * (V_TILE / 2); }
  __device__ __forceinline__ size_t row(int t) const { return (size_t)t; }
};
}  // namespace fa

namespace fa {
// bytes of the tiled planes per 128-key tile: Q hi, Q lo, K hi, K lo (4 heads x 2048 halves each) and V^T (4 x 5120)
constexpr size_t TILE_BYTES = (4 * 4 * 2048 + 4 * 5120) * sizeof(__half);
// shortest key range worth a CTA of its own: a split item costs a second launch (a few us) and every part refills the
// K / V ring, while a key tile takes ~1.3 us (H100 SXM, 700 W)
constexpr int MIN_PART_TILES = 16;

// How one attention call covers the SMs.  The 4 ceil(N / ROWS) items of ntiles key tiles run one CTA per SM; when the
// last wave is partial, its `split` items (the last ones) are each cut into `parts` contiguous key ranges whose lengths
// differ by at most one tile, so that the wave runs on up to `sms` SMs instead of `split`.  The parts' partials take
// the workspace beyond the tiled planes (`region_bytes` in all).  split = 0, parts = 1: every item runs whole.
struct SplitPlan { int items, split, parts; };
template <int NWG>
inline SplitPlan split_plan(int N, int sms, size_t region_bytes) {
  using A = Layout<NWG>;
  const int ntiles = (N + 127) / 128, items = 4 * ((N + A::ROWS - 1) / A::ROWS), r = items % sms;
  const size_t planes = (size_t)ntiles * TILE_BYTES;
  const size_t slots = region_bytes > planes ? (region_bytes - planes) / (A::PART_FLOATS * sizeof(float)) : 0;
  const int k = r ? (int)std::min({(size_t)(sms / r), slots / r, (size_t)(ntiles / MIN_PART_TILES)}) : 0;
  return k >= 2 ? SplitPlan{items, r, k} : SplitPlan{items, 0, 1};
}
}  // namespace fa

// out: fp32 rows [N][64] and / or out2: fp16 hi|lo rows [N][hi(64) | lo(64)].  NWG (3 shipped) is in the kernel's name.
// 1-D grid of fa::split_plan: the whole items first, then the `parts` key ranges of each of the last `split` items (the
// block scheduler starts the short ranges last), which write their partials to `partials` for attention_merge_kernel.
template <int NWG>
__global__ void __launch_bounds__(fa::Layout<NWG>::THREADS, 1)
attention_fa_kernel(const __half* __restrict__ tiled, float* __restrict__ out, __half* __restrict__ out2, int N, int ntiles,
                    int split, int parts, float* __restrict__ partials) {
  using A = fa::Layout<NWG>;
  const int groups = (N + A::ROWS - 1) / A::ROWS, whole = 4 * groups - split;
  int item = blockIdx.x, t0 = 0, t1 = ntiles;
  float* part = nullptr;
  if (item >= whole) {
    const int b = item - whole, p = b % parts;
    item = whole + b / parts;
    t0 = p * ntiles / parts;
    t1 = (p + 1) * ntiles / parts;
    part = partials + (size_t)b * A::PART_FLOATS;
  }
  const int head = item / groups;
  const size_t head_tiles = (size_t)head * ntiles;
  const A lay{tiled, tiled + head_tiles * 2048, (size_t)4 * ntiles * 2048, head_tiles, head, item % groups, t0, t1, part};
  attn::softmax_attention(lay, out, 64, out2, N, ntiles);
}

// The outputs of the split items: per row, the `parts` partials (o, m, l) merged in part order, m* = max m, o and l
// weighted by 2^(m - m*), then the epilogue of softmax_attention.  One thread per (split item, row); no CTA of the
// attention kernel waits for another.
template <int NWG>
__global__ void attention_merge_kernel(const float* __restrict__ partials, float* __restrict__ out, __half* __restrict__ out2,
                                       int N, int split, int parts) {
  using A = fa::Layout<NWG>;
  constexpr int HD = A::HD, W = A::NH * A::HD, ROWS = A::ROWS;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= split * ROWS) return;
  const int groups = (N + ROWS - 1) / ROWS, s = i / ROWS, rr = i % ROWS, item = 4 * groups - split + s;
  const int head = item / groups, t = (item % groups) * ROWS + rr;
  if (t >= N) return;
  const float* p0 = partials + (size_t)s * parts * A::PART_FLOATS + (size_t)rr * (HD + 2);
  float mx = -1e30f;
  for (int p = 0; p < parts; ++p) mx = fmaxf(mx, p0[(size_t)p * A::PART_FLOATS + HD]);
  float o[HD], l = 0.f;
#pragma unroll
  for (int d = 0; d < HD; ++d) o[d] = 0.f;
  for (int p = 0; p < parts; ++p) {
    const float* pp = p0 + (size_t)p * A::PART_FLOATS;
    const float w = gmma::ex2f(pp[HD] - mx);
    l = fmaf(pp[HD + 1], w, l);
#pragma unroll
    for (int d = 0; d < HD; ++d) o[d] = fmaf(pp[d], w, o[d]);
  }
  const float inv = __fdiv_rn(1.0f, l);
#pragma unroll
  for (int d = 0; d < HD; d += 2) {
    const int col = head * HD + d;
    const float r0 = o[d] * inv, r1 = o[d + 1] * inv;
    if (out) *reinterpret_cast<float2*>(out + (size_t)t * W + col) = make_float2(r0, r1);
    if (out2) split_store2(out2 + (size_t)t * (2 * W) + col, out2 + (size_t)t * (2 * W) + W + col, r0, r1);
  }
}

}  // namespace mvsf
