// Softmax attention of the DINOv2 ViT-B blocks (models/dino/layers/attention.py:77-101: 12 heads of 64, non-causal,
// scale head_dim ** -0.5 = 1/8) on wgmma.  Included by vit.cu.
//
// Same structure as the stage-1 kernel (attention_fa.cuh), re-laid out for head dim 64.  One CTA works on 128 query
// rows of one (image, head):
//   warpgroup 2    bulk-copy producer (one thread): the two 64-row Q blocks, then K and V^T tiles of 128 keys
//                  (pre-tiled by vit_qkv_tile_kernel into the canonical K-major layouts) through two mbarrier rings of
//                  NKV = 2 stages
//   warpgroups 0-1 64 query rows each.  Per 128-key tile: S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi (three m64n128 products
//                  per 16 head dims, fp32 scores in registers), online softmax (a row lives in the 4 threads of a quad),
//                  P rounded to fp16 IN REGISTERS and used directly as the A operand of P*V: P against the V^T tile's
//                  rows [V_hi (64) | 1 | 0 (7)] (N = 72; the ones row makes the tensor core produce the softmax
//                  normaliser from the same rounded P), then P against the V_lo rows (N = 64) into the same
//                  accumulator.  The tile is folded into the running output with round-to-nearest adds.
// Schedule (after FlashAttention-3, as attention_fa.cuh): each warpgroup issues the scores of tile j+1 and P*V of tile j
// back to back; the softmax of tile j+1 runs while P*V of tile j is in flight.
// Shared memory: a stage holds K hi + lo (32 KB) and the V^T tile (34 KB), so two stages and two consumer warpgroups
// (164 KB with the Q blocks) fit one SM; a third stage would not.  Per thread the loop keeps 64 scores, 36 P*V
// accumulators, 32 running outputs and 32 packed P registers: the producer gives its registers to the consumers
// (setmaxnreg 40 / 232).  At hd 64 a key tile costs 64 exponentials per row against 6 x 128 x 64 + 2 x 136 x 128
// multiply-adds, so unlike the hd-16 kernel the loop is bound by the tensor core, not the exp unit.
#pragma once
#include "linear_tc.cuh"
#include "wgmma.cuh"

namespace mvsf {
namespace vfa {
using namespace gmma;
constexpr int NH = 12, HD = 64, NKV = 2, NWG = 2, THREADS = 128 * (NWG + 1);
constexpr uint32_t LBO_K = 2048, LBO_Q = 1024;          // k-chunk (8 head dims) strides: K 128 rows, Q block 64 rows
constexpr uint32_t K_TILE = 8 * LBO_K;                   // 16 KB: one 128-key x 64-dim fp16 tile (hi or lo)
constexpr uint32_t Q_TILE = 8 * LBO_Q;                   // 8 KB: one 64-query block (hi or lo)
constexpr int VROWS = 136;                               // V^T rows: V_hi dims 0-63 | ones | 7 zero rows | V_lo dims 0-63
constexpr uint32_t LBO_V = VROWS * 16, V_TILE = 16 * LBO_V, V_LO = 9 * 128;   // 16 key chunks; V_lo starts at row 72
// K ring (hi, lo) | V ring | per warpgroup: Q hi, Q lo | barriers
constexpr uint32_t OFF_K = 0, OFF_V = OFF_K + NKV * 2 * K_TILE, OFF_Q = OFF_V + NKV * V_TILE,
                   OFF_BAR = OFF_Q + NWG * 2 * Q_TILE, SMEM = OFF_BAR + 8 + 32 * NKV;
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
      const __half hi = __float2half_rn(v[d]);
      pv[(oct * 8 + d) * 8] = hi;
      pv[(72 + oct * 8 + d) * 8] = __float2half_rn(v[d] - __half2float(hi));
    }
    if (oct == 0) pv[64 * 8] = __float2half_rn(t < N ? 1.0f : 0.0f);
    if (oct == 1) {
#pragma unroll
      for (int z = 65; z < 72; ++z) pv[z * 8] = __float2half_rn(0.f);
    }
  }
}

namespace vfa {
// S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi over the 64 head dims (the small products first), issued and committed
__device__ __forceinline__ void issue_scores(float (&S)[64], uint32_t q, uint32_t kt) {
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
__device__ __forceinline__ void issue_pv(float (&O)[36], const uint32_t (&ph)[8][4], uint32_t vt) {
#pragma unroll
  for (int i = 0; i < 8; ++i) mma_rs_n72(O, ph[i], make_desc(vt + 2 * i * LBO_V, LBO_V, 128), i > 0 ? 1u : 0u);
#pragma unroll
  for (int i = 0; i < 8; ++i) mma_rs_n64(O, ph[i], make_desc(vt + 2 * i * LBO_V + V_LO, LBO_V, 128), 1u);
  wg_commit();
}
// online softmax of score tile j, in place: S becomes 2^(S - m + 14) for the updated running maxima m of the thread's two
// rows, corr = 2^(m_old - m).  The 2^14 bias keeps probabilities down to 4e-12 representable in fp16 (see
// attention_fa.cuh); it cancels in O / l.
__device__ __forceinline__ void softmax_tile(float (&S)[64], float (&m)[2], float (&corr)[2], int j, int N, int q) {
  if (j * 128 + 128 > N) {                 // last, partial tile only: keys >= N never win the max and get P = 0
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (j * 128 + 8 * (i >> 2) + 2 * q + (i & 1) >= N) S[i] = -1e30f;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float pmax = -1e30f;
#pragma unroll
    for (int b = 0; b < 16; ++b) pmax = fmaxf(pmax, fmaxf(S[4 * b + 2 * h], S[4 * b + 2 * h + 1]));
    pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, 1));
    pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, 2));
    const float mx = fmaxf(m[h], pmax);
    corr[h] = ex2f(m[h] - mx);
    m[h] = mx;
  }
  const float mb[2] = {m[0] - 14.0f, m[1] - 14.0f};
#pragma unroll
  for (int i = 0; i < 64; ++i) S[i] = ex2f(S[i] - mb[(i >> 1) & 1]);
}
// P as the A operand of the P*V products: k-step i (keys 16 i .. 16 i + 15) = registers 8 i .. 8 i + 7 of S
__device__ __forceinline__ void pack_p(const float (&S)[64], uint32_t (&ph)[8][4]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int r = 0; r < 4; ++r) ph[i][r] = pack_half2(S[8 * i + 2 * r], S[8 * i + 2 * r + 1]);
}
// running output and normaliser of the thread's two rows <- tile (O, corr)
__device__ __forceinline__ void fold_tile(float (&o)[2][16], float (&l)[2], const float (&O)[36], const float (&corr)[2],
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
}  // namespace vfa

// grid (query tiles of 128, heads, images).  out: fp32 rows (row stride ldo) and / or out2: fp16 hi|lo rows
// [hi(768) | lo(768)]; rows follow vfa::token_row.
__global__ void __launch_bounds__(vfa::THREADS, 1)
vit_attention_kernel(const __half* __restrict__ tiled, float* __restrict__ out, int ldo, __half* __restrict__ out2, int n,
                     int N, int nt, bool cls_last) {
  using namespace vfa;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = blockIdx.y, img = blockIdx.z;
  const size_t bh = (size_t)img * NH + head, planes = (size_t)n * NH;
  const size_t qp = q_plane(2 * nt), kp = k_plane(nt);
  const __half* qbase = tiled + bh * qp;
  const __half* kbase = tiled + 2 * planes * qp + bh * kp;
  const __half* vbase = tiled + 2 * planes * (qp + kp) + bh * v_plane(nt);
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar_q = sb + OFF_BAR, bar_kf = bar_q + 8, bar_ke = bar_kf + 8 * NKV, bar_vf = bar_ke + 8 * NKV,
                 bar_ve = bar_vf + 8 * NKV;
  if (tid == 0) {
    mbar_init(bar_q, 1);
    for (int i = 0; i < NKV; ++i) { mbar_init(bar_kf + 8 * i, 1); mbar_init(bar_ke + 8 * i, NWG); mbar_init(bar_vf + 8 * i, 1); mbar_init(bar_ve + 8 * i, NWG); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 4 * NWG) {
    // ------------------------------------------------------------------------------------------ producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 4 * NWG && lane == 0) {
      // Q block 2 blockIdx.x + w for warpgroup w (hi, lo: 8 KB each).  A block past the last one has only rows >= N,
      // which are computed and not stored: it reads the last block instead.
      const int nqb = (N + 63) / 64;
      expect_tx(bar_q, NWG * 2 * Q_TILE);
      for (int w = 0; w < NWG; ++w) {
        const int qb = min(NWG * (int)blockIdx.x + w, nqb - 1);
        for (int p = 0; p < 2; ++p)
          bulk_load(sb + OFF_Q + (2 * w + p) * Q_TILE, qbase + p * planes * qp + (size_t)qb * (Q_TILE / 2), Q_TILE, bar_q);
      }
      for (int t = 0; t < nt; ++t) {
        const int s = t % NKV;
        const uint32_t par = (uint32_t)(((t / NKV) & 1) ^ 1);
        mbar_wait(bar_ke + 8 * s, par);
        expect_tx(bar_kf + 8 * s, 2 * K_TILE);
        bulk_load(sb + OFF_K + (2 * s) * K_TILE, kbase + (size_t)t * (K_TILE / 2), K_TILE, bar_kf + 8 * s);
        bulk_load(sb + OFF_K + (2 * s + 1) * K_TILE, kbase + planes * kp + (size_t)t * (K_TILE / 2), K_TILE, bar_kf + 8 * s);
        mbar_wait(bar_ve + 8 * s, par);
        expect_tx(bar_vf + 8 * s, V_TILE);
        bulk_load(sb + OFF_V + s * V_TILE, vbase + (size_t)t * (V_TILE / 2), V_TILE, bar_vf + 8 * s);
      }
    }
    return;
  }
  // -------------------------------------------------------------------------------------------- MMA + softmax warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // thread (warpgroup wg, warp wq of it, lane): query rows 64 (2 blockIdx.x + wg) + 16 wq + lane / 4 + 8 h (h = 0, 1);
  // score / output columns 8 b + 2 (lane % 4) + e of accumulator register 4 b + 2 h + e
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  const bool leader = (tid & 127) == 0;
  const uint32_t qs = sb + OFF_Q + wg * 2 * Q_TILE;
  float o[2][16];
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int d = 0; d < 16; ++d) o[h][d] = 0.f;
  float S[64], O[36], corr[2];
  uint32_t ph[8][4];
  mbar_wait(bar_q, 0u);
  mbar_wait(bar_kf, 0u);
  wg_fence();
  issue_scores(S, qs, sb + OFF_K);             // scores of tile 0
  wg_wait<0>();
  fence_regs<64>(S);
  if (leader) mbar_arrive(bar_ke);
  softmax_tile(S, m, corr, 0, N, q);
  pack_p(S, ph);
  if (nt > 1) {                                // operands of iteration 0
    mbar_wait(bar_kf + 8, 0u);
    mbar_wait(bar_vf, 0u);
  }
  // iteration j: scores of tile j + 1 and P*V of tile j; the softmax of tile j + 1 overlaps P*V of tile j
  for (int j = 0; j + 1 < nt; ++j) {
    const int s = j % NKV, s1 = (j + 1) % NKV, s2 = (j + 2) % NKV;
    wg_fence();
    issue_scores(S, qs, sb + OFF_K + (2 * s1) * K_TILE);
    issue_pv(O, ph, sb + OFF_V + s * V_TILE);
    wg_wait<1>();                              // the scores (the older group) are complete, P*V may still run
    fence_regs<64>(S);
    if (leader) mbar_arrive(bar_ke + 8 * s1);
    float corr1[2];
    softmax_tile(S, m, corr1, j + 1, N, q);
    if (j + 2 < nt) mbar_wait(bar_kf + 8 * s2, (uint32_t)(((j + 2) / NKV) & 1));
    mbar_wait(bar_vf + 8 * s1, (uint32_t)(((j + 1) / NKV) & 1));
    wg_wait<0>();
    fence_regs<36>(O);
    if (leader) mbar_arrive(bar_ve + 8 * s);
    fold_tile(o, l, O, corr, lane);
    pack_p(S, ph);
    corr[0] = corr1[0];
    corr[1] = corr1[1];
  }
  {                                            // P*V of the last tile
    const int j = nt - 1, s = j % NKV;
    mbar_wait(bar_vf + 8 * s, (uint32_t)((j / NKV) & 1));
    wg_fence();
    issue_pv(O, ph, sb + OFF_V + s * V_TILE);
    wg_wait<0>();
    fence_regs<36>(O);
    fold_tile(o, l, O, corr, lane);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = 64 * (NWG * (int)blockIdx.x + wg) + 16 * wq + (lane >> 2) + 8 * h;
    if (t >= N) continue;
    const size_t r = token_row(img, t, n, N, cls_last);
    const float inv = __fdiv_rn(1.0f, l[h]);
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const int col = head * HD + 8 * b + 2 * q;
      const float r0 = o[h][2 * b] * inv, r1 = o[h][2 * b + 1] * inv;
      if (out) *reinterpret_cast<float2*>(out + r * ldo + col) = make_float2(r0, r1);
      if (out2) split_store2(out2 + r * (2 * NH * HD) + col, out2 + r * (2 * NH * HD) + NH * HD + col, r0, r1);
    }
  }
}

}  // namespace mvsf
