// Softmax attention on wgmma: the one kernel body of the stage-1 regulariser's attention (attention_fa.cuh, head dim 16)
// and of the ViT's (vit_attention.cuh, head dim 64).  A layout policy L supplies what differs between them: head dim,
// warpgroup and stage counts, register split, tile sizes, the Q / K / V source addresses, the products and the output
// row map.
//
// One CTA works on L::NWG x 64 query rows (grid x) of one head (grid y), over all keys, or (L::SPLIT) on the query
// group, head and key-tile range the layout gives it:
//   warpgroup NWG   bulk-copy producer (one thread): the CTA's Q blocks, then K (hi, lo) and V^T tiles of 128 keys,
//                   pre-tiled into the canonical K-major layouts, through two mbarrier rings of L::NKV stages
//   warpgroups 0..NWG-1   64 query rows each.  Per 128-key tile: S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi (fp32 scores in
//                   registers), online softmax (a row lives in the 4 threads of a quad), P rounded to fp16 IN REGISTERS
//                   and used directly as the A operand of the P*V products against V^T tiles that carry a ones row: the
//                   tensor core produces the softmax normaliser of the tile from the same rounded P.  The tile's partial
//                   products are added (round to nearest) while folding the tile into the running output.
// Schedule (after FlashAttention-3): each warpgroup issues the scores of tile j+1 and P*V of tile j back to back; the
// softmax of tile j+1 runs once the scores are complete (wgmma.wait_group 1) while P*V of tile j is still in flight, and
// tile j is folded into the output after it.  Measured on the stage-1 kernel, H100 SXM at 700 W (N = 27 648, two
// warpgroups): 1.51-1.55 ms per launch against 1.72-1.73 ms for a loop that waits for each product before its softmax.
// Variants measured slower on the same kind of card and dropped: a named-barrier ping-pong that alternates the two
// warpgroups' MMA issue (+4 %), and computing 1/8 or 1/4 of the exponentials with a polynomial on the FMA pipe as
// FlashAttention-4 does (+3 % and +9 % on top of the ping-pong loop).
// P is fp16 only (11 bits; the SAME rounded P feeds the numerator and the normaliser, so the rounding is an unbiased 2^-12
// relative perturbation of the softmax weights).  Scores keep all three products: a one-product variant has 20x the error,
// 5.2e-3 vs fp64, and a stage-2 cascade probability error of 1.5e-4.
//
// Policy L:
//   NWG, NKV                         consumer warpgroups, ring stages
//   REGS_PRODUCER, REGS_CONSUMER     setmaxnreg of the producer and the consumer warpgroups
//   HD, NH                           head dim (running output: HD / 4 registers per row), heads of an output row
//   O_REGS                           P*V accumulator registers
//   K_TILE, V_TILE, Q_BLOCK          bytes of one K tile (hi or lo), one V^T tile and one warpgroup's Q block (hi + lo)
//   OFF_K, OFF_V, OFF_Q, OFF_BAR     shared memory: K ring (hi, lo per stage) | V^T ring | per consumer warpgroup its Q
//                                    block at OFF_Q + wg * Q_BLOCK (hi, then lo at + Q_BLOCK / 2) | mbarriers
//   QOperand, q_operand(q)           the Q operand of issue_scores, made once from the warpgroup's Q block at q
//   issue_scores(S, q, k), issue_pv(O, P, v), fold_tile(o, l, O, corr, lane)   the products and the fold of one tile
//   load_q(dst, b, bar), q_blocks(N, ntiles)   bulk copies of 64-row Q block b, the number of Q blocks (a block past
//                                    the last one has only rows >= N, which are computed and not stored: it reads the
//                                    last one instead)
//   k_tile(t, p), v_tile(t)          global source of K tile t (p = 0 hi, 1 lo) and V^T tile t
//   row(t)                           output row of query t
//   SPLIT                            false: grid (query group, head), all key tiles.  true: members head, group (query
//                                    group of L::NWG x 64 rows), key tiles [t0, t1) and part: null, or the CTA's
//                                    partial slot, which gets per row the unnormalised output (HD), m and l instead
//                                    of the output rows
#pragma once
#include <cuda_fp16.h>

#include "wgmma.cuh"

namespace mvsf {
namespace attn {
using namespace gmma;

// online softmax of score tile j, in place: S becomes 2^(S - m + 14) for the updated running maxima m of the thread's two
// rows, corr = 2^(m_old - m)
__device__ __forceinline__ void softmax_tile(float (&S)[64], float (&m)[2], float (&corr)[2], int j, int N, int q) {
  if (j * 128 + 128 > N) {                 // last, partial tile only: keys >= N never win the max and get P = 0
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (j * 128 + 8 * (i >> 2) + 2 * q + (i & 1) >= N) S[i] = -1e30f;
  }
  float mb[2];
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
    // P is stored as fp16: scale it by 2^14 (largest element 16384 < 65504) so that probabilities down to 4e-12 survive
    // - without the bias every p < 3e-8 underflows to zero, a SYSTEMATIC loss of up to N * 3e-8 in the normaliser for
    // peaked rows.  The factor cancels in O / l.
    mb[h] = mx - 14.0f;
  }
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

// the CTA's head and query group (of L::NWG x 64 rows)
template <class L>
__device__ __forceinline__ int item_head(const L& lay) {
  if constexpr (L::SPLIT) return lay.head; else return blockIdx.y;
}
template <class L>
__device__ __forceinline__ int item_group(const L& lay) {
  if constexpr (L::SPLIT) return lay.group; else return blockIdx.x;
}

// out: fp32 rows (row stride ldo) and / or out2: fp16 hi|lo rows [hi(NH HD) | lo(NH HD)], rows from lay.row
template <class L>
__device__ __forceinline__ void softmax_attention(const L& lay, float* __restrict__ out, int ldo, __half* __restrict__ out2,
                                                  int N, int ntiles) {
  constexpr int NWG = L::NWG, NKV = L::NKV;
  static_assert(128 * (L::REGS_PRODUCER + NWG * L::REGS_CONSUMER) <= 65536, "setmaxnreg exceeds the register file");
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = item_head(lay);
  int t0 = 0, nt = ntiles;                 // key tiles t0 .. t0 + nt - 1
  float* part = nullptr;
  if constexpr (L::SPLIT) {
    t0 = lay.t0; nt = lay.t1 - lay.t0; part = lay.part;
  }
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar_q = sb + L::OFF_BAR, bar_kf = bar_q + 8, bar_ke = bar_kf + 8 * NKV, bar_vf = bar_ke + 8 * NKV,
                 bar_ve = bar_vf + 8 * NKV;
  if (tid == 0) {
    mbar_init(bar_q, 1);
    // a K / V stage is free once every warpgroup's products that read it are complete (K and V are released at different
    // points of the loop, each by one thread per warpgroup)
    for (int i = 0; i < NKV; ++i) { mbar_init(bar_kf + 8 * i, 1); mbar_init(bar_ke + 8 * i, NWG); mbar_init(bar_vf + 8 * i, 1); mbar_init(bar_ve + 8 * i, NWG); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 4 * NWG) {
    // ------------------------------------------------------------------------------------------ producer
    // the CTA starts every thread with an equal share of the register file, fewer than the consumers' loop needs: the
    // producer warpgroup hands its registers to them
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(L::REGS_PRODUCER));
    if (warp == 4 * NWG && lane == 0) {
      const int nqb = L::q_blocks(N, ntiles);
      expect_tx(bar_q, NWG * L::Q_BLOCK);
      for (int w = 0; w < NWG; ++w) lay.load_q(sb + L::OFF_Q + w * L::Q_BLOCK, min(NWG * item_group(lay) + w, nqb - 1), bar_q);
      for (int t = 0; t < nt; ++t) {
        const int s = t % NKV;
        const uint32_t par = (uint32_t)(((t / NKV) & 1) ^ 1);
        mbar_wait(bar_ke + 8 * s, par);
        expect_tx(bar_kf + 8 * s, 2 * L::K_TILE);
        bulk_load(sb + L::OFF_K + (2 * s) * L::K_TILE, lay.k_tile(t0 + t, 0), L::K_TILE, bar_kf + 8 * s);
        bulk_load(sb + L::OFF_K + (2 * s + 1) * L::K_TILE, lay.k_tile(t0 + t, 1), L::K_TILE, bar_kf + 8 * s);
        mbar_wait(bar_ve + 8 * s, par);
        expect_tx(bar_vf + 8 * s, L::V_TILE);
        bulk_load(sb + L::OFF_V + s * L::V_TILE, lay.v_tile(t0 + t), L::V_TILE, bar_vf + 8 * s);
      }
    }
    return;
  }
  // -------------------------------------------------------------------------------------------- MMA + softmax warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(L::REGS_CONSUMER));
  // thread (warpgroup wg, warp wq of it, lane): query rows 64 (NWG group + wg) + 16 wq + lane / 4 + 8 h (h = 0, 1);
  // score / output columns 8 b + 2 (lane % 4) + e of accumulator register 4 b + 2 h + e
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  const bool leader = (tid & 127) == 0;
  const typename L::QOperand qs = L::q_operand(sb + L::OFF_Q + wg * L::Q_BLOCK);
  float o[2][L::HD / 4];   // per row: head dims 8 b + 2 q + e at 2 b + e
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int d = 0; d < L::HD / 4; ++d) o[h][d] = 0.f;
  float S[64], O[L::O_REGS], corr[2];
  uint32_t ph[8][4];
  mbar_wait(bar_q, 0u);
  mbar_wait(bar_kf, 0u);
  wg_fence();
  L::issue_scores(S, qs, sb + L::OFF_K);       // scores of tile 0
  wg_wait<0>();
  fence_regs<64>(S);
  if (leader) mbar_arrive(bar_ke);
  softmax_tile(S, m, corr, t0, N, q);
  pack_p(S, ph);
  if (nt > 1) {                                // operands of iteration 0
    mbar_wait(bar_kf + 8, 0u);
    mbar_wait(bar_vf, 0u);
  }
  // iteration j: scores of tile j + 1 and P*V of tile j; the softmax of tile j + 1 overlaps P*V of tile j
  for (int j = 0; j + 1 < nt; ++j) {
    const int s = j % NKV, s1 = (j + 1) % NKV, s2 = (j + 2) % NKV;
    wg_fence();
    L::issue_scores(S, qs, sb + L::OFF_K + (2 * s1) * L::K_TILE);
    L::issue_pv(O, ph, sb + L::OFF_V + s * L::V_TILE);
    wg_wait<1>();                              // the scores (the older group) are complete, P*V may still run
    fence_regs<64>(S);
    if (leader) mbar_arrive(bar_ke + 8 * s1);
    float corr1[2];
    softmax_tile(S, m, corr1, t0 + j + 1, N, q);
    // operands of the next iteration.  Waiting for them here, between the softmax and the wait for P*V, also keeps ptxas
    // from hoisting that wait above the softmax: it does not move it across the polling loop.
    if (j + 2 < nt) mbar_wait(bar_kf + 8 * s2, (uint32_t)(((j + 2) / NKV) & 1));
    mbar_wait(bar_vf + 8 * s1, (uint32_t)(((j + 1) / NKV) & 1));
    wg_wait<0>();
    fence_regs<L::O_REGS>(O);
    if (leader) mbar_arrive(bar_ve + 8 * s);
    L::fold_tile(o, l, O, corr, lane);
    pack_p(S, ph);
    corr[0] = corr1[0];
    corr[1] = corr1[1];
  }
  {                                            // P*V of the last tile
    const int j = nt - 1, s = j % NKV;
    mbar_wait(bar_vf + 8 * s, (uint32_t)((j / NKV) & 1));
    wg_fence();
    L::issue_pv(O, ph, sb + L::OFF_V + s * L::V_TILE);
    wg_wait<0>();
    fence_regs<L::O_REGS>(O);
    L::fold_tile(o, l, O, corr, lane);
  }
  if constexpr (L::SPLIT) {
    if (part) {                                // a key range of the item: its partial, rows >= N included
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* pr = part + (size_t)(64 * wg + 16 * wq + (lane >> 2) + 8 * h) * (L::HD + 2);
#pragma unroll
        for (int b = 0; b < L::HD / 8; ++b)
          *reinterpret_cast<float2*>(pr + 8 * b + 2 * q) = make_float2(o[h][2 * b], o[h][2 * b + 1]);
        if (q == 0) *reinterpret_cast<float2*>(pr + L::HD) = make_float2(m[h], l[h]);
      }
      return;
    }
  }
  constexpr int W = L::NH * L::HD;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = 64 * (NWG * item_group(lay) + wg) + 16 * wq + (lane >> 2) + 8 * h;
    if (t >= N) continue;
    const size_t r = lay.row(t);
    const float inv = __fdiv_rn(1.0f, l[h]);
#pragma unroll
    for (int b = 0; b < L::HD / 8; ++b) {
      const int col = head * L::HD + 8 * b + 2 * q;
      const float r0 = o[h][2 * b] * inv, r1 = o[h][2 * b + 1] * inv;
      if (out) *reinterpret_cast<float2*>(out + r * ldo + col) = make_float2(r0, r1);
      if (out2) split_store2(out2 + r * (2 * W) + col, out2 + r * (2 * W) + W + col, r0, r1);
    }
  }
}

}  // namespace attn
}  // namespace mvsf
