// Softmax attention of the stage-1 transformer regulariser (models/module.py:507-600 -> attention.py:141-170) on wgmma.
// Included by costreg_tr.cu (uses its split_f16 / ex2f helpers).
//
// One CTA works on NWG x 64 query rows of one head (head dim 16): 192 for the shipped fp16-P kernel, 128 for the hi + lo one.
//   warpgroup NWG   bulk-copy producer (one thread): the CTA's Q blocks, then K / V^T tiles (pre-tiled by qkv_tile_kernel
//                   into the canonical K-major layouts, 4 KB and 10 KB) through two mbarrier rings of NKV stages
//   warpgroups 0..NWG-1   64 query rows each.  Per 128-key tile: S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi (three
//                 m64n128k16 MMAs, fp32 scores in registers), online softmax (a row lives in the 4 threads of a quad), P
//                 rounded to fp16 IN REGISTERS and used directly as the A operand of the P*V MMAs against
//                 [V_lo | V_hi | 1 | 0] (N = 40): the ones row of V makes the tensor core produce the softmax normaliser of
//                 the tile as well.  The tile's partial products are added (round to nearest) while folding the tile into
//                 the running output.
// Schedule (after FlashAttention-3): each warpgroup issues the scores of tile j+1 and P*V of tile j back to back; the
// softmax of tile j+1 runs once the scores are complete (wgmma.wait_group 1) while P*V of tile j is still in flight, and
// tile j is folded into the output after it.  Measured on an H100 SXM at 700 W (N = 27 648, two warpgroups): 1.51-1.55 ms
// per launch against 1.72-1.73 ms for a loop that waits for each product before its softmax.  Variants measured slower on
// the same kind of card and dropped: a named-barrier ping-pong that alternates the two warpgroups' MMA issue (+4 %), and
// computing 1/8 or 1/4 of the exponentials with a polynomial on the FMA pipe as FlashAttention-4 does
// (+3 % and +9 % on top of the ping-pong loop).
// The exp unit (MUFU.EX2, 64 per row and key tile) bounds the loop.  While a warpgroup waits for its scores or reduces
// its row maxima it feeds no exps, so three warpgroups (three softmax warps per SM sub-partition instead of two) keep the
// unit busier; each row still sees the same products in the same order, so the results are bit-identical to two.  A
// 416-thread CTA (three warpgroups + one producer warp) would cap every thread at 128 registers (four of its warps share
// one sub-partition's 16 384), below the loop's ~150: the producer is a whole warpgroup that gives its registers away
// (setmaxnreg 32 / 160).  On an H100 SXM at a 400 W limit: 1.63-1.73 ms per launch at N = 27 648 (two warpgroups
// 1.83-1.92), 2.44-2.48 ms at N = 32 640 (2.59-2.64), though 192-row CTAs leave a coarser last wave (DTU 576 CTAs on 132
// SMs: 5 waves, busiest SM 960 rows against 896 with 128-row CTAs).
#pragma once

namespace fa {
using namespace gmma;
constexpr int NKV = 3;
constexpr uint32_t TILE = 4096;                 // one canonical 128 x 16 (Q, K) fp16 tile
// k-chunk strides: K 128 rows; the Q block of one warpgroup 64 rows; V^T 40 rows = V_lo dims | V_hi dims | ones row + 7 zero rows
constexpr uint32_t LBO_QK = 2048, LBO_Q = 1024, LBO_V = 640;
constexpr uint32_t V_TILE = 16 * LBO_V;         // 10 KB
// K ring (hi, lo) | V ring | per warpgroup: Q hi, Q lo (64 rows each, 4 KB together) | barriers
constexpr uint32_t OFF_K = 0, OFF_V = OFF_K + NKV * 2 * TILE, OFF_Q = OFF_V + NKV * V_TILE;
constexpr int threads(int nwg) { return 128 * (nwg + 1); }   // nwg consumer warpgroups + the producer warpgroup
constexpr uint32_t smem_bytes(int nwg) { return OFF_Q + nwg * TILE + 8 + 32 * NKV; }
}  // namespace fa

// tiled layout: planes Qh, Ql, Kh, Kl of 4 heads x ntiles x 2048 halves (tile = [2 k-chunks][128 rows][8]) and one V plane
// of 4 heads x ntiles x 5120 halves: V^T tile = [16 k-chunks of 8 keys][40 rows][8 keys] with rows 0-15 = dims of V_lo,
// 16-31 = dims of V_hi, row 32 = ones (its product with P is the softmax normaliser of the tile), rows 33-39 = zero.
// P_hi multiplies all 40 rows (N = 40), P_lo rows 16-39 (N = 24: V_hi and the ones row).  Rows / keys >= N of Q, K, V are zero.
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
// S = Q_lo K_hi + Q_hi K_lo + Q_hi K_hi of the K tile at kt (issued and committed, not waited for)
__device__ __forceinline__ void issue_scores(float (&S)[64], uint64_t q_hi, uint64_t q_lo, uint32_t kt) {
  const uint64_t k_hi = make_desc(kt, LBO_QK, 128), k_lo = make_desc(kt + TILE, LBO_QK, 128);
  mma_ss<128>(S, q_lo, k_hi, 0u);
  mma_ss<128>(S, q_hi, k_lo, 1u);
  mma_ss<128>(S, q_hi, k_hi, 1u);
  wg_commit();
}
// O columns: [P V_lo (16) | P V_hi (16) | sum of P (1) | 0 (7)];  P_lo multiplies [V_hi | 1 | 0] onto columns 16..39
template <bool PLO>
__device__ __forceinline__ void issue_pv(float (&O)[20], const uint32_t (&ph)[8][4], const uint32_t (&pl)[8][4], uint32_t vt) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    mma_rs_n40(O, ph[i], make_desc(vt + 2 * i * LBO_V, LBO_V, 128), i > 0 ? 1u : 0u);
    if (PLO) mma_rs_n24(O + 8, pl[i], make_desc(vt + 2 * i * LBO_V + 256, LBO_V, 128), 1u);
  }
  wg_commit();
}
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
    // P is stored as fp16 (hi + lo): scale it by 2^14 (largest element 16384 < 65504) so that probabilities down to 4e-12
    // survive - without the bias every p < 3e-8 underflows to zero, a SYSTEMATIC loss of up to N * 3e-8 in the
    // normaliser for peaked rows.  The factor cancels in O / l.
    mb[h] = mx - 14.0f;
  }
#pragma unroll
  for (int i = 0; i < 64; ++i) S[i] = ex2f(S[i] - mb[(i >> 1) & 1]);
}
// P as the A operand of the P*V MMAs: k-step i (keys 16 i .. 16 i + 15) = registers 8 i .. 8 i + 7 of S
template <bool PLO>
__device__ __forceinline__ void pack_p(const float (&S)[64], uint32_t (&ph)[8][4], uint32_t (&pl)[8][4]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float p0 = S[8 * i + 2 * r], p1 = S[8 * i + 2 * r + 1];
      const __half2 hh = __floats2half2_rn(p0, p1);
      ph[i][r] = *reinterpret_cast<const uint32_t*>(&hh);
      if (PLO) {
        const float2 hf = __half22float2(hh);
        pl[i][r] = pack_half2(p0 - hf.x, p1 - hf.y);
      }
    }
}
// running output and normaliser of the thread's two rows <- tile (O, corr)
__device__ __forceinline__ void fold_tile(float (&o)[2][4], float (&l)[2], const float (&O)[20], const float (&corr)[2], int lane) {
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
}  // namespace fa

// PLO = true : P = P_hi + P_lo (22 mantissa bits), three partial products P_hi V_lo + P_hi V_hi + P_lo V_hi  (round-1 kernel)
// PLO = false: P = P_hi only (fp16, 11 bits; the SAME rounded P feeds the numerator and the normaliser, so the rounding is an
//              unbiased 2^-12 relative perturbation of the softmax weights): half the P*V MMAs, no P_lo shared-memory
//              traffic, no lo-split arithmetic in the softmax threads.  Measured against fp64 in tests/test_gpu_parity.py.
// (Scores keep all three products Q_lo K_hi + Q_hi K_lo + Q_hi K_hi: a one-product variant has 20x the error, 5.2e-3 vs
//  fp64, and a stage-2 cascade probability error of 1.5e-4.)
template <bool PLO, int NWG>
__global__ void __launch_bounds__(fa::threads(NWG), 1)
attention_fa_kernel(const __half* __restrict__ tiled, float* __restrict__ out, __half* __restrict__ out2, int N, int ntiles) {
  using namespace fa;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = blockIdx.y;
  const size_t plane = (size_t)4 * ntiles * 2048;
  const __half* base = tiled + (size_t)head * ntiles * 2048;       // + plane index * plane + tile * 2048
  const uint32_t sb = smem_u32(smem);
  const uint32_t bar_q = sb + OFF_Q + NWG * TILE, bar_kf = bar_q + 8, bar_ke = bar_kf + 8 * NKV, bar_vf = bar_ke + 8 * NKV,
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
    // 512 threads start with 128 registers each, fewer than the consumers' loop needs: the producer warpgroup hands
    // its registers to them (32 + 3 x 160 = 512 per thread slot)
    if constexpr (NWG == 3) asm volatile("setmaxnreg.dec.sync.aligned.u32 32;");
    if (warp == 4 * NWG && lane == 0) {
      // Q: 64-row block NWG * blockIdx.x + w of the 128-row tiles for warpgroup w, as four 1 KB copies (hi, lo x two
      // k-chunks).  A block past the last tile has only rows >= N, which are computed and not stored: it reads the last
      // block instead, so that no CTA reads past the Q planes.
      expect_tx(bar_q, NWG * TILE);
      for (int w = 0; w < NWG; ++w) {
        const int b = min(NWG * (int)blockIdx.x + w, 2 * ntiles - 1);
        for (int p = 0; p < 2; ++p)
          for (int kc = 0; kc < 2; ++kc)
            bulk_load(sb + OFF_Q + w * TILE + p * (TILE / 2) + kc * LBO_Q,
                      base + p * plane + (size_t)(b >> 1) * 2048 + kc * 1024 + (b & 1) * 512, LBO_Q, bar_q);
      }
      for (int t = 0; t < ntiles; ++t) {
        const int s = t % NKV;
        const uint32_t par = (uint32_t)(((t / NKV) & 1) ^ 1);
        mbar_wait(bar_ke + 8 * s, par);
        expect_tx(bar_kf + 8 * s, 2 * TILE);
        bulk_load(sb + OFF_K + (2 * s) * TILE, base + 2 * plane + (size_t)t * 2048, TILE, bar_kf + 8 * s);
        bulk_load(sb + OFF_K + (2 * s + 1) * TILE, base + 3 * plane + (size_t)t * 2048, TILE, bar_kf + 8 * s);
        mbar_wait(bar_ve + 8 * s, par);
        expect_tx(bar_vf + 8 * s, V_TILE);
        bulk_load(sb + OFF_V + s * V_TILE, tiled + 4 * plane + ((size_t)head * ntiles + t) * (V_TILE / 2), V_TILE, bar_vf + 8 * s);
      }
    }
    return;
  }
  // -------------------------------------------------------------------------------------------- MMA + softmax warpgroups
  if constexpr (NWG == 3) asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");
  // thread (warpgroup wg, warp wq of it, lane): query rows 64 (NWG blockIdx.x + wg) + 16 wq + lane / 4 + 8 h (h = 0, 1);
  // score columns 8 b + 2 (lane % 4) + e of accumulator register 4 b + 2 h + e
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  const bool leader = (tid & 127) == 0;
  const uint64_t q_hi = make_desc(sb + OFF_Q + wg * TILE, LBO_Q, 128), q_lo = make_desc(sb + OFF_Q + wg * TILE + TILE / 2, LBO_Q, 128);
  float o[2][4];   // per row: head dims 2q, 2q + 1, 8 + 2q, 9 + 2q
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int d = 0; d < 4; ++d) o[h][d] = 0.f;
  float S[64], O[20], corr[2];
  uint32_t ph[8][4], pl[8][4];
  mbar_wait(bar_q, 0u);
  mbar_wait(bar_kf, 0u);
  wg_fence();
  issue_scores(S, q_hi, q_lo, sb + OFF_K);     // scores of tile 0
  wg_wait<0>();
  fence_regs<64>(S);
  if (leader) mbar_arrive(bar_ke);
  softmax_tile(S, m, corr, 0, N, q);
  pack_p<PLO>(S, ph, pl);
  if (ntiles > 1) {                            // operands of iteration 0
    mbar_wait(bar_kf + 8, 0u);
    mbar_wait(bar_vf, 0u);
  }
  // iteration j: scores of tile j + 1 and P*V of tile j; the softmax of tile j + 1 overlaps P*V of tile j
  for (int j = 0; j + 1 < ntiles; ++j) {
    const int s = j % NKV, s1 = (j + 1) % NKV, s2 = (j + 2) % NKV;
    wg_fence();
    issue_scores(S, q_hi, q_lo, sb + OFF_K + (2 * s1) * TILE);
    issue_pv<PLO>(O, ph, pl, sb + OFF_V + s * V_TILE);
    wg_wait<1>();                              // the scores (the older group) are complete, P*V may still run
    fence_regs<64>(S);
    if (leader) mbar_arrive(bar_ke + 8 * s1);
    float corr1[2];
    softmax_tile(S, m, corr1, j + 1, N, q);
    // operands of the next iteration.  Waiting for them here, between the softmax and the wait for P*V, also keeps ptxas
    // from hoisting that wait above the softmax: it does not move it across the polling loop.
    if (j + 2 < ntiles) mbar_wait(bar_kf + 8 * s2, (uint32_t)(((j + 2) / NKV) & 1));
    mbar_wait(bar_vf + 8 * s1, (uint32_t)(((j + 1) / NKV) & 1));
    wg_wait<0>();
    fence_regs<20>(O);
    if (leader) mbar_arrive(bar_ve + 8 * s);
    fold_tile(o, l, O, corr, lane);
    pack_p<PLO>(S, ph, pl);
    corr[0] = corr1[0];
    corr[1] = corr1[1];
  }
  {                                            // P*V of the last tile
    const int j = ntiles - 1, s = j % NKV;
    mbar_wait(bar_vf + 8 * s, (uint32_t)((j / NKV) & 1));
    wg_fence();
    issue_pv<PLO>(O, ph, pl, sb + OFF_V + s * V_TILE);
    wg_wait<0>();
    fence_regs<20>(O);
    fold_tile(o, l, O, corr, lane);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = 64 * (NWG * (int)blockIdx.x + wg) + 16 * wq + (lane >> 2) + 8 * h;
    if (r >= N) continue;
    const float inv = __fdiv_rn(1.0f, l[h]);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int col = head * 16 + 8 * b + 2 * q;
      const float r0 = o[h][2 * b] * inv, r1 = o[h][2 * b + 1] * inv;
      if (out) *reinterpret_cast<float2*>(out + (size_t)r * 64 + col) = make_float2(r0, r1);
      if (out2) split_store2(out2 + (size_t)r * 128 + col, out2 + (size_t)r * 128 + 64 + col, r0, r1);
    }
  }
}
