// Token-wise linear layers on the Hopper tensor cores:  C[M,N] = epi(A[M,K] * W[N,K]^T), fp32-class accuracy.
//   * operands are split into fp16 hi + lo parts (hi+lo carries 22 mantissa bits); three wgmma.m64nNk16 products per
//     K-step (lo*hi, hi*lo, hi*hi) accumulate in fp32 registers - a single-pass fp16/bf16/tf32 GEMM would move the
//     depth probabilities by ~1e-3 (SURVEY.md 7.3), the split stays at ~1e-6 relative;
//   * tile = 128 rows x all N columns (N <= 256); persistent CTAs (one per SM) keep the weights resident in shared memory
//     and stream A in K-blocks of 64 through a 4-stage cp.async ring in the canonical no-swizzle K-major layout
//     (wgmma.cuh); mbarriers full[s] / empty[s] hand the stages between the producer warpgroup and the two MMA warpgroups;
//   * each MMA warpgroup owns 64 rows of the tile and runs its epilogue from the accumulator registers: bias / GELU /
//     ELU+1 / residual element-wise, LayerNorm with the row reduced over the four threads that share it; optionally also
//     emits the fp16 hi|lo split of the result for the next GEMM.  While the MMA warpgroups run an epilogue the producer
//     is already filling the ring with the next tile's K-blocks.
// Used by the stage-1 transformer regulariser (module.py:507-646) and FMT (FMT.py, block.py:336-346).
#include "linear_tc.cuh"

#include <utility>

#include "wgmma.cuh"

namespace mvsf {

using namespace gmma;

constexpr int TC_BM = 128, TC_BK = 64;

// 384 threads: warpgroup 0 = producers (cp.async fills of the A ring), warpgroups 1 and 2 = MMA + epilogue of rows
// [0, 64) and [64, 128) of every tile.  The weight tiles of all K-blocks stay resident in shared memory for the CTA's
// lifetime.  Each MMA warpgroup keeps one K-block of MMAs in flight while it issues the next, and releases a ring stage
// as soon as the MMAs that read it have retired.
constexpr int TC_NPROD = 128, TC_THREADS = 384;
constexpr int TC_RING = 4;   // A-tile stages; two fills stay in flight behind the block whose MMAs are being issued

// element-wise epilogue of the two adjacent columns (col, col + 1) of one row, shared by the resident and streamed GEMMs
template <int EPI>
__device__ __forceinline__ void epi_pair(const TcLinArgs& a, int col, const float* resrow, bool mvalid, float (&t)[2]) {
  const float2 b2 = a.bias ? *reinterpret_cast<const float2*>(a.bias + col) : make_float2(0.f, 0.f);
  t[0] += b2.x; t[1] += b2.y;
  if (EPI == LIN_RES) {
    const float2 g2 = *reinterpret_cast<const float2*>(a.gamma + col);
    const float2 r2 = mvalid ? *reinterpret_cast<const float2*>(resrow + col) : make_float2(0.f, 0.f);
    t[0] = r2.x + g2.x * t[0]; t[1] = r2.y + g2.y * t[1];
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (EPI == LIN_GELU) t[e] = gelu_erf_lean(t[e]);
    if (EPI == LIN_ELU1) t[e] = (col + e < a.elu_cols) ? ((t[e] > 0.f ? t[e] : expm1f(t[e])) + 1.0f) : t[e];
    if (EPI == LIN_SILU) t[e] = __fdiv_rn(t[e], 1.0f + expf(-t[e]));
  }
}
// fp32 and / or fp16 hi|lo stores of the pair; the lo part of the split row sits lo_off halves after the hi part
__device__ __forceinline__ void epi_store2(float* crow, __half* c2row, int lo_off, int col, const float (&t)[2]) {
  if (crow) *reinterpret_cast<float2*>(crow + col) = make_float2(t[0], t[1]);
  if (c2row) split_store2(c2row + col, c2row + lo_off + col, t[0], t[1]);
}

// LayerNorm of a 64-wide row whose values sit in the accumulator layout: 16 per thread (columns 8b + 2q + e, b < 8,
// e < 2, q = lane & 3), the row spread over the 4 threads of a quad.  Shared by every LayerNorm epilogue, so the fused
// token MLP and the single GEMMs round alike.
__device__ __forceinline__ void ln64_stats(const float (&x)[16], float eps, float& mean, float& sd) {
  float s = 0.f;
#pragma unroll
  for (int b = 0; b < 8; ++b) s += x[2 * b] + x[2 * b + 1];
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  mean = s * (1.0f / 64.0f);
  float v = 0.f;
#pragma unroll
  for (int e = 0; e < 16; ++e) { const float d = x[e] - mean; v = fmaf(d, d, v); }
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  sd = sqrtf(v * (1.0f / 64.0f) + eps);
}
__device__ __forceinline__ float ln64_apply(float x, float mean, float sd, const float* w, const float* b, int col) {
  return __fdiv_rn(x - mean, sd) * __ldg(w + col) + __ldg(b + col);
}

template <int N, int EPI>
__device__ __forceinline__ void tc_epilogue(const TcLinArgs& a, const float (&acc)[N / 2], int row0, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = row0 + 8 * h;
    const bool mvalid = m < a.M;
    const float* resrow = (EPI == LIN_RES || EPI == LIN_RES_LN) ? a.res + (size_t)(mvalid ? m : 0) * a.ldres : nullptr;
    float* crow = a.C ? a.C + (size_t)(mvalid ? m : 0) * a.ldc : nullptr;
    __half* c2row = a.C2 ? a.C2 + (size_t)(mvalid ? m : 0) * a.ldc2 : nullptr;
    if constexpr (EPI == LIN_RES_LN || EPI == LIN_LN) {   // N == 64: a row is spread over the 4 threads of a quad
      float x[16];
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        const int col = 8 * b + 2 * q;
        const float2 b2 = a.bias ? *reinterpret_cast<const float2*>(a.bias + col) : make_float2(0.f, 0.f);
        float t0 = acc[4 * b + 2 * h] + b2.x, t1 = acc[4 * b + 2 * h + 1] + b2.y;
        if (EPI == LIN_RES_LN) {
          const float2 g2 = *reinterpret_cast<const float2*>(a.gamma + col);
          const float2 r2 = mvalid ? *reinterpret_cast<const float2*>(resrow + col) : make_float2(0.f, 0.f);
          t0 = r2.x + g2.x * t0; t1 = r2.y + g2.y * t1;
        }
        x[2 * b] = t0; x[2 * b + 1] = t1;
      }
      if (a.Cpre && mvalid) {
        float* prow = a.Cpre + (size_t)m * a.ldcpre;
#pragma unroll
        for (int b = 0; b < 8; ++b) *reinterpret_cast<float2*>(prow + 8 * b + 2 * q) = make_float2(x[2 * b], x[2 * b + 1]);
      }
      float mean, sd;
      ln64_stats(x, a.ln_eps, mean, sd);
      if (mvalid) {
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int col = 8 * b + 2 * q;
          const float o0 = ln64_apply(x[2 * b], mean, sd, a.ln_w, a.ln_b, col);
          const float o1 = ln64_apply(x[2 * b + 1], mean, sd, a.ln_w, a.ln_b, col + 1);
          if (crow) *reinterpret_cast<float2*>(crow + col) = make_float2(o0, o1);
          if (c2row) split_store2(c2row + col, c2row + N + col, o0, o1);
        }
      }
    } else {
#pragma unroll
      for (int b = 0; b < N / 8; ++b) {
        const int col = 8 * b + 2 * q;
        float t[2] = {acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]};
        epi_pair<EPI>(a, col, resrow, mvalid, t);
        if (mvalid) epi_store2(crow, c2row, N, col, t);
      }
    }
  }
}

template <int N, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
linear_tc_kernel(TcLinArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const int K = a.K;
  const int nkb = K / TC_BK;
  constexpr uint32_t a_bytes = tile_bytes(TC_BM), b_bytes = tile_bytes(N);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sB = sbase;                                   // [nkb][hi tile | lo tile]
  const uint32_t sA = sB + nkb * 2 * b_bytes;                  // ring [TC_RING][hi tile | lo tile]
  const uint32_t bar_full = sA + TC_RING * 2 * a_bytes, bar_empty = bar_full + 8 * TC_RING;

  if (tid == 0) {
    for (int i = 0; i < TC_RING; ++i) { mbar_init(bar_full + 8 * i, TC_NPROD); mbar_init(bar_empty + 8 * i, 2); }
    fence_barrier_init();
  }
  // resident weights: all K-blocks, hi and lo
  for (int kb = 0; kb < nkb; ++kb) {
    fill_tile<TC_THREADS>(sB + (2 * kb) * b_bytes, a.Bh + kb * TC_BK, a.ldb, N, N, tid);
    fill_tile<TC_THREADS>(sB + (2 * kb + 1) * b_bytes, a.Bl + kb * TC_BK, a.ldb, N, N, tid);
  }
  cp_async_commit_group();
  cp_async_wait_group<0>();
  fence_proxy_async();
  __syncthreads();

  const int ntiles = (a.M + TC_BM - 1) / TC_BM;
  const int my_tiles = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  constexpr uint32_t lbo_a = tile_lbo(TC_BM), lbo_b = tile_lbo(N);

  if (wg == 0) {
    // ------------------------------------------------------------------ producers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // registers go to the accumulators of the MMA warpgroups
    // Blocks g = 0, 1, ... enumerate the (tile, kb) pairs of this CTA in order; block g uses ring stage g % TC_RING.  The
    // copies of blocks g, g-1 are still in flight when block g-2 is handed to the MMA warpgroups (two cp.async groups of
    // prefetch keep the L2 / HBM latency of the 32 KB blocks hidden).
    const int nblk = my_tiles * nkb;
    auto publish = [&](int gb) {   // this thread's copies of block gb have landed: make them visible to the async proxy
      fence_proxy_async();
      mbar_arrive(bar_full + 8 * (gb % TC_RING));
    };
    int g = 0;
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int m0 = ((int)blockIdx.x + t_it * (int)gridDim.x) * TC_BM;
      const int valid_rows = min(TC_BM, a.M - m0);
      for (int kb = 0; kb < nkb; ++kb, ++g) {
        const int st = g % TC_RING;
        mbar_wait(bar_empty + 8 * st, (uint32_t)((((g / TC_RING) & 1)) ^ 1));  // stage free (first use passes)
        const uint32_t s0 = sA + st * 2 * a_bytes;
        fill_tile<TC_NPROD>(s0, a.Ah + (size_t)m0 * a.lda + kb * TC_BK, a.lda, TC_BM, valid_rows, tid);
        fill_tile<TC_NPROD>(s0 + a_bytes, a.Al + (size_t)m0 * a.lda + kb * TC_BK, a.lda, TC_BM, valid_rows, tid);
        cp_async_commit_group();
        if (g >= 2) {
          cp_async_wait_group<2>();
          publish(g - 2);
        }
      }
    }
    if (nblk >= 2) {
      cp_async_wait_group<1>();
      publish(nblk - 2);
    }
    if (nblk >= 1) {
      cp_async_wait_group<0>();
      publish(nblk - 1);
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int half = wg - 1;                     // rows [64 half, 64 half + 64) of every tile
    const int t128 = tid & 127, lane = tid & 31;
    const int row_in_tile = 64 * half + 16 * (t128 >> 5) + (lane >> 2);
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    auto release = [&](int gb) { if (t128 == 0) mbar_arrive(bar_empty + 8 * (gb % TC_RING)); };
    int g = 0;
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int m0 = ((int)blockIdx.x + t_it * (int)gridDim.x) * TC_BM;
      int pend = -1;
      for (int kb = 0; kb < nkb; ++kb, ++g) {
        const int st = g % TC_RING;
        mbar_wait(bar_full + 8 * st, (uint32_t)((g / TC_RING) & 1));
        const uint32_t sa = sA + st * 2 * a_bytes + (uint32_t)half * 1024u;   // 8 row groups of 128 B
        const uint32_t sb = sB + kb * 2 * b_bytes;
        wg_fence();
#pragma unroll
        for (int i = 0; i < TC_BK / 16; ++i) {
          const uint64_t ah = make_desc(sa + 2 * i * lbo_a, lbo_a, 128);
          const uint64_t al = make_desc(sa + a_bytes + 2 * i * lbo_a, lbo_a, 128);
          const uint64_t bh = make_desc(sb + 2 * i * lbo_b, lbo_b, 128);
          const uint64_t bl = make_desc(sb + b_bytes + 2 * i * lbo_b, lbo_b, 128);
          mma_ss<N>(acc, al, bh, (kb > 0 || i > 0) ? 1u : 0u);
          mma_ss<N>(acc, ah, bl, 1u);
          mma_ss<N>(acc, ah, bh, 1u);
        }
        wg_commit();
        if (pend >= 0) {
          wg_wait<1>();
          release(pend);
        }
        pend = g;
      }
      wg_wait<0>();
      fence_regs<N / 2>(acc);
      release(pend);
      tc_epilogue<N, EPI>(a, acc, m0 + row_in_tile, lane);
    }
  }
}

static size_t tc_smem_bytes(int N, int K) {
  return (size_t)(K / TC_BK) * 2 * tile_bytes(N) + (size_t)TC_RING * 2 * tile_bytes(TC_BM) + 128;
}

template <int N, int EPI>
static int launch_tc(const TcLinArgs& a, size_t smem, int grid, cudaStream_t s) {
  static DeviceOnce once;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(linear_tc_kernel<N, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.done(dev);
  }
  linear_tc_kernel<N, EPI><<<grid, TC_THREADS, smem, s>>>(a);
  MVSF_LAUNCH_CHECK("linear_tc");
  return MVSF_OK;
}

// The (N, epilogue) pairs linear_tc_kernel is built for, and the only ones launch_linear_tc accepts: those the transformer
// regulariser (costreg_tr.cu) and FMT (fmt.cu) run, and the single GEMMs the fused token MLP is compared against bit for bit
// (tests/test_gpu_token_mlp.py).
struct TcPair { int n, epi; };
constexpr TcPair kTcPairs[] = {
    {64, LIN_LN}, {192, LIN_BIAS}, {256, LIN_BIAS},      // transformer regulariser
    {192, LIN_ELU1}, {64, LIN_ELU1}, {128, LIN_ELU1},    // FMT
    {64, LIN_RES_LN}, {256, LIN_GELU}, {64, LIN_RES}};   // token MLP reference
constexpr size_t kNumTcPairs = sizeof(kTcPairs) / sizeof(kTcPairs[0]);

static bool tc_pair_built(int n, int epi) {
  for (const TcPair& p : kTcPairs)
    if (p.n == n && p.epi == epi) return true;
  return false;
}

template <size_t... I>
static int launch_tc_pair(const TcLinArgs& a, int epi, size_t smem, int grid, cudaStream_t s, std::index_sequence<I...>) {
  int rc = MVSF_ERR_INVALID;   // not reached: check_linear_tc admits built pairs only
  ((a.N == kTcPairs[I].n && epi == kTcPairs[I].epi &&
    (rc = launch_tc<kTcPairs[I].n, kTcPairs[I].epi>(a, smem, grid, s), true)) || ...);
  return rc;
}

// host-side argument checks of launch_linear_tc; touch no device state, so callers can run them before any launch
static int check_linear_tc(const TcLinArgs& a, int epi) {
  MVSF_REQUIRE(epi >= LIN_BIAS && epi <= LIN_LN, "linear_tc: unknown epilogue %d", epi);
  MVSF_REQUIRE(a.Ah && a.Al && a.Bh && a.Bl && (a.C || a.C2) && a.M > 0, "linear_tc: bad arguments");
  MVSF_REQUIRE(a.K % TC_BK == 0 && a.K >= TC_BK, "linear_tc: need K %% 64 == 0");
  MVSF_REQUIRE((a.lda % 8) == 0 && (a.ldb % 8) == 0 && ((uintptr_t)a.Ah & 15) == 0 && ((uintptr_t)a.Al & 15) == 0 &&
                   ((uintptr_t)a.Bh & 15) == 0 && ((uintptr_t)a.Bl & 15) == 0, "linear_tc: operands must be 16-byte aligned");
  if (a.C) MVSF_REQUIRE((a.ldc % 4) == 0 && ((uintptr_t)a.C & 15) == 0, "linear_tc: C must be 16-byte aligned");
  if (a.C2) MVSF_REQUIRE((a.ldc2 % 8) == 0 && ((uintptr_t)a.C2 & 15) == 0, "linear_tc: C2 must be 16-byte aligned");
  if (epi == LIN_RES_LN || epi == LIN_LN) MVSF_REQUIRE(a.N == 64 && a.ln_w && a.ln_b, "linear_tc: LayerNorm epilogue needs N == 64");
  if (epi == LIN_RES || epi == LIN_RES_LN)
    MVSF_REQUIRE(a.res && a.gamma && ((uintptr_t)a.res & 15) == 0 && ((uintptr_t)a.gamma & 15) == 0 && (a.ldres % 4) == 0,
                 "linear_tc: residual epilogue needs 16-byte aligned res and gamma");
  if (a.bias) MVSF_REQUIRE(((uintptr_t)a.bias & 15) == 0, "linear_tc: bias must be 16-byte aligned");
  if (a.Cpre) MVSF_REQUIRE((epi == LIN_RES_LN || epi == LIN_LN) && (a.ldcpre % 4) == 0 && ((uintptr_t)a.Cpre & 15) == 0,
                           "linear_tc: Cpre needs a LayerNorm epilogue and 16-byte alignment");
  MVSF_REQUIRE(tc_pair_built(a.N, epi), "linear_tc: no kernel for (N = %d, epilogue %d); need N in a built pair (kTcPairs)",
               a.N, epi);
  const size_t smem = tc_smem_bytes(a.N, a.K);
  MVSF_REQUIRE(smem <= 227 * 1024, "linear_tc: N*K too large for resident weights (%zu bytes of shared memory)", smem);
  return MVSF_OK;
}

int launch_linear_tc(const TcLinArgs& a, int epi, cudaStream_t s) {
  int rc;
  if ((rc = check_linear_tc(a, epi))) return rc;
  const size_t smem = tc_smem_bytes(a.N, a.K);
  const int num_sms = device_sm_count(current_device());
  const int ntiles = cdiv(a.M, TC_BM);
  const int grid = ntiles < num_sms ? ntiles : num_sms;  // persistent: one CTA per SM, tiles strided by gridDim.x
  return launch_tc_pair(a, epi, smem, grid, s, std::make_index_sequence<kNumTcPairs>{});
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused token MLP (launch_token_mlp, TokenMlpArgs in linear_tc.cuh): proj (64 -> 64) + its epilogue, FFN1 (64 -> 256,
// GELU) and FFN2 (256 -> 64) + its epilogue in one kernel, so neither the LayerNorm split that feeds FFN1 nor the 256-wide
// hidden layer goes through memory.  Same roles as linear_tc_kernel: one CTA per SM, 128-row tiles, a producer warpgroup
// streaming the attention output (the A of proj) through a 2-stage cp.async ring, two MMA warpgroups of 64 rows each.
// All three weight matrices stay resident (hi and lo: 16.3 + 64.3 + 65 KB).  Per warpgroup and tile:
//   proj from shared memory -> epilogue in registers: the residual of FFN2 stays there, the FFN1 input becomes fp16 hi|lo
//   register A fragments (an m64n16 accumulator slice is the A fragment of a k16 step, as the attention feeds P);
//   FFN1 in 4 chunks of 64 hidden columns, each -> bias + GELU -> hi|lo A fragments of FFN2's K-block of that chunk,
//   accumulated into the one N = 64 FFN2 accumulator; chunk c + 1's FFN1 products run during chunk c's GELU.
// Every product is the one the three single GEMMs issue, in the same order (lo*hi, hi*lo, hi*hi per k16 step, FFN2
// K-blocks 0..3 into one accumulator), and every epilogue runs the same arithmetic, so the outputs match those of the
// three launches bit for bit.
constexpr int MLP_RING = 2;
constexpr uint32_t MLP_T64 = tile_bytes(64), MLP_T256 = tile_bytes(256), MLP_TA = tile_bytes(TC_BM);
constexpr uint32_t MLP_OFF_F1 = 2 * MLP_T64, MLP_OFF_F2 = MLP_OFF_F1 + 2 * MLP_T256, MLP_OFF_A = MLP_OFF_F2 + 8 * MLP_T64,
                   MLP_OFF_BAR = MLP_OFF_A + MLP_RING * 2 * MLP_TA, MLP_SMEM = MLP_OFF_BAR + 16 * MLP_RING;
static_assert(MLP_SMEM <= 227 * 1024, "token MLP: resident weights + ring exceed shared memory");

// D (+)= A * B^T over K = 64 with the three split products per k16 step; A = register fragments [k16 step][4],
// B = hi tile at b (lo tile b_lo bytes after it), leading byte offset lbo
__device__ __forceinline__ void mlp_mma_rs(float (&d)[32], const uint32_t (&ah)[4][4], const uint32_t (&al)[4][4], uint32_t b,
                                           uint32_t b_lo, uint32_t lbo, bool accumulate) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint64_t bh = make_desc(b + 2 * i * lbo, lbo, 128), bl = make_desc(b + b_lo + 2 * i * lbo, lbo, 128);
    mma_rs_n64(d, al[i], bh, (accumulate || i > 0) ? 1u : 0u);
    mma_rs_n64(d, ah[i], bl, 1u);
    mma_rs_n64(d, ah[i], bh, 1u);
  }
}

template <int FORM>
__global__ void __launch_bounds__(TC_THREADS, 1)
token_mlp_kernel(TokenMlpArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t sP = smem_u32(smem);     // proj W [64][64]: hi tile | lo tile
  const uint32_t sF1 = sP + MLP_OFF_F1;   // FFN1 W [256][64]: hi tile | lo tile
  const uint32_t sF2 = sP + MLP_OFF_F2;   // FFN2 W [64][256]: 4 K-blocks x (hi tile | lo tile)
  const uint32_t sA = sP + MLP_OFF_A;     // ring [MLP_RING][hi tile | lo tile] of the attention output
  const uint32_t bar_full = sP + MLP_OFF_BAR, bar_empty = bar_full + 8 * MLP_RING;

  if (tid == 0) {
    for (int i = 0; i < MLP_RING; ++i) { mbar_init(bar_full + 8 * i, TC_NPROD); mbar_init(bar_empty + 8 * i, 2); }
    fence_barrier_init();
  }
  fill_tile<TC_THREADS>(sP, a.pw_h, 64, 64, 64, tid);
  fill_tile<TC_THREADS>(sP + MLP_T64, a.pw_l, 64, 64, 64, tid);
  fill_tile<TC_THREADS>(sF1, a.f1w_h, 64, 256, 256, tid);
  fill_tile<TC_THREADS>(sF1 + MLP_T256, a.f1w_l, 64, 256, 256, tid);
  for (int kb = 0; kb < 4; ++kb) {
    fill_tile<TC_THREADS>(sF2 + 2 * kb * MLP_T64, a.f2w_h + kb * TC_BK, 256, 64, 64, tid);
    fill_tile<TC_THREADS>(sF2 + (2 * kb + 1) * MLP_T64, a.f2w_l + kb * TC_BK, 256, 64, 64, tid);
  }
  cp_async_commit_group();
  cp_async_wait_group<0>();
  fence_proxy_async();
  __syncthreads();

  const int ntiles = (a.M + TC_BM - 1) / TC_BM;
  const int my_tiles = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (wg == 0) {
    // ------------------------------------------------------------------ producer: tile t into stage t % MLP_RING
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int m0 = ((int)blockIdx.x + t_it * (int)gridDim.x) * TC_BM, st = t_it % MLP_RING;
      mbar_wait(bar_empty + 8 * st, (uint32_t)(((t_it / MLP_RING) & 1) ^ 1));   // stage free (first use passes)
      const uint32_t s0 = sA + st * 2 * MLP_TA;
      fill_tile<TC_NPROD>(s0, a.A + (size_t)m0 * 128, 128, TC_BM, min(TC_BM, a.M - m0), tid);
      fill_tile<TC_NPROD>(s0 + MLP_TA, a.A + (size_t)m0 * 128 + 64, 128, TC_BM, min(TC_BM, a.M - m0), tid);
      cp_async_commit_group();
      cp_async_wait_group<0>();   // the MMA warpgroups spend a whole tile's MLP on the other stage meanwhile
      fence_proxy_async();
      mbar_arrive(bar_full + 8 * st);
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int half = wg - 1;
    const int t128 = tid & 127, lane = tid & 31, q = lane & 3;
    const int row_in_tile = 64 * half + 16 * (t128 >> 5) + (lane >> 2);
    constexpr uint32_t lbo_a = tile_lbo(TC_BM), lbo64 = tile_lbo(64), lbo256 = tile_lbo(256);
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int m0 = ((int)blockIdx.x + t_it * (int)gridDim.x) * TC_BM, st = t_it % MLP_RING;
      // ---- proj
      float acc[32];
      mbar_wait(bar_full + 8 * st, (uint32_t)((t_it / MLP_RING) & 1));
      const uint32_t sa = sA + st * 2 * MLP_TA + (uint32_t)half * 1024u;
      wg_fence();
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint64_t ah = make_desc(sa + 2 * i * lbo_a, lbo_a, 128), al = make_desc(sa + MLP_TA + 2 * i * lbo_a, lbo_a, 128);
        const uint64_t bh = make_desc(sP + 2 * i * lbo64, lbo64, 128), bl = make_desc(sP + MLP_T64 + 2 * i * lbo64, lbo64, 128);
        mma_ss<64>(acc, al, bh, i > 0 ? 1u : 0u);
        mma_ss<64>(acc, ah, bl, 1u);
        mma_ss<64>(acc, ah, bh, 1u);
      }
      wg_commit();
      wg_wait<0>();
      fence_regs<32>(acc);
      if (t128 == 0) mbar_arrive(bar_empty + 8 * st);
      // ---- proj epilogue: r = FFN2's residual (pre-norm: x + gamma1 proj; post-norm: LN_mid of it), the FFN1 input
      //      (pre-norm: LN_mid(x + gamma1 proj); post-norm: r) as hi|lo A fragments: k16 step b / 2, register 2 (b % 2) + h
      float r[2][16];
      uint32_t xh[4][4], xl[4][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + row_in_tile + 8 * h;
        const bool mvalid = m < a.M;
        const float* resrow = a.res + (size_t)(mvalid ? m : 0) * 64;
        float x[16];
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int col = 8 * b + 2 * q;
          const float2 b2 = *reinterpret_cast<const float2*>(a.proj_b + col);
          const float2 g2 = *reinterpret_cast<const float2*>(a.gamma1 + col);
          const float2 r2 = mvalid ? *reinterpret_cast<const float2*>(resrow + col) : make_float2(0.f, 0.f);
          float t0 = acc[4 * b + 2 * h] + b2.x, t1 = acc[4 * b + 2 * h + 1] + b2.y;
          t0 = r2.x + g2.x * t0; t1 = r2.y + g2.y * t1;
          x[2 * b] = t0; x[2 * b + 1] = t1;
        }
        float mean, sd;
        ln64_stats(x, a.mid_eps, mean, sd);
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int col = 8 * b + 2 * q;
          const float o0 = ln64_apply(x[2 * b], mean, sd, a.mid_w, a.mid_b, col);
          const float o1 = ln64_apply(x[2 * b + 1], mean, sd, a.mid_w, a.mid_b, col + 1);
          r[h][2 * b] = FORM == MLP_POST_NORM ? o0 : x[2 * b];
          r[h][2 * b + 1] = FORM == MLP_POST_NORM ? o1 : x[2 * b + 1];
          split_pack2(o0, o1, xh[b >> 1][2 * (b & 1) + h], xl[b >> 1][2 * (b & 1) + h]);
        }
      }
      // ---- FFN1 chunk c (hidden columns [64c, 64c + 64)) -> GELU -> A fragments of FFN2's K-block c
      float hid[2][32], acc2[32];
      uint32_t gh[4][4], gl[4][4];
      wg_fence();
      mlp_mma_rs(hid[0], xh, xl, sF1, MLP_T256, lbo256, false);
      wg_commit();
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (c + 1 < 4) {
          wg_fence();
          mlp_mma_rs(hid[(c + 1) & 1], xh, xl, sF1 + (c + 1) * 1024u, MLP_T256, lbo256, false);
          wg_commit();
          wg_wait<1>();   // FFN1 chunk c and FFN2 K-block c - 1 (whose A fragments are overwritten next) are done
        } else {
          wg_wait<0>();
        }
        fence_regs<32>(hid[c & 1]);
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const float2 b2 = *reinterpret_cast<const float2*>(a.f1_b + 64 * c + 8 * b + 2 * q);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float t0 = hid[c & 1][4 * b + 2 * h] + b2.x, t1 = hid[c & 1][4 * b + 2 * h + 1] + b2.y;
            t0 = gelu_erf_lean(t0); t1 = gelu_erf_lean(t1);
            split_pack2(t0, t1, gh[b >> 1][2 * (b & 1) + h], gl[b >> 1][2 * (b & 1) + h]);
          }
        }
        wg_fence();
        mlp_mma_rs(acc2, gh, gl, sF2 + 2 * c * MLP_T64, MLP_T64, lbo64, c > 0);
        wg_commit();
      }
      wg_wait<0>();
      fence_regs<32>(acc2);
      // ---- FFN2 epilogue: x = r + gamma2 (ffn + bias) -> C, and C2 = split(LN_out(x)) (post-norm: C = LN_out(x) too)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + row_in_tile + 8 * h;
        const bool mvalid = m < a.M;
        float* crow = a.C + (size_t)(mvalid ? m : 0) * 64;
        __half* c2row = a.C2 ? a.C2 + (size_t)(mvalid ? m : 0) * 128 : nullptr;
        float x[16];
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int col = 8 * b + 2 * q;
          const float2 b2 = *reinterpret_cast<const float2*>(a.f2_b + col);
          const float2 g2 = *reinterpret_cast<const float2*>(a.gamma2 + col);
          float t0 = acc2[4 * b + 2 * h] + b2.x, t1 = acc2[4 * b + 2 * h + 1] + b2.y;
          t0 = r[h][2 * b] + g2.x * t0; t1 = r[h][2 * b + 1] + g2.y * t1;
          x[2 * b] = t0; x[2 * b + 1] = t1;
        }
        if (FORM != MLP_POST_NORM && mvalid) {
#pragma unroll
          for (int b = 0; b < 8; ++b) *reinterpret_cast<float2*>(crow + 8 * b + 2 * q) = make_float2(x[2 * b], x[2 * b + 1]);
        }
        if constexpr (FORM != MLP_PRE_NORM_LAST) {
          float mean, sd;
          ln64_stats(x, a.out_eps, mean, sd);
          if (mvalid) {
#pragma unroll
            for (int b = 0; b < 8; ++b) {
              const int col = 8 * b + 2 * q;
              const float o0 = ln64_apply(x[2 * b], mean, sd, a.out_w, a.out_b, col);
              const float o1 = ln64_apply(x[2 * b + 1], mean, sd, a.out_w, a.out_b, col + 1);
              if (FORM == MLP_POST_NORM) *reinterpret_cast<float2*>(crow + col) = make_float2(o0, o1);
              split_store2(c2row + col, c2row + 64 + col, o0, o1);
            }
          }
        }
      }
    }
  }
}

template <int FORM>
static int launch_mlp(const TokenMlpArgs& a, int grid, cudaStream_t s) {
  static DeviceOnce once;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(token_mlp_kernel<FORM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MLP_SMEM));
    once.done(dev);
  }
  token_mlp_kernel<FORM><<<grid, TC_THREADS, MLP_SMEM, s>>>(a);
  MVSF_LAUNCH_CHECK("token_mlp");
  return MVSF_OK;
}

// host-side argument checks of launch_token_mlp; touch no device state
static int check_token_mlp(const TokenMlpArgs& a, int form) {
  MVSF_REQUIRE(form == MLP_PRE_NORM || form == MLP_PRE_NORM_LAST || form == MLP_POST_NORM, "token_mlp: unknown form %d", form);
  MVSF_REQUIRE(a.M > 0 && a.A && a.res && a.C && a.pw_h && a.pw_l && a.f1w_h && a.f1w_l && a.f2w_h && a.f2w_l && a.proj_b &&
                   a.gamma1 && a.mid_w && a.mid_b && a.f1_b && a.f2_b && a.gamma2,
               "token_mlp: bad arguments");
  if (form != MLP_PRE_NORM_LAST) MVSF_REQUIRE(a.C2 && a.out_w && a.out_b, "token_mlp: the output LayerNorm needs C2, out_w, out_b");
  const void* ptrs16[] = {a.A, a.res, a.C, a.C2, a.pw_h, a.pw_l, a.f1w_h, a.f1w_l, a.f2w_h, a.f2w_l,
                          a.proj_b, a.gamma1, a.f1_b, a.f2_b, a.gamma2};
  for (const void* p : ptrs16) MVSF_REQUIRE(((uintptr_t)p & 15) == 0, "token_mlp: operands must be 16-byte aligned");
  return MVSF_OK;
}

int launch_token_mlp(const TokenMlpArgs& a, int form, cudaStream_t s) {
  int rc;
  if ((rc = check_token_mlp(a, form))) return rc;
  const int ntiles = cdiv(a.M, TC_BM), num_sms = device_sm_count(current_device());
  const int grid = ntiles < num_sms ? ntiles : num_sms;
  switch (form) {
    case MLP_PRE_NORM: return launch_mlp<MLP_PRE_NORM>(a, grid, s);
    case MLP_PRE_NORM_LAST: return launch_mlp<MLP_PRE_NORM_LAST>(a, grid, s);
    default: return launch_mlp<MLP_POST_NORM>(a, grid, s);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Streamed-weight GEMM (launch_linear_tcs, TcsArgs in linear_tc.cuh).  Same split-operand arithmetic and warpgroup
// roles as linear_tc_kernel, but the weights stream too: a ring stage holds the 128-row A block and the BN-row W block of
// one K-block (hi and lo tiles of each), and persistent CTAs walk (M tile, N tile) pairs, N tiles fastest, so CTAs that
// run at the same time share A rows in L2.
//   * BN = 128: a stage is 64.5 KB, three stages fit in shared memory (BN = 256 would allow two, and one stage in flight
//     behind the one being multiplied does not hide the L2 latency of a 96 KB block).  Prefetch depth: stage g + 1 is
//     filled while the MMA warpgroups multiply stage g and stage g - 1 retires.  BN = 64 serves N = 64 (conv head).
//   * Two independent accumulator chains per warpgroup (even and odd K-blocks), added with round-to-nearest in the
//     epilogue: the tensor core's fp32 accumulation truncates, and fc2 (K = 3072) and the 3x3 head conv (K = 6912) would
//     otherwise chain 576 / 1296 products into one accumulator.  2 x 64 accumulator registers at BN = 128.
//   * The producer (56 registers after setmaxnreg; the grid positions of a tile's rows sit in shared memory) resolves
//     every A row through the implicit-GEMM grid with zero fill, so one kernel runs the token linears, the 3x3
//     convolution and the four parity classes of a transposed convolution.
constexpr int TCS_RING = 3;

__device__ __forceinline__ size_t tcs_store_row(const TcsArgs& a, int m) {
  const int hw = a.H * a.W, img = m / hw, rem = m - img * hw, y = rem / a.W, x = rem - y * a.W;
  return ((size_t)img * (a.sy * a.H) + a.sy * y + a.py) * (size_t)(a.sx * a.W) + a.sx * x + a.px;
}

template <int BN>
__device__ __forceinline__ void tcs_mma_block(float* acc, uint32_t sa, uint32_t sb) {
  constexpr uint32_t a_bytes = tile_bytes(TC_BM), b_bytes = tile_bytes(BN), lbo_a = tile_lbo(TC_BM), lbo_b = tile_lbo(BN);
#pragma unroll
  for (int i = 0; i < TC_BK / 16; ++i) {
    const uint64_t ah = make_desc(sa + 2 * i * lbo_a, lbo_a, 128);
    const uint64_t al = make_desc(sa + a_bytes + 2 * i * lbo_a, lbo_a, 128);
    const uint64_t bh = make_desc(sb + 2 * i * lbo_b, lbo_b, 128);
    const uint64_t bl = make_desc(sb + b_bytes + 2 * i * lbo_b, lbo_b, 128);
    mma_ss<BN>(acc, al, bh, 1u);
    mma_ss<BN>(acc, ah, bl, 1u);
    mma_ss<BN>(acc, ah, bh, 1u);
  }
}

template <int BN, int EPI>
__device__ __forceinline__ void tcs_epilogue(const TcsArgs& a, const float (&acc)[BN / 2], int row0, int n0, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = row0 + 8 * h;
    const bool mvalid = m < a.M;
    const size_t p = tcs_store_row(a, mvalid ? m : 0);
    const float* resrow = EPI == LIN_RES ? a.res + p * a.ldres : nullptr;
    float* crow = a.C ? a.C + p * a.ldc : nullptr;
    __half* c2row = a.C2 ? a.C2 + p * a.ldc2 : nullptr;
#pragma unroll
    for (int b = 0; b < BN / 8; ++b) {
      const int col = n0 + 8 * b + 2 * q;
      float t[2] = {acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]};
      epi_pair<EPI>(a, col, resrow, mvalid, t);
      if (mvalid) epi_store2(crow, c2row, a.N, col, t);
    }
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1)
linear_tcs_kernel(TcsArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const int nkb = a.K / TC_BK, kpt = a.cin / TC_BK;
  constexpr uint32_t a_bytes = tile_bytes(TC_BM), b_bytes = tile_bytes(BN), st_bytes = 2 * a_bytes + 2 * b_bytes;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = sbase + TCS_RING * st_bytes, bar_empty = bar_full + 8 * TCS_RING;
  if (tid == 0) {
    for (int i = 0; i < TCS_RING; ++i) { mbar_init(bar_full + 8 * i, TC_NPROD); mbar_init(bar_empty + 8 * i, 2); }
    fence_barrier_init();
  }
  __syncthreads();
  const int ntn = a.N / BN, ntiles = ((a.M + TC_BM - 1) / TC_BM) * ntn;
  const int my_tiles = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (wg == 0) {
    // ------------------------------------------------------------------ producers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    constexpr uint32_t lbo_a = tile_lbo(TC_BM), lbo_b = tile_lbo(BN);
    const int c = tid & 7, r0 = tid >> 3;   // this thread copies 16-byte chunk c of rows r0 + 16 j
    const int hw = a.H * a.W;
    int* syx = reinterpret_cast<int*>(smem + TCS_RING * st_bytes + 16 * TCS_RING);   // [2][128] row grid positions
    auto publish = [&](int gb) {
      fence_proxy_async();
      mbar_arrive(bar_full + 8 * (gb % TCS_RING));
    };
    int g = 0;
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int t = (int)blockIdx.x + t_it * (int)gridDim.x;
      const int m0 = (t / ntn) * TC_BM, n0 = (t % ntn) * BN;
      int* yx = syx + 128 * (t_it & 1);   // (y << 16 | x) of the tile's rows; rows past M get a y no tap reaches
      {
        const int m = m0 + tid, rem = m % hw, y = rem / a.W;
        yx[tid] = m < a.M ? (y << 16) | (rem - y * a.W) : (0x4000 << 16);
      }
      named_bar_sync(1, TC_NPROD);
      for (int kb = 0; kb < nkb; ++kb, ++g) {
        const int st = g % TCS_RING;
        mbar_wait(bar_empty + 8 * st, (uint32_t)(((g / TCS_RING) & 1) ^ 1));
        const uint32_t s0 = sbase + st * st_bytes;
        const int tap = kb / kpt;
        const int nib = (int)((a.taps >> (4 * tap)) & 15ull), dy = (nib & 3) - 1, dx = (nib >> 2) - 1;
        const long long toff = (long long)(dy * a.W + dx) * a.lda + (kb - tap * kpt) * TC_BK + c * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = r0 + 16 * j, p = yx[r], y = (p >> 16) + dy, x = (p & 0xffff) + dx;
          const bool ok = (unsigned)y < (unsigned)a.H && (unsigned)x < (unsigned)a.W;
          const size_t off = ok ? (size_t)((long long)(m0 + r) * a.lda + toff) : 0;
          const uint32_t dst = s0 + c * lbo_a + (r >> 3) * 128 + (r & 7) * 16;
          cp_async16_zfill(dst, a.Ah + off, ok);
          cp_async16_zfill(dst + a_bytes, a.Al + off, ok);
        }
        const size_t boff = (size_t)n0 * a.ldb + kb * TC_BK + c * 8;
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          const int r = r0 + 16 * j;
          const uint32_t dst = s0 + 2 * a_bytes + c * lbo_b + (r >> 3) * 128 + (r & 7) * 16;
          cp_async16_zfill(dst, a.Bh + boff + (size_t)r * a.ldb, true);
          cp_async16_zfill(dst + b_bytes, a.Bl + boff + (size_t)r * a.ldb, true);
        }
        cp_async_commit_group();
        if (g >= 1) {
          cp_async_wait_group<1>();
          publish(g - 1);
        }
      }
    }
    if (g >= 1) {
      cp_async_wait_group<0>();
      publish(g - 1);
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int half = wg - 1;
    const int t128 = tid & 127, lane = tid & 31;
    const int row_in_tile = 64 * half + 16 * (t128 >> 5) + (lane >> 2);
    float acc0[BN / 2], acc1[BN / 2];
    auto release = [&](int gb) { if (t128 == 0) mbar_arrive(bar_empty + 8 * (gb % TCS_RING)); };
    int g = 0;
    for (int t_it = 0; t_it < my_tiles; ++t_it) {
      const int t = (int)blockIdx.x + t_it * (int)gridDim.x;
      const int m0 = (t / ntn) * TC_BM, n0 = (t % ntn) * BN;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
      int pend = -1;
      auto step = [&](float* acc) {   // multiply ring block g into acc, keep it in flight, retire the previous block
        const int st = g % TCS_RING;
        mbar_wait(bar_full + 8 * st, (uint32_t)((g / TCS_RING) & 1));
        const uint32_t sa = sbase + st * st_bytes + (uint32_t)half * 1024u, sb = sbase + st * st_bytes + 2 * a_bytes;
        wg_fence();
        tcs_mma_block<BN>(acc, sa, sb);
        wg_commit();
        if (pend >= 0) {
          wg_wait<1>();
          release(pend);
        }
        pend = g++;
      };
      int kb = 0;
      for (; kb + 1 < nkb; kb += 2) {   // even K-blocks into acc0, odd ones into acc1
        step(acc0);
        step(acc1);
      }
      if (kb < nkb) step(acc0);
      wg_wait<0>();
      fence_regs<BN / 2>(acc0);
      fence_regs<BN / 2>(acc1);
      release(pend);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc0[i] = __fadd_rn(acc0[i], acc1[i]);
      tcs_epilogue<BN, EPI>(a, acc0, m0 + row_in_tile, n0, lane);
    }
  }
}

static size_t tcs_smem_bytes(int BN) {   // ring, mbarriers, row grid positions
  return (size_t)TCS_RING * (2 * tile_bytes(TC_BM) + 2 * tile_bytes(BN)) + 16 * TCS_RING + 2 * 128 * sizeof(int);
}

template <int BN, int EPI>
static int launch_tcs(const TcsArgs& a, cudaStream_t s) {
  static DeviceOnce once;
  const int dev = current_device();
  const size_t smem = tcs_smem_bytes(BN);
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(linear_tcs_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    once.done(dev);
  }
  const int ntiles = cdiv(a.M, TC_BM) * (a.N / BN), num_sms = device_sm_count(dev);
  linear_tcs_kernel<BN, EPI><<<ntiles < num_sms ? ntiles : num_sms, TC_THREADS, smem, s>>>(a);
  MVSF_LAUNCH_CHECK("linear_tcs");
  return MVSF_OK;
}

template <int BN>
static int launch_tcs_bn(const TcsArgs& a, int epi, cudaStream_t s) {
  switch (epi) {
    case LIN_BIAS: return launch_tcs<BN, LIN_BIAS>(a, s);
    case LIN_GELU: return launch_tcs<BN, LIN_GELU>(a, s);
    case LIN_ELU1: return launch_tcs<BN, LIN_ELU1>(a, s);
    case LIN_RES: return launch_tcs<BN, LIN_RES>(a, s);
    case LIN_SILU: return launch_tcs<BN, LIN_SILU>(a, s);
    default: return fail(MVSF_ERR_INVALID, "linear_tcs: unknown epilogue %d", epi);
  }
}

void tcs_token_rows(TcsArgs& a) {
  a.H = a.W = 1; a.cin = a.K; a.ntaps = 1; a.taps = 0x5ull; a.sy = a.sx = 1; a.py = a.px = 0;
}

// host-side argument checks of launch_linear_tcs; touch no device state
static int check_linear_tcs(const TcsArgs& a, int epi) {
  MVSF_REQUIRE(epi == LIN_BIAS || epi == LIN_GELU || epi == LIN_ELU1 || epi == LIN_RES || epi == LIN_SILU,
               "linear_tcs: unknown epilogue %d (streamed epilogues: 0 bias, 1 gelu, 2 elu+1, 3 residual, 6 silu)", epi);
  MVSF_REQUIRE(a.Ah && a.Al && a.Bh && a.Bl && (a.C || a.C2) && a.M > 0, "linear_tcs: bad arguments");
  MVSF_REQUIRE(a.N > 0 && a.N % 64 == 0 && a.cin > 0 && a.cin % TC_BK == 0 && a.ntaps >= 1 && a.ntaps <= 9 &&
                   a.K == a.ntaps * a.cin, "linear_tcs: need N %% 64 == 0, K = taps * cin, cin %% 64 == 0, 1 <= taps <= 9");
  MVSF_REQUIRE(a.H > 0 && a.W > 0 && a.H < 8192 && a.W < 8192 && a.M % (a.H * a.W) == 0 && a.sy >= 1 && a.sy <= 2 &&
                   a.sx >= 1 && a.sx <= 2 && a.py >= 0 && a.py < a.sy && a.px >= 0 && a.px < a.sx,
               "linear_tcs: bad implicit-GEMM grid");
  MVSF_REQUIRE((a.lda % 8) == 0 && (a.ldb % 8) == 0 && ((uintptr_t)a.Ah & 15) == 0 && ((uintptr_t)a.Al & 15) == 0 &&
                   ((uintptr_t)a.Bh & 15) == 0 && ((uintptr_t)a.Bl & 15) == 0, "linear_tcs: operands must be 16-byte aligned");
  if (a.C) MVSF_REQUIRE((a.ldc % 4) == 0 && ((uintptr_t)a.C & 15) == 0, "linear_tcs: C must be 16-byte aligned");
  if (a.C2) MVSF_REQUIRE((a.ldc2 % 8) == 0 && ((uintptr_t)a.C2 & 15) == 0, "linear_tcs: C2 must be 16-byte aligned");
  if (epi == LIN_RES)
    MVSF_REQUIRE(a.res && a.gamma && ((uintptr_t)a.res & 15) == 0 && ((uintptr_t)a.gamma & 15) == 0 && (a.ldres % 4) == 0,
                 "linear_tcs: residual epilogue needs 16-byte aligned res and gamma");
  if (a.bias) MVSF_REQUIRE(((uintptr_t)a.bias & 15) == 0, "linear_tcs: bias must be 16-byte aligned");
  MVSF_REQUIRE(!a.Cpre, "linear_tcs: no LayerNorm epilogues");
  return MVSF_OK;
}

int launch_linear_tcs(const TcsArgs& a, int epi, cudaStream_t s) {
  int rc;
  if ((rc = check_linear_tcs(a, epi))) return rc;
  return a.N % 128 == 0 ? launch_tcs_bn<128>(a, epi, s) : launch_tcs_bn<64>(a, epi, s);
}

// The fp16 hi + lo split of M rows of K fp32 values (launch_split_f16 in common.cuh): 8 values per thread, 16-byte
// loads and stores
__global__ void split_hi_lo_f16_kernel(const float* __restrict__ x, size_t ldx, __half* __restrict__ out, size_t ldo,
                                       size_t K, unsigned total) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x, k8 = (unsigned)(K / 8);
  if (i >= total) return;
  const unsigned m = i / k8;
  const size_t k = (size_t)(i - m * k8) * 8;
  const float4 a = ldg4(x + m * ldx + k), b = ldg4(x + m * ldx + k + 4);
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  split_store8(out + m * ldo + k, out + m * ldo + K + k, v);
}
int launch_split_f16(const float* x, size_t ldx, __half* out, size_t ldo, int M, size_t K, cudaStream_t s) {
  MVSF_REQUIRE(x && out && M > 0 && K > 0 && K % 8 == 0 && ldx >= K && ldx % 4 == 0 && ldo >= 2 * K && ldo % 8 == 0 &&
                   ((uintptr_t)x & 15) == 0 && ((uintptr_t)out & 15) == 0 && (size_t)M * (K / 8) <= 0xffffffffu,
               "split_f16: bad arguments");
  const unsigned total = (unsigned)((size_t)M * (K / 8));
  split_hi_lo_f16_kernel<<<cdiv(total, 256), 256, 0, s>>>(x, ldx, out, ldo, K, total);
  MVSF_LAUNCH_CHECK("split_hi_lo_f16");
  return MVSF_OK;
}

}  // namespace mvsf

using namespace mvsf;

extern "C" int mvsf_linear_tc_epilogue(int epi, const float* A, int lda, const float* W, const float* bias,
                                       const float* res, int ldres, const float* gamma, const float* ln_w,
                                       const float* ln_b, float ln_eps, int elu_cols, float* C, int ldc, float* Cpre,
                                       int ldcpre, void* C2, int ldc2, void* workspace, size_t workspace_bytes, int M,
                                       int N, int K, mvsf_stream_t stream) {
  MVSF_REQUIRE(A && W && workspace && M > 0 && K > 0, "linear_tc_epilogue: null pointer or empty shape");
  MVSF_REQUIRE(lda >= K && (lda % 4) == 0 && ((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0 &&
                   ((uintptr_t)workspace & 15) == 0,
               "linear_tc_epilogue: need lda >= K, lda %% 4 == 0, and A, W and workspace must be 16-byte aligned");
  const size_t need = ((size_t)M * 2 * K + (size_t)N * 2 * K) * sizeof(__half) + 256;
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "linear_tc_epilogue: workspace %zu < %zu bytes", workspace_bytes, need);
  __half* A2 = reinterpret_cast<__half*>(workspace);
  __half* B2 = A2 + align_up((size_t)M * 2 * K, 64);
  TcLinArgs a{};
  a.Ah = A2; a.Al = A2 + K; a.lda = 2 * K; a.Bh = B2; a.Bl = B2 + K; a.ldb = 2 * K;
  a.M = M; a.N = N; a.K = K; a.bias = bias; a.res = res; a.ldres = ldres; a.gamma = gamma;
  a.ln_w = ln_w; a.ln_b = ln_b; a.ln_eps = ln_eps; a.elu_cols = elu_cols;
  a.C = C; a.ldc = ldc; a.Cpre = Cpre; a.ldcpre = ldcpre; a.C2 = reinterpret_cast<__half*>(C2); a.ldc2 = ldc2;
  int rc;
  if ((rc = check_linear_tc(a, epi))) return rc;   // every rejection happens before the first launch
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = launch_split_f16(A, lda, A2, 2 * K, M, K, s))) return rc;
  if ((rc = launch_split_f16(W, K, B2, 2 * K, N, K, s))) return rc;
  return launch_linear_tc(a, epi, s);
}

extern "C" int mvsf_token_mlp_forward(int form, const float* A, const float* res, const float* proj_w, const float* proj_b,
                                      const float* gamma1, const float* mid_w, const float* mid_b, float mid_eps,
                                      const float* f1_w, const float* f1_b, const float* f2_w, const float* f2_b,
                                      const float* gamma2, const float* out_w, const float* out_b, float out_eps, float* C,
                                      void* C2, void* workspace, size_t workspace_bytes, int M, mvsf_stream_t stream) {
  MVSF_REQUIRE(A && proj_w && f1_w && f2_w && workspace && M > 0, "token_mlp_forward: null pointer or empty shape");
  MVSF_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)workspace & 15) == 0, "token_mlp_forward: A and workspace must be 16-byte aligned");
  constexpr size_t NP = 64 * 64, NF = 256 * 64;   // weights of proj, of FFN1 (and of FFN2)
  const size_t need = ((size_t)M * 128 + 2 * (NP + 2 * NF)) * sizeof(__half);
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "token_mlp_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  __half* A2 = reinterpret_cast<__half*>(workspace);
  __half* wp = A2 + (size_t)M * 128;   // hi | lo of each weight matrix, same indexing as the fp32 matrix
  __half* w1 = wp + 2 * NP;
  __half* w2 = w1 + 2 * NF;
  TokenMlpArgs a{};
  a.A = A2; a.res = res; a.C = C; a.C2 = reinterpret_cast<__half*>(C2); a.M = M;
  a.pw_h = wp; a.pw_l = wp + NP; a.f1w_h = w1; a.f1w_l = w1 + NF; a.f2w_h = w2; a.f2w_l = w2 + NF;
  a.proj_b = proj_b; a.gamma1 = gamma1; a.f1_b = f1_b; a.f2_b = f2_b; a.gamma2 = gamma2;
  a.mid_w = mid_w; a.mid_b = mid_b; a.mid_eps = mid_eps; a.out_w = out_w; a.out_b = out_b; a.out_eps = out_eps;
  int rc;
  if ((rc = check_token_mlp(a, form))) return rc;   // every rejection happens before the first launch
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = launch_split_f16(A, 64, A2, 128, M, 64, s))) return rc;
  if ((rc = launch_split_f16(proj_w, NP, wp, 2 * NP, 1, NP, s))) return rc;
  if ((rc = launch_split_f16(f1_w, NF, w1, 2 * NF, 1, NF, s))) return rc;
  if ((rc = launch_split_f16(f2_w, NF, w2, 2 * NF, 1, NF, s))) return rc;
  return launch_token_mlp(a, form, s);
}

extern "C" int mvsf_linear_tc_streamed_epilogue(int epi, const float* A, int lda, const float* W, const float* bias,
                                                const float* res, int ldres, const float* gamma, int elu_cols, float* C,
                                                int ldc, void* C2, int ldc2, void* workspace, size_t workspace_bytes,
                                                int M, int N, int K, mvsf_stream_t stream) {
  MVSF_REQUIRE(A && W && workspace && M > 0 && K > 0 && N > 0, "linear_tc_streamed_epilogue: null pointer or empty shape");
  MVSF_REQUIRE(lda >= K && (lda % 4) == 0 && ((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0 &&
                   ((uintptr_t)workspace & 15) == 0,
               "linear_tc_streamed_epilogue: need lda >= K, lda %% 4 == 0, and A, W and workspace must be 16-byte aligned");
  const size_t need = ((size_t)M * 2 * K + (size_t)N * 2 * K) * sizeof(__half) + 256;
  if (workspace_bytes < need)
    return fail(MVSF_ERR_WORKSPACE, "linear_tc_streamed_epilogue: workspace %zu < %zu bytes", workspace_bytes, need);
  __half* A2 = reinterpret_cast<__half*>(workspace);
  __half* B2 = A2 + align_up((size_t)M * 2 * K, 64);
  TcsArgs a{};
  a.Ah = A2; a.Al = A2 + K; a.lda = 2 * K; a.Bh = B2; a.Bl = B2 + K; a.ldb = 2 * K;
  a.M = M; a.N = N; a.K = K; a.bias = bias; a.res = res; a.ldres = ldres; a.gamma = gamma; a.elu_cols = elu_cols;
  a.C = C; a.ldc = ldc; a.C2 = reinterpret_cast<__half*>(C2); a.ldc2 = ldc2;
  tcs_token_rows(a);
  int rc;
  if ((rc = check_linear_tcs(a, epi))) return rc;   // every rejection happens before the first launch
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = launch_split_f16(A, lda, A2, 2 * K, M, K, s))) return rc;
  if ((rc = launch_split_f16(W, K, B2, 2 * K, N, K, s))) return rc;
  return launch_linear_tcs(a, epi, s);
}

/* fp32 weight blob -> fp16 hi / lo blobs with identical indexing (install time): out16 = [hi(n) | lo(n)] */
extern "C" int mvsf_split_weights_f16(const float* wts, void* out16, size_t n, mvsf_stream_t stream) {
  MVSF_REQUIRE(wts && out16 && n > 0 && (n % 8) == 0, "split_weights_f16: n must be a multiple of 8");
  __half* hi = reinterpret_cast<__half*>(out16);
  return launch_split_f16(wts, n, hi, 2 * n, 1, n, (cudaStream_t)stream);
}
