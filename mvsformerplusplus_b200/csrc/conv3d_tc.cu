// 3x3x3 convolutions of the U-Net cost regularisers (models/module.py:367-408 CostRegNet, :453-504 CostRegNet3D) as
// implicit GEMMs on the Hopper tensor cores (wgmma), fp32-class accuracy.
//
//   * activations live in HBM as two fp16 tensors (hi, lo; x ~= hi + lo carries 22 mantissa bits), NDHWC.  A tile is
//     16 (h) x 8*NT (w) cells of one depth slice.  Per (input depth slice, group of KG channel octets) "unit" ONE thread
//     issues TMA box loads (cp.async.bulk.tensor.5d over (c, w, h, d, hi|lo); the conv padding is TMA's out-of-bounds
//     zero fill) that land the halo of the tile in shared memory as PLANES of voxel octets: plane[row][col] = 8 channels
//     = 16 bytes.  Eight w-neighbours are then 128 contiguous bytes = one "core matrix" of the canonical no-swizzle
//     K-major layout, the h rows are the 8-row groups (SBO = row pitch) and hi / lo planes (or the two octets) are the
//     two K-chunks of a K = 16 MMA (LBO = plane distance).  A filter tap (kh, kw) is nothing but a different descriptor
//     start address: no im2col, no per-element address arithmetic anywhere;
//   * an M-tile is 16 x 8 cells = 128 GEMM rows; its two m64 halves (h rows 0-7 / 8-15) belong to the two MMA warpgroups,
//     which keep the fp32 accumulators in registers and run the epilogue themselves;
//   * KG = 1: per tap two wgmma (M = 64 cells, N = Cout, K = 16)
//         [x_hi | x_lo] x [w_hi ; w_hi]   and   [x_hi | x_lo] x [w_lo ; 0]       (x_lo*w_lo ~ 2^-22 is dropped)
//     KG = 2 (16 channels per unit): K = 16 spans the two octets and three MMAs x_lo*w_hi, x_hi*w_lo, x_hi*w_hi are
//     issued; the weight slabs come pre-arranged from conv3d_tc_pack and travel with the unit (one cp.async.bulk)
//     through the same mbarrier ring (expect_tx / complete_tx);
//   * stride-(SD,2,2) convolutions keep four parity planes (even/odd h x even/odd w, one strided tensor map each) so
//     that every tap is again a dense plane access; transposed convolutions run in gather form over INPUT cells with
//     four accumulators, one per output parity class (every (kh, kw) tap feeds exactly one class).  Taps that read the
//     same input shift (dih, diw) are fused along N: every shift is ONE MMA of N = 4 * NPAD over all four class
//     accumulators (in the order [0, 1, 3, 2]), with zero weight blocks for the classes it does not feed (9 of the 16
//     blocks are taps).  Each MMA thus writes the same register tuple with the same N, which is what lets ptxas keep
//     the MMAs in flight; MMAs into overlapping sub-ranges of one tuple with different N are serialised (C7511);
//   * persistent, warp-specialised CTAs (one per SM, tiles strided by gridDim.x): warpgroup 0 = TMA producer (one
//     thread), warpgroups 1-2 = MMA + epilogue (bias (folded BatchNorm), ReLU, skip add, fp16 hi|lo split or the fused
//     1x1x1 `prob` conv).  Ring: full[s] / empty[s]; each MMA warpgroup keeps one unit of MMAs in flight while it issues
//     the next, so loads and MMAs of consecutive units overlap, and the producer runs ahead into the next tile while the
//     epilogue of the current one runs.
#include "conv3d_tc.cuh"

#include <type_traits>

#include "linear_tc.cuh"
#include "wgmma.cuh"

namespace mvsf {

using namespace gmma;

namespace c3 {
constexpr int THREADS = 384, MAX_STAGES = 8;   // warpgroup 0: TMA (one thread), warpgroups 1-2: MMA + epilogue
template <int MODE, int NT>
struct Geo {
  static constexpr int TW = 8 * NT, TH = 16;
  static constexpr int PR = MODE == CONV_S1 ? TH + 2 : TH + 1;   // plane rows
  static constexpr int PC = MODE == CONV_S1 ? TW + 2 : TW + 1;   // plane columns (voxel octets)
  static constexpr int NSUB = MODE == CONV_S2 ? 4 : 1;           // parity sub-planes
  static constexpr uint32_t SUB_BYTES = PR * PC * 16;            // one plane; a TMA box = hi plane + lo plane
  static constexpr uint32_t PAIR = (2 * SUB_BYTES + 127) / 128 * 128;
  static constexpr uint32_t OCT_BYTES = NSUB * PAIR;             // everything of one channel octet
  static constexpr uint32_t PITCH = PC * 16;
};
__host__ __device__ inline int npad(int cout) { return cout < 16 ? 16 : cout; }
// one (kd, channel group) weight slab: 9 (conv) or 16 (transposed conv) blocks x 2 variants x (2 x NPAD x 16 B)
__host__ __device__ inline uint32_t slab_bytes(int mode, int cout) { return (uint32_t)npad(cout) * (mode == DECONV_S2 ? 1024u : 576u); }

struct alignas(64) Maps { CUtensorMap m[4]; };   // CONV_S2: one map per (h, w) parity; otherwise m[0]
}  // namespace c3

// depth taps (kd, id) of output slice od
struct DepthTaps { int n, kd[3], id[3]; };
template <int MODE>
__device__ __forceinline__ DepthTaps depth_taps(int od, int SD, int ID) {
  DepthTaps t;
  t.n = 0;
#pragma unroll
  for (int kd = 0; kd < 3; ++kd) {
    int id;
    bool ok = true;
    if (MODE == CONV_S1) id = od + kd - 1;
    else if (MODE == CONV_S2) id = od * SD + kd - 1;
    else {
      const int num = od + 1 - kd;
      if (SD == 1) id = num;
      else { ok = (num & 1) == 0; id = num >> 1; }
    }
    if (ok && id >= 0 && id < ID) { t.kd[t.n] = kd; t.id[t.n] = id; ++t.n; }
  }
  return t;
}

// epilogue of one GEMM row (cell) of one accumulator: channels 8 b + 2 q, + 1 (q = lane % 4) of accumulator row half h.
// Returns this thread's share of the fused 1x1x1 prob conv (OUT_PROB); the four threads of a quad hold one cell.
template <int OUT, int NPAD>
__device__ __forceinline__ float conv_epilogue_frag(const ConvTcArgs& a, const float* acc, int h, int q, bool valid, size_t vox) {
  const int COUT = a.COUT;
  float prob = 0.f;
#pragma unroll
  for (int b = 0; b < NPAD / 8; ++b) {
    const int c = 8 * b + 2 * q;
    if (8 * b >= COUT) continue;
    const float2 b2 = *reinterpret_cast<const float2*>(a.bias + c);
    float x0 = fmaxf(acc[4 * b + 2 * h] + b2.x, 0.f), x1 = fmaxf(acc[4 * b + 2 * h + 1] + b2.y, 0.f);
    if (!valid) continue;
    if (OUT == OUT_SPLIT) {
      if (a.skip_hi) {
        const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(a.skip_hi + vox * COUT + c));
        const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(a.skip_lo + vox * COUT + c));
        x0 += fh.x + fl.x;
        x1 += fh.y + fl.y;
      }
      split_store2(a.out_hi + vox * COUT + c, a.out_lo + vox * COUT + c, x0, x1);
    } else {
      const float2 s2 = *reinterpret_cast<const float2*>(a.skip32 + vox * COUT + c);
      x0 += s2.x; x1 += s2.y;
      if (OUT == OUT_F32) *reinterpret_cast<float2*>(a.out32 + vox * COUT + c) = make_float2(x0, x1);
      else prob = fmaf(x1, __ldg(a.probw + c + 1), x0 * __ldg(a.probw + c));
    }
  }
  return prob;
}

template <int NREG>
__device__ __forceinline__ void fence_acc(float (&acc)[NREG]) { fence_regs<NREG>(acc); }

// Persistent kernel: CTA i works on tiles i, i + gridDim.x, ...; tile = (output depth slice, 16 x 8*NT cells).
template <int MODE, int NT, int OUT, int NPAD>
__global__ void __launch_bounds__(c3::THREADS, 1)
conv3d_tc_kernel(const __grid_constant__ c3::Maps maps, ConvTcArgs a, int NS, int OD, int OH, int OW, int tiles_w,
                 int tiles_h, int ntiles) {
  using G = c3::Geo<MODE, NT>;
  constexpr int PC = G::PC, NSUB = G::NSUB;
  constexpr int NCLS = MODE == DECONV_S2 ? 4 : 1;
  constexpr int ACC = NCLS * NPAD / 2;                            // accumulator registers per M-tile
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int CIN = a.CIN, SD = a.SD, ID = a.ID, IH = a.IH, IW = a.IW;
  const int KG = a.KG;                                            // channel octets per unit
  const uint32_t b_bytes = c3::slab_bytes(MODE, NPAD);
  const uint32_t a_bytes = (uint32_t)KG * G::OCT_BYTES;
  const uint32_t stage_bytes = (a_bytes + b_bytes + 127u) / 128u * 128u;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + NS * stage_bytes;                 // full[8] | empty[8]
  const uint32_t bar_full = bars, bar_empty = bars + 64;
  const int ngroups = (CIN >> 3) / KG;

  if (tid == 0) {
    for (int i = 0; i < c3::MAX_STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // --------------------------------------------------------------------------------------- TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // registers go to the accumulators of the MMA warpgroups
    if (tid == 0) {
      uint32_t g = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, od = tile / (tiles_w * tiles_h);
        const int c0h = th * 16, c0w = tw * G::TW;
        const DepthTaps dt = depth_taps<MODE>(od, SD, ID);
        for (int ds = 0; ds < dt.n; ++ds) {
          for (int grp = 0; grp < ngroups; ++grp, ++g) {
            const int s = g % NS;
            mbar_wait(bar_empty + 8 * s, (uint32_t)(((g / NS) & 1) ^ 1));
            const uint32_t st = sbase + s * stage_bytes, full = bar_full + 8 * s;
            expect_tx(full, (uint32_t)(KG * NSUB) * 2u * G::SUB_BYTES + b_bytes);
            for (int og = 0; og < KG; ++og) {
              const int c = (grp * KG + og) * 8;
#pragma unroll
              for (int sub = 0; sub < NSUB; ++sub) {
                int w0, h0;
                if (MODE == CONV_S1) { w0 = c0w - 1; h0 = c0h - 1; }
                else if (MODE == CONV_S2) { w0 = c0w - (sub & 1); h0 = c0h - (sub >> 1); }   // odd plane: index j <-> 2j + 1
                else { w0 = c0w; h0 = c0h; }
                tma_load_5d(st + (uint32_t)(og * NSUB + sub) * G::PAIR, &maps.m[sub], c, w0, h0, dt.id[ds], 0, full);
              }
            }
            bulk_load(st + a_bytes, a.wtc + (size_t)(dt.kd[ds] * ngroups + grp) * (b_bytes / 2), b_bytes, full);
          }
        }
      }
    }
    return;
  }
  // ----------------------------------------------------------------------------------------- MMA + epilogue warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int half = (warp >> 2) - 1, wq = warp & 3, q = lane & 3, t128 = tid & 127;
  const uint32_t blk = (uint32_t)NPAD * 32u;   // one weight block: NPAD rows x 2 k-chunks
  float acc[NT][ACC];
  auto release = [&](uint32_t gb) { if (t128 == 0) mbar_arrive(bar_empty + 8 * (gb % NS)); };
  uint32_t g = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, od = tile / (tiles_w * tiles_h);
    const DepthTaps dt = depth_taps<MODE>(od, SD, ID);
    const int U = dt.n * ngroups;
    int pend = -1;
    for (int u = 0; u < U; ++u, ++g) {
      const int s = g % NS;
      mbar_wait(bar_full + 8 * s, (uint32_t)((g / NS) & 1));
      const uint32_t sA = sbase + s * stage_bytes + (uint32_t)half * 8u * G::PITCH, sB = sbase + s * stage_bytes + a_bytes;
      // one tap (conv) or input shift (transposed conv): A start offset, first weight block; N = NCLS * NPAD = all of acc[t]
      auto issue = [&](uint32_t aoff, int bstart, bool overwrite) {
        constexpr uint32_t n = (uint32_t)(NCLS * NPAD);
        const uint32_t t0 = sB + (uint32_t)bstart * 2u * blk, t1 = t0 + (uint32_t)NCLS * blk;
        const uint64_t b0 = make_desc(t0, n * 16u, 128), b1 = make_desc(t1, n * 16u, 128);
        // consecutive MMAs go to different accumulators (M-tiles): back-to-back MMAs on one accumulator serialise
        if (KG == 1) {
#pragma unroll
          for (int t = 0; t < NT; ++t)                                                       // K = [hi | lo] of one octet
            mma_ss<n>(acc[t], make_desc(sA + aoff + t * 128, G::SUB_BYTES, G::PITCH), b0, overwrite ? 0u : 1u);  // x [w_hi ; w_hi]
#pragma unroll
          for (int t = 0; t < NT; ++t)
            mma_ss<n>(acc[t], make_desc(sA + aoff + t * 128, G::SUB_BYTES, G::PITCH), b1, 1u);                 // x [w_lo ; 0]
        } else {
#pragma unroll
          for (int t = 0; t < NT; ++t)                                                       // K = two octets; lo planes
            mma_ss<n>(acc[t], make_desc(sA + G::SUB_BYTES + aoff + t * 128, G::OCT_BYTES, G::PITCH), b0, overwrite ? 0u : 1u);  // x_lo * w_hi
#pragma unroll
          for (int t = 0; t < NT; ++t)
            mma_ss<n>(acc[t], make_desc(sA + aoff + t * 128, G::OCT_BYTES, G::PITCH), b1, 1u);                 // x_hi * w_lo
#pragma unroll
          for (int t = 0; t < NT; ++t)
            mma_ss<n>(acc[t], make_desc(sA + aoff + t * 128, G::OCT_BYTES, G::PITCH), b0, 1u);                 // x_hi * w_hi
        }
      };
      wg_fence();
      if constexpr (MODE == DECONV_S2) {
        // input shift (dih, diw) -> classes [0, 1, 3, 2]; weight blocks in conv3d_tc_pack's order, zero where a class is not fed
        issue(0u, 0, u == 0);                               // (0,0): taps (1,1) (1,2) (2,2) (2,1)
        issue(16u, 4, false);                               // (0,1): -      (1,0) (2,0) -
        issue((uint32_t)PC * 16u, 8, false);                // (1,0): -      -     (0,2) (0,1)
        issue((uint32_t)(PC + 1) * 16u, 12, false);         // (1,1): -      -     (0,0) -
      } else {
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            int sub = 0, rs = kh, cs = kw;
            if (MODE == CONV_S2) {
              sub = (kh == 1 ? 0 : 2) + (kw == 1 ? 0 : 1);
              rs = kh == 2 ? 1 : 0; cs = kw == 2 ? 1 : 0;
            }
            issue((uint32_t)sub * G::PAIR + (uint32_t)(rs * PC + cs) * 16u, kh * 3 + kw, u == 0 && kh == 0 && kw == 0);
          }
        }
      }
      wg_commit();
      if (pend >= 0) {
        wg_wait<1>();
        release((uint32_t)pend);
      }
      pend = (int)g;
    }
    wg_wait<0>();
#pragma unroll
    for (int t = 0; t < NT; ++t) fence_acc(acc[t]);
    release((uint32_t)pend);
    // ---- epilogue: GEMM row 64 half + 16 wq + lane / 4 + 8 h = cell (h = 8 half + 2 wq + h, w = lane / 4) of an M-tile
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
      for (int cls = 0; cls < NCLS; ++cls)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ch = th * 16 + 8 * half + 2 * wq + h;
          const int cw = tw * G::TW + t * 8 + (lane >> 2);
          int oh, ow;
          bool valid;
          if (MODE == DECONV_S2) { oh = 2 * ch + (cls >> 1); ow = 2 * cw + (cls & 1); valid = ch < IH && cw < IW; }
          else { oh = ch; ow = cw; valid = ch < OH && cw < OW; }
          const size_t vox = valid ? ((size_t)od * OH + oh) * OW + ow : 0;
          float prob = conv_epilogue_frag<OUT, NPAD>(a, acc[t] + (cls ^ (cls >> 1)) * (NPAD / 2), h, q, valid, vox);   // class order [0, 1, 3, 2]
          if (OUT == OUT_PROB) {
            prob += __shfl_xor_sync(0xffffffffu, prob, 1);
            prob += __shfl_xor_sync(0xffffffffu, prob, 2);
            if (q == 0 && valid) a.out32[vox] = prob + __ldg(a.probw + a.COUT);
          }
        }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Depth-streaming variant for layers whose DEPTH stride is 1 (every 3x3x3 conv of CostRegNet3D, the stride-1 convs of
// CostRegNet).  The MMAs above are bound by the shared-memory read of the A operand, so instead of visiting an input
// slice three times - once per output slice it feeds - a work item is a COLUMN: a tile x a run of output depth slices
// [d0, d1).  Input slice `id` is loaded ONCE and one MMA per tap multiplies it with [W(kd=2) ; W(kd=1) ; W(kd=0)]
// (N = 3 * Cout), feeding the accumulators of the output slices id-1, id, id+1 at once.  The accumulators are a window
// of those three slices per M-tile, written whole by every MMA (one register tuple, one N: the MMAs stay pipelined);
// slice id-1 is complete once the MMAs of input slice id have retired and goes through the epilogue, then the window
// moves down one slice and its last third is zeroed before the next input slice is multiplied.  Thirds that fall
// outside the depth run [d0, d1) are computed and thrown away.  3x fewer A-operand reads and TMA bytes.
template <int MODE, int NT, int NPAD>
__global__ void __launch_bounds__(c3::THREADS, 1)
conv3d_col_kernel(const __grid_constant__ c3::Maps maps, ConvTcArgs a, int NS, int wres, int OH, int OW, int tiles_w,
                  int tiles_h, int DC, int nitems) {
  using G = c3::Geo<MODE, NT>;
  constexpr int PC = G::PC, NSUB = G::NSUB;
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int CIN = a.CIN, D = a.ID;
  const int KG = a.KG;
  const int ngroups = (CIN >> 3) / KG;
  const uint32_t slab = (uint32_t)NPAD * 1728u;                   // 9 taps x 2 variants x (2 k-chunks x 3*NPAD rows x 16 B)
  const uint32_t a_bytes = (uint32_t)KG * G::OCT_BYTES;
  const uint32_t stage_bytes = (a_bytes + (wres ? 0u : slab) + 127u) / 128u * 128u;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t wbase = sbase;                                   // resident weight slabs (wres)
  const uint32_t ring = sbase + (wres ? ((uint32_t)ngroups * slab + 127u) / 128u * 128u : 0u);
  const uint32_t bars = ring + NS * stage_bytes;                  // full[8] | empty[8] | wbar
  const uint32_t bar_full = bars, bar_empty = bars + 64, bar_w = bars + 128;

  if (tid == 0) {
    for (int i = 0; i < c3::MAX_STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 2); }
    mbar_init(bar_w, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int tiles_hw = tiles_w * tiles_h;

  if (warp < 4) {
    // --------------------------------------------------------------------------------------- TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0) {
      if (wres) {
        expect_tx(bar_w, (uint32_t)ngroups * slab);
        for (int grp = 0; grp < ngroups; ++grp) bulk_load(wbase + grp * slab, a.wtc + (size_t)grp * (slab / 2), slab, bar_w);
      }
      uint32_t g = 0;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int tw = item % tiles_w, th = (item / tiles_w) % tiles_h, ck = item / tiles_hw;
        const int c0h = th * 16, c0w = tw * G::TW;
        const int d0 = ck * DC, d1 = min(D, d0 + DC);
        const int first_id = max(d0 - 1, 0), last_id = min(d1, D - 1);
        for (int id = first_id; id <= last_id; ++id) {
          for (int grp = 0; grp < ngroups; ++grp, ++g) {
            const int s = g % NS;
            mbar_wait(bar_empty + 8 * s, (uint32_t)(((g / NS) & 1) ^ 1));
            const uint32_t st = ring + s * stage_bytes, full = bar_full + 8 * s;
            expect_tx(full, (uint32_t)(KG * NSUB) * 2u * G::SUB_BYTES + (wres ? 0u : slab));
            for (int og = 0; og < KG; ++og) {
              const int c = (grp * KG + og) * 8;
#pragma unroll
              for (int sub = 0; sub < NSUB; ++sub) {
                int w0, h0;
                if (MODE == CONV_S1) { w0 = c0w - 1; h0 = c0h - 1; }
                else { w0 = c0w - (sub & 1); h0 = c0h - (sub >> 1); }
                tma_load_5d(st + (uint32_t)(og * NSUB + sub) * G::PAIR, &maps.m[sub], c, w0, h0, id, 0, full);
              }
            }
            if (!wres) bulk_load(st + a_bytes, a.wtc + (size_t)grp * (slab / 2), slab, full);
          }
        }
      }
    }
    return;
  }
  // ----------------------------------------------------------------------------------------- MMA + epilogue warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int half = (warp >> 2) - 1, wq = warp & 3, q = lane & 3, t128 = tid & 127;
  if (wres) mbar_wait(bar_w, 0u);
  constexpr uint32_t btile = (uint32_t)NPAD * 96u;    // one (tap, variant) weight tile: 2 k-chunks x 3*NPAD rows x 16 B
  constexpr uint32_t blbo = (uint32_t)NPAD * 48u;     // k-chunk stride inside a weight tile
  constexpr int SL = NPAD / 2;                        // accumulator registers of one output slice
  float acc[NT][3 * SL];                              // [M-tile][output slices id-1, id, id+1 x NPAD columns]
  auto release = [&](uint32_t gb) { if (t128 == 0) mbar_arrive(bar_empty + 8 * (gb % NS)); };
  auto epilogue = [&](int od, int th, int tw, auto third_c) {   // output slice od (window third third_c) is complete
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ch = th * 16 + 8 * half + 2 * wq + h;
        const int cw = tw * G::TW + t * 8 + (lane >> 2);
        const bool valid = ch < OH && cw < OW;
        const size_t vox = valid ? ((size_t)od * OH + ch) * OW + cw : 0;
        conv_epilogue_frag<OUT_SPLIT, NPAD>(a, acc[t] + decltype(third_c)::value * SL, h, q, valid, vox);
      }
  };
  uint32_t g = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int tw = item % tiles_w, th = (item / tiles_w) % tiles_h, ck = item / tiles_hw;
    const int d0 = ck * DC, d1 = min(D, d0 + DC);
    const int first_id = max(d0 - 1, 0), last_id = min(d1, D - 1);
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
      for (int i = 0; i < 3 * SL; ++i) acc[t][i] = 0.f;
    for (int id = first_id; id <= last_id; ++id) {
      int pend = -1;
      for (int grp = 0; grp < ngroups; ++grp, ++g) {
        const int s = g % NS;
        mbar_wait(bar_full + 8 * s, (uint32_t)((g / NS) & 1));
        const uint32_t sA = ring + s * stage_bytes + (uint32_t)half * 8u * G::PITCH;
        const uint32_t sB = wres ? wbase + grp * slab : ring + s * stage_bytes + a_bytes;
        wg_fence();
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            int sub = 0, rs = kh, cs = kw;
            if (MODE == CONV_S2) {
              sub = (kh == 1 ? 0 : 2) + (kw == 1 ? 0 : 1);
              rs = kh == 2 ? 1 : 0; cs = kw == 2 ? 1 : 0;
            }
            const uint32_t aoff = sA + (uint32_t)sub * G::PAIR + (uint32_t)(rs * PC + cs) * 16u;
            const uint32_t t0 = sB + (uint32_t)(kh * 3 + kw) * 2u * btile, t1 = t0 + btile;   // w_hi tile, w_lo tile
            // variant list: (A start, A k-chunk stride, weight tile)
            const uint32_t va[3] = {KG == 1 ? aoff : aoff + G::SUB_BYTES, KG == 1 ? aoff : aoff, aoff};
            const uint32_t vl = KG == 1 ? G::SUB_BYTES : G::OCT_BYTES;
            const uint32_t vt[3] = {t0, t1, t0};
            const int nv = KG == 1 ? 2 : 3;     // KG 1: x [w_hi;w_hi], x [w_lo;0]   KG 2: x_lo*w_hi, x_hi*w_lo, x_hi*w_hi
#pragma unroll
            for (int v = 0; v < 3; ++v) {
              if (v >= nv) break;
              const uint64_t bd = make_desc(vt[v], blbo, 128);
#pragma unroll
              for (int t = 0; t < NT; ++t) mma_ss<3 * NPAD>(acc[t], make_desc(va[v] + t * 128, vl, G::PITCH), bd, 1u);
            }
          }
        }
        wg_commit();
        if (pend >= 0) {
          wg_wait<1>();
          release((uint32_t)pend);
        }
        pend = (int)g;
      }
      wg_wait<0>();
#pragma unroll
      for (int t = 0; t < NT; ++t) fence_acc(acc[t]);
      release((uint32_t)pend);
      if (id - 1 >= d0) epilogue(id - 1, th, tw, std::integral_constant<int, 0>{});
      if (id == last_id && id <= d1 - 1) epilogue(id, th, tw, std::integral_constant<int, 1>{});
#pragma unroll
      for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int i = 0; i < SL; ++i) {
          acc[t][i] = acc[t][SL + i];
          acc[t][SL + i] = acc[t][2 * SL + i];
          acc[t][2 * SL + i] = 0.f;
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------------- host
int conv3d_tc_kg(int mode, int cin) { return (mode != CONV_S2 && cin >= 16) ? 2 : 1; }
// depth-streaming kernel: convolutions with depth stride 1 whose 3*Cout-wide weight tiles still fit shared memory
int conv3d_tc_col(int mode, int sd, int cout) { return (mode == CONV_S1 || (mode == CONV_S2 && sd == 1)) && c3::npad(cout) <= 32; }

size_t conv3d_tc_packed_halves(int mode, int cin, int cout) {   // the same for the col layout
  return (size_t)3 * (cin / 8 / conv3d_tc_kg(mode, cin)) * (c3::slab_bytes(mode, cout) / 2);
}

// slab (kd, channel group g) = weight blocks of [2 MMA variants][2 k-chunks][NPAD rows][8 halves]; blocks that are fused
// into one MMA are interleaved as [variant][k-chunk][nb * NPAD rows][8] (conv: 9 taps, nb = 1; deconv: 4 input shifts,
// nb = 4 classes in the order [0, 1, 3, 2], zero where the shift does not feed the class)
// col layout (depth-streaming kernel): slab (channel group g) = [9 taps][2 variants][2 k-chunks][kd = 2, 1, 0][NPAD rows][8]
__global__ void conv3d_tc_pack_kernel(const float* __restrict__ w32, __half* __restrict__ out, int cin, int cout, int NPAD,
                                      int KG, int deconv, int col, size_t total) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int e = (int)(i & 7);
  const size_t q = i >> 3;                           // 16-byte chunk
  const int per_slab = col ? NPAD * 108 : (deconv ? NPAD * 64 : NPAD * 36);
  const int slab = (int)(q / per_slab), c = (int)(q % per_slab);
  const int ngroups = cin / 8 / KG;
  int kd = slab / ngroups, g = slab % ngroups;
  int mm, kc, n, kh = 0, kw = 0;
  bool tap = true;
  if (col) {
    g = slab;
    n = c % NPAD;
    int r = c / NPAD;
    kd = 2 - r % 3; r /= 3;
    kc = r & 1; r >>= 1;
    mm = r & 1; r >>= 1;
    kh = r / 3; kw = r % 3;
  } else if (!deconv) {
    n = c % NPAD;
    int r = c / NPAD;
    kc = r & 1; r >>= 1;
    mm = r & 1; r >>= 1;
    kh = r / 3; kw = r % 3;
  } else {
    // tap (kh, kw) of input shift t feeding class column b; -1: zero block
    const int tkh[4][4] = {{1, 1, 2, 2}, {-1, 1, 2, -1}, {-1, -1, 0, 0}, {-1, -1, 0, -1}};
    const int tkw[4][4] = {{1, 2, 2, 1}, {-1, 0, 0, -1}, {-1, -1, 2, 1}, {-1, -1, 0, -1}};
    const int t = c / (16 * NPAD), cc = c % (16 * NPAD);
    mm = cc / (8 * NPAD);
    kc = (cc / (4 * NPAD)) & 1;
    const int nn = cc % (4 * NPAD);
    const int b = nn / NPAD;
    n = nn % NPAD;
    kh = tkh[t][b]; kw = tkw[t][b];
    tap = kh >= 0;
  }
  const int ci = (KG == 1 ? g : g * 2 + kc) * 8 + e;
  float w = 0.f;
  if (tap && n < cout) w = w32[((size_t)((kd * 3 + kh) * 3 + kw) * cin + ci) * cout + n];
  __half hi, lo;
  split_f16(w, hi, lo);
  __half v;
  if (KG == 1) v = mm == 0 ? hi : (kc == 0 ? lo : __float2half_rn(0.f));
  else v = mm == 0 ? hi : lo;
  out[i] = v;
}

int conv3d_tc_pack(const float* w32, __half* out, int mode, int sd, int cin, int cout, cudaStream_t s) {
  MVSF_REQUIRE(w32 && out && cin % 8 == 0 && cout % 8 == 0, "conv3d_tc_pack: bad arguments");
  const size_t total = conv3d_tc_packed_halves(mode, cin, cout);
  conv3d_tc_pack_kernel<<<cdiv((long long)total, 256), 256, 0, s>>>(w32, out, cin, cout, c3::npad(cout),
                                                                     conv3d_tc_kg(mode, cin), mode == DECONV_S2 ? 1 : 0,
                                                                     conv3d_tc_col(mode, sd, cout), total);
  MVSF_LAUNCH_CHECK("conv3d_tc_pack");
  return MVSF_OK;
}

__global__ void merge_vec8_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ x, size_t n8) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 h = *reinterpret_cast<const uint4*>(hi + i * 8), l = *reinterpret_cast<const uint4*>(lo + i * 8);
  const __half2* h2 = reinterpret_cast<const __half2*>(&h);
  const __half2* l2 = reinterpret_cast<const __half2*>(&l);
  float r[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 fh = __half22float2(h2[e]), fl = __half22float2(l2[e]);
    r[2 * e] = fh.x + fl.x;
    r[2 * e + 1] = fh.y + fl.y;
  }
  *reinterpret_cast<float4*>(x + i * 8) = make_float4(r[0], r[1], r[2], r[3]);
  *reinterpret_cast<float4*>(x + i * 8 + 4) = make_float4(r[4], r[5], r[6], r[7]);
}
int launch_merge_vec8(const __half* hi, const __half* lo, float* x, size_t n, cudaStream_t s) {
  MVSF_REQUIRE(x && hi && lo && n > 0 && n % 8 == 0, "merge_vec8: bad arguments");
  merge_vec8_kernel<<<cdiv((long long)(n / 8), 256), 256, 0, s>>>(hi, lo, x, n / 8);
  MVSF_LAUNCH_CHECK("merge_vec8");
  return MVSF_OK;
}

// 5-D map (c, w, h, d, hi|lo) over the fp16 activation pair; sh/sw = 2 and (ph, pw) select one parity plane of (h, w)
static int make_map(CUtensorMap* m, const __half* hi, const __half* lo, int C, int D, int H, int W, int sh, int sw, int ph,
                    int pw, int box_w, int box_h) {
  EncodeTiledFn enc = encode_tiled_fn();
  MVSF_REQUIRE(enc, "conv3d_tc: cuTensorMapEncodeTiled is not available from this driver");
  const long long lo_off = (lo - hi) * (long long)sizeof(__half);
  MVSF_REQUIRE(lo_off > 0 && lo_off % 16 == 0, "conv3d_tc: the lo tensor must follow the hi tensor at a 16-byte multiple");
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)((W - pw + sw - 1) / sw), (cuuint64_t)((H - ph + sh - 1) / sh), (cuuint64_t)D, 2};
  const cuuint64_t strides[4] = {(cuuint64_t)sw * C * 2, (cuuint64_t)sh * W * C * 2, (cuuint64_t)H * W * C * 2, (cuuint64_t)lo_off};
  const cuuint32_t box[5] = {8, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 2};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  void* base = const_cast<__half*>(hi + ((size_t)ph * W + pw) * C);
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MVSF_ERR_CUDA, "conv3d_tc: cuTensorMapEncodeTiled failed (%d) for C=%d D=%d H=%d W=%d", (int)r, C, D, H, W);
  return MVSF_OK;
}

template <int MODE, int NT, int OUT, int NPAD>
static int launch_one(const ConvTcArgs& a, int NS, size_t smem, int OD, int OH, int OW, int cells_h, int cells_w,
                      int num_sms, cudaStream_t s) {
  using G = c3::Geo<MODE, NT>;
  auto kern = conv3d_tc_kernel<MODE, NT, OUT, NPAD>;
  static DeviceOnce once;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.done(dev);
  }
  c3::Maps maps;
  int rc;
  if (MODE == CONV_S2) {
    for (int sub = 0; sub < 4; ++sub)
      if ((rc = make_map(&maps.m[sub], a.in_hi, a.in_lo, a.CIN, a.ID, a.IH, a.IW, 2, 2, sub >> 1, sub & 1, G::PC, G::PR))) return rc;
  } else {
    if ((rc = make_map(&maps.m[0], a.in_hi, a.in_lo, a.CIN, a.ID, a.IH, a.IW, 1, 1, 0, 0, G::PC, G::PR))) return rc;
    maps.m[1] = maps.m[2] = maps.m[3] = maps.m[0];
  }
  const int tiles_w = cdiv(cells_w, 8 * NT), tiles_h = cdiv(cells_h, 16);
  const long long ntiles = (long long)tiles_w * tiles_h * OD;
  MVSF_REQUIRE(ntiles < (1ll << 30), "conv3d_tc: volume too large");
  const int grid = (int)(ntiles < num_sms ? ntiles : num_sms);
  kern<<<grid, c3::THREADS, smem, s>>>(maps, a, NS, OD, OH, OW, tiles_w, tiles_h, (int)ntiles);
  MVSF_LAUNCH_CHECK("conv3d_tc");
  return MVSF_OK;
}

// accumulator registers per MMA thread: NT x NCLS x NPAD / 2 <= 128
template <int MODE, int OUT, int NPAD>
static int launch_nt(const ConvTcArgs& a, int nt, int NS, size_t smem, int OD, int OH, int OW, int cells_h, int cells_w,
                     int num_sms, cudaStream_t s) {
  constexpr int NCLS = MODE == DECONV_S2 ? 4 : 1;
  if constexpr (4 * NCLS * NPAD <= 256)
    if (nt == 4) return launch_one<MODE, 4, OUT, NPAD>(a, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
  if constexpr (2 * NCLS * NPAD <= 256)
    if (nt == 2) return launch_one<MODE, 2, OUT, NPAD>(a, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
  return launch_one<MODE, 1, OUT, NPAD>(a, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
}

template <int MODE, int OUT>
static int launch_mode(const ConvTcArgs& a, cudaStream_t s) {
  int OD, OH, OW, cells_h, cells_w;
  if (MODE == CONV_S1) { OD = a.ID; OH = a.IH; OW = a.IW; cells_h = OH; cells_w = OW; }
  else if (MODE == CONV_S2) { OD = (a.ID - 1) / a.SD + 1; OH = (a.IH - 1) / 2 + 1; OW = (a.IW - 1) / 2 + 1; cells_h = OH; cells_w = OW; }
  else { OD = a.ID * a.SD; OH = a.IH * 2; OW = a.IW * 2; cells_h = a.IH; cells_w = a.IW; }
  const int num_sms = device_sm_count(current_device());
  const int NPAD = c3::npad(a.COUT);
  const uint32_t b_bytes = c3::slab_bytes(MODE, a.COUT);
  const int ncls = MODE == DECONV_S2 ? 4 : 1;
  // tile width: the widest tile (least halo) whose accumulators fit the registers of the MMA warpgroups and that keeps
  // the persistent CTAs busy
  int best_nt = 0;
  double best_eff = -1.0;
  const int nts[3] = {4, 2, 1};
  size_t stage_of[5] = {0, 0, 0, 0, 0};
  for (int k = 0; k < 3; ++k) {
    const int nt = nts[k];
    const uint32_t oct = nt == 4 ? c3::Geo<MODE, 4>::OCT_BYTES : (nt == 2 ? c3::Geo<MODE, 2>::OCT_BYTES : c3::Geo<MODE, 1>::OCT_BYTES);
    const size_t stage = align_up((size_t)a.KG * oct + b_bytes, 128);
    stage_of[nt] = stage;
    if (nt * ncls * NPAD > 256 || 2 * stage + 256 > 227 * 1024) continue;
    const long long ntiles = (long long)cdiv(cells_w, 8 * nt) * cdiv(cells_h, 16) * OD;
    const double eff = (double)ntiles / (double)(cdiv(ntiles, num_sms) * (long long)num_sms);
    if (eff >= 0.85) { best_nt = nt; break; }
    if (eff > best_eff) { best_eff = eff; best_nt = nt; }
  }
  MVSF_REQUIRE(best_nt > 0, "conv3d_tc: no tile shape fits (COUT %d)", a.COUT);
  const size_t stage = stage_of[best_nt];
  int NS = (int)((227 * 1024 - 256) / stage);
  if (NS > c3::MAX_STAGES) NS = c3::MAX_STAGES;
  const size_t smem = NS * stage + 256;
  if constexpr (OUT == OUT_SPLIT) {
    if (NPAD == 32) return launch_nt<MODE, OUT, 32>(a, best_nt, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
    if (NPAD == 64) return launch_nt<MODE, OUT, 64>(a, best_nt, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
  }
  return launch_nt<MODE, OUT, 16>(a, best_nt, NS, smem, OD, OH, OW, cells_h, cells_w, num_sms, s);
}


template <int MODE, int NT, int NPAD>
static int launch_col_one(const ConvTcArgs& a, int NS, int wres, size_t smem, int OH, int OW, int DC, int num_sms, cudaStream_t s) {
  using G = c3::Geo<MODE, NT>;
  auto kern = conv3d_col_kernel<MODE, NT, NPAD>;
  static DeviceOnce once;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    once.done(dev);
  }
  c3::Maps maps;
  int rc;
  if (MODE == CONV_S2) {
    for (int sub = 0; sub < 4; ++sub)
      if ((rc = make_map(&maps.m[sub], a.in_hi, a.in_lo, a.CIN, a.ID, a.IH, a.IW, 2, 2, sub >> 1, sub & 1, G::PC, G::PR))) return rc;
  } else {
    if ((rc = make_map(&maps.m[0], a.in_hi, a.in_lo, a.CIN, a.ID, a.IH, a.IW, 1, 1, 0, 0, G::PC, G::PR))) return rc;
    maps.m[1] = maps.m[2] = maps.m[3] = maps.m[0];
  }
  const int tiles_w = cdiv(OW, 8 * NT), tiles_h = cdiv(OH, 16);
  const long long nitems = (long long)tiles_w * tiles_h * cdiv(a.ID, DC);
  MVSF_REQUIRE(nitems < (1ll << 30), "conv3d_tc: volume too large");
  const int grid = (int)(nitems < num_sms ? nitems : num_sms);
  kern<<<grid, c3::THREADS, smem, s>>>(maps, a, NS, wres, OH, OW, tiles_w, tiles_h, DC, (int)nitems);
  MVSF_LAUNCH_CHECK("conv3d_col");
  return MVSF_OK;
}

template <int MODE>
static int launch_col(const ConvTcArgs& a, cudaStream_t s) {
  const int D = a.ID;
  const int OH = MODE == CONV_S1 ? a.IH : (a.IH - 1) / 2 + 1, OW = MODE == CONV_S1 ? a.IW : (a.IW - 1) / 2 + 1;
  const int num_sms = device_sm_count(current_device());
  const int NPAD = c3::npad(a.COUT);
  const int ngroups = a.CIN / 8 / a.KG;
  const size_t slab = (size_t)NPAD * 1728;
  const size_t wres_bytes = align_up(ngroups * slab, 128);
  const int wres = wres_bytes <= 112 * 1024 ? 1 : 0;            // all weight slabs stay resident in shared memory
  // (tile width, depth run) with the least redundant halo traffic per useful output at full occupancy of the persistent CTAs
  int best_nt = 0, best_dc = 0, best_ns = 0;
  size_t best_smem = 0;
  double best_cost = 1e30;
  const int nts[3] = {4, 2, 1};
  for (int k = 0; k < 3; ++k) {
    const int nt = nts[k];
    if (3 * nt * NPAD > 128) continue;                          // accumulator registers: 3 slices x NT x NPAD / 2 <= 64
    const uint32_t oct = nt == 4 ? c3::Geo<MODE, 4>::OCT_BYTES : (nt == 2 ? c3::Geo<MODE, 2>::OCT_BYTES : c3::Geo<MODE, 1>::OCT_BYTES);
    const size_t stage = align_up((size_t)a.KG * oct + (wres ? 0 : slab), 128);
    const size_t fixed = (wres ? wres_bytes : 0) + 256;
    int ns = (int)((227 * 1024 - fixed) / stage);
    if (ns > c3::MAX_STAGES) ns = c3::MAX_STAGES;
    if (ns < 2) continue;
    for (int div = 1; div <= 8; div *= 2) {
      const int dc = cdiv(D, div);
      if (div > 1 && dc == cdiv(D, div / 2)) continue;
      const long long items = (long long)cdiv(OW, 8 * nt) * cdiv(OH, 16) * cdiv(D, dc);
      const double eff = (double)items / (double)(cdiv(items, num_sms) * (long long)num_sms);
      const double halo_w = MODE == CONV_S1 ? (8.0 * nt + 2) / (8.0 * nt) : (16.0 * nt + 1) / (16.0 * nt);
      const double halo_d = dc >= D ? 1.0 : (dc + 2.0) / dc;
      const double cost = halo_w * halo_d / eff;
      if (cost < best_cost) { best_cost = cost; best_nt = nt; best_dc = dc; best_ns = ns; best_smem = fixed + ns * stage; }
    }
  }
  MVSF_REQUIRE(best_nt > 0, "conv3d_col: no tile shape fits (CIN %d COUT %d)", a.CIN, a.COUT);
  if (NPAD == 16) {
    if (best_nt == 2) return launch_col_one<MODE, 2, 16>(a, best_ns, wres, best_smem, OH, OW, best_dc, num_sms, s);
    return launch_col_one<MODE, 1, 16>(a, best_ns, wres, best_smem, OH, OW, best_dc, num_sms, s);
  }
  return launch_col_one<MODE, 1, 32>(a, best_ns, wres, best_smem, OH, OW, best_dc, num_sms, s);
}

int launch_conv3d_tc(const ConvTcArgs& a, int mode, int out_mode, cudaStream_t s) {
  MVSF_REQUIRE(a.in_hi && a.in_lo && a.wtc && a.bias, "conv3d_tc: null pointer");
  MVSF_REQUIRE(a.CIN % 8 == 0 && a.CIN >= 8 && a.CIN <= 64 && (a.COUT == 8 || a.COUT == 16 || a.COUT == 32 || a.COUT == 64),
               "conv3d_tc: input channels must be a multiple of 8 up to 64, output channels 8, 16, 32 or 64");
  MVSF_REQUIRE(a.SD == 1 || a.SD == 2, "conv3d_tc: depth stride must be 1 or 2");
  MVSF_REQUIRE(a.KG == conv3d_tc_kg(mode, a.CIN), "conv3d_tc: KG must be conv3d_tc_kg(mode, CIN) (it fixes the weight slab layout)");
  MVSF_REQUIRE(((uintptr_t)a.in_hi & 15) == 0 && ((uintptr_t)a.in_lo & 15) == 0 && ((uintptr_t)a.wtc & 15) == 0,
               "conv3d_tc: operands must be 16-byte aligned");
  MVSF_REQUIRE(a.col == conv3d_tc_col(mode, a.SD, a.COUT), "conv3d_tc: col must be conv3d_tc_col(mode, SD, COUT) (weight slab layout)");
  if (out_mode == OUT_SPLIT) {
    MVSF_REQUIRE(a.out_hi && a.out_lo, "conv3d_tc: split output missing");
    if (a.col) return mode == CONV_S1 ? launch_col<CONV_S1>(a, s) : launch_col<CONV_S2>(a, s);
    if (mode == CONV_S1) return launch_mode<CONV_S1, OUT_SPLIT>(a, s);
    if (mode == CONV_S2) return launch_mode<CONV_S2, OUT_SPLIT>(a, s);
    if (mode == DECONV_S2) return launch_mode<DECONV_S2, OUT_SPLIT>(a, s);
  } else if (mode == DECONV_S2 && (out_mode == OUT_F32 || out_mode == OUT_PROB)) {
    MVSF_REQUIRE(a.out32 && a.skip32 && a.COUT == 8 && (out_mode == OUT_F32 || a.probw), "conv3d_tc: fp32 output needs out32, skip32, COUT == 8");
    if (out_mode == OUT_F32) return launch_mode<DECONV_S2, OUT_F32>(a, s);
    return launch_mode<DECONV_S2, OUT_PROB>(a, s);
  }
  return fail(MVSF_ERR_INVALID, "conv3d_tc: unsupported mode %d / output %d", mode, out_mode);
}

}  // namespace mvsf

using namespace mvsf;

/* Test entry: one 3x3x3 layer through the tensor-core path with fp32 in/out (split, pack and merge done here).
 * in [ID][IH][IW][cin]; w32 = [27][cin][cout] then bias[cout]; skip (optional) and out [OD][OH][OW][cout]. */
extern "C" int mvsf_conv3d_tc_layer(int mode, int sd, const float* in, const float* w32, const float* skip, float* out,
                                    void* workspace, size_t workspace_bytes, int cin, int cout, int ID, int IH, int IW,
                                    mvsf_stream_t stream) {
  MVSF_REQUIRE(in && w32 && out && workspace && (mode >= 0 && mode <= 2) && (sd == 1 || sd == 2), "conv3d_tc_layer: bad arguments");
  MVSF_REQUIRE(cin % 8 == 0 && cout % 8 == 0, "conv3d_tc_layer: channels must be multiples of 8");
  int OD, OH, OW;
  if (mode == CONV_S1) { OD = ID; OH = IH; OW = IW; }
  else if (mode == CONV_S2) { OD = (ID - 1) / sd + 1; OH = (IH - 1) / 2 + 1; OW = (IW - 1) / 2 + 1; }
  else { OD = ID * sd; OH = IH * 2; OW = IW * 2; }
  const size_t nin = (size_t)ID * IH * IW * cin, nout = (size_t)OD * OH * OW * cout;
  const size_t nw = align_up(conv3d_tc_packed_halves(mode, cin, cout), 64);
  const size_t need = (2 * nin + 4 * nout + nw) * sizeof(__half) + 256;
  if (workspace_bytes < need) return fail(MVSF_ERR_WORKSPACE, "conv3d_tc_layer: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  __half* xin = reinterpret_cast<__half*>(workspace);
  __half* xout = xin + 2 * nin;
  __half* xskip = xout + 2 * nout;
  __half* wtc = xskip + 2 * nout;
  int rc;
  if ((rc = launch_split_f16(in, nin, xin, 2 * nin, 1, nin, s))) return rc;
  if (skip && (rc = launch_split_f16(skip, nout, xskip, 2 * nout, 1, nout, s))) return rc;
  if ((rc = conv3d_tc_pack(w32, wtc, mode, sd, cin, cout, s))) return rc;
  ConvTcArgs a{};
  a.in_hi = xin; a.in_lo = xin + nin; a.wtc = wtc; a.bias = w32 + (size_t)27 * cin * cout;
  if (skip) { a.skip_hi = xskip; a.skip_lo = xskip + nout; }
  a.out_hi = xout; a.out_lo = xout + nout;
  a.CIN = cin; a.COUT = cout; a.SD = sd; a.ID = ID; a.IH = IH; a.IW = IW; a.KG = conv3d_tc_kg(mode, cin);
  a.col = conv3d_tc_col(mode, sd, cout);
  if ((rc = launch_conv3d_tc(a, mode, OUT_SPLIT, s))) return rc;
  return launch_merge_vec8(xout, xout + nout, out, nout, s);
}
