// 2-D convolution layer as an implicit GEMM on wgmma, one launch per layer: conv2d_tc_kernel<L, Src, Dst>.  Used by the
// FPN (fpn.cu: every 3x3 / 5x5 layer of the encoder and decoder) and by the FMT pathway (fmt.cu: the 3x3 smooth convs).
//   phase 1 (SIMT)   a "source" writes the input of the layer for one output tile plus its halo as fp16 hi|lo voxel-octet
//                    PLANES in shared memory (plane[row][col] = 8 channels = 16 B; zero outside the image = the padding), so
//                    a tap is a descriptor start address.  Strided layers use S x S PARITY planes (conv3d_tc.cu): plane
//                    (py, px) holds input rows S i + py, columns S j + px, and tap (kh, kw) of output (r, c) is row
//                    r + kh / S, column c + kw / S of parity plane (kh % S, kw % S).
//   phase 2 (wgmma)  M = 8 x 8 output pixels per m64 block, N = NS output channels of the CTA's N block.  Per 16 input
//                    channels: x_hi x [w_hi | w_lo] (N = 2 NS) and x_lo x w_hi (N = NS, onto the first half); 8 input
//                    channels: one MMA [x_hi | x_lo] x [[w_hi; w_hi] | [w_lo; 0]].  fp32 accumulators in registers.
//   phase 3          the two accumulator halves are added, plus the bias if the "destination" takes one (Dst::BIAS), and
//                    the destination applies its activation and stores the result.
// The weight tiles are packed once from fp32 by conv2d_pack_kernel and copied into shared memory by every CTA.
#pragma once
#include "wgmma.cuh"

namespace mvsf {
namespace c2d {
using namespace gmma;

// one layer: CI -> CO channels, KS x KS kernel, stride S, output tile TR rows x 32 columns, NS output channels per CTA
template <int CI_, int CO_, int KS_, int S_, int TR_, int NS_>
struct Conv {
  static constexpr int CI = CI_, CO = CO_, KS = KS_, S = S_, TR = TR_, NS = NS_;
  static constexpr int PAD = (KS - 1) / 2, HALO = (KS - 1) / S;
  static constexpr int PR = TR + HALO, PC = 32 + HALO;          // plane rows / columns
  static constexpr int NO = CI / 8, NP = S * S, NG = CI < 16 ? 1 : CI / 16, NB = CO / NS;
  static constexpr uint32_t PLANE = PR * PC * 16, PITCH = PC * 16;
  static constexpr uint32_t BT = 64 * NS;                      // (tap, group) weight tile: [2 k-chunks][2 NS rows][8 halves]
  static constexpr uint32_t WBYTES = KS * KS * NG * BT;        // weight tiles of one N block
  static constexpr uint32_t OFF_W = NP * NO * 2 * PLANE, SMEM = OFF_W + WBYTES;
  static_assert(CI % 8 == 0 && (CI == 8 || CI % 16 == 0) && CO % NS == 0 && TR % 8 == 0, "conv2d_tc shape");
  static_assert(NS == 8 || NS == 16 || NS == 32, "conv2d_tc N block");
  // plane of parity `par`, channel octet o, part hl (0 hi, 1 lo): groups of 16 channels are [hi o | lo o | hi o+1 | lo o+1]
  __device__ static constexpr uint32_t plane(int par, int o, int hl) { return (uint32_t)((par * NO + o) * 2 + hl) * PLANE; }
};

// Src::fill(smem, n, y0, x0, tid) is called by all 256 threads and writes the planes of the tile at (n, y0, x0); it may use
// Src::EXTRA bytes of shared memory after L::SMEM.  Dst::store(n, OH, OW, y, x, ch, a, b) receives the sums of the two
// accumulator halves (+ bias[ch], bias[ch + 1] when Dst::BIAS) of channels ch, ch + 1 of one output pixel.  The bias is a
// kernel parameter rather than a member of Dst: ptxas then schedules the FPN layers as it did before the template was
// shared (a bias pointer read from the Dst struct costs up to 63 registers).
template <class L, class Src, class Dst>
__global__ void __launch_bounds__(256)
conv2d_tc_kernel(const Src src, const Dst dst, const __half* __restrict__ wtc, const float* __restrict__ bias, int OH, int OW,
                 int tiles_x, int tiles_y, int ntiles) {
  constexpr int NS = L::NS, KS = L::KS, S = L::S, NG = L::NG;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb = blockIdx.y;
  const uint32_t sb = smem_u32(smem);
  // ---- once per CTA: the weight tiles of N block nb (packed by conv2d_pack_kernel)
  {
    const uint4* wsrc = reinterpret_cast<const uint4*>(wtc) + (size_t)nb * (L::WBYTES / 16);
    uint4* wdst = reinterpret_cast<uint4*>(smem + L::OFF_W);
    for (int i = tid; i < (int)(L::WBYTES / 16); i += 256) wdst[i] = __ldg(wsrc + i);
  }
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  float acc[2][NS];   // the m64 blocks of column groups 2 wg and 2 wg + 1: N = 2 NS accumulator columns [first | second]

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, n = tile / (tiles_x * tiles_y);
    const int x0 = tx * 32, y0 = ty * L::TR;
    src.fill(smem, n, y0, x0, tid);
    fence_proxy_async();
    __syncthreads();
#pragma unroll 1
    for (int rg = 0; rg < L::TR / 8; ++rg) {
      wg_fence();
#pragma unroll
      for (int kh = 0; kh < KS; ++kh) {
#pragma unroll
        for (int kw = 0; kw < KS; ++kw) {
          const int par = (kh % S) * S + (kw % S);
          const uint32_t aoff = (uint32_t)((8 * rg + kh / S) * L::PC + kw / S) * 16u;
#pragma unroll
          for (int g = 0; g < NG; ++g) {
            const uint64_t wb = make_desc(sb + L::OFF_W + (uint32_t)((kh * KS + kw) * NG + g) * L::BT, 2 * NS * 16, 128);
            const uint32_t first = (kh | kw | g) ? 1u : 0u;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const uint32_t arow = sb + aoff + (uint32_t)(2 * wg + k) * 128u;
              if constexpr (L::CI == 8) {   // K = [hi | lo] planes of the single octet
                mma_ss<2 * NS>(acc[k], make_desc(arow + L::plane(par, 0, 0), L::PLANE, L::PITCH), wb, first);
              } else {                      // K chunks = the hi (or lo) planes of octets 2 g and 2 g + 1
                const uint32_t ah = arow + L::plane(par, 2 * g, 0);
                mma_ss<2 * NS>(acc[k], make_desc(ah, 2 * L::PLANE, L::PITCH), wb, first);
                mma_ss<NS>(acc[k], make_desc(ah + L::PLANE, 2 * L::PLANE, L::PITCH), wb, 1u);
              }
            }
          }
        }
      }
      wg_commit();
      wg_wait<0>();
      fence_regs<NS>(acc[0]);
      fence_regs<NS>(acc[1]);
      // ---- epilogue: accumulator i of this thread = row 16 wq + lane / 4 + 8 h of the m64 block (pixel row 2 wq + h,
      //      column lane / 4), column 8 b + 2 q + e (+ NS for the x_hi w_lo half)
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int y = y0 + 8 * rg + 2 * wq + h, x = x0 + 8 * (2 * wg + k) + (lane >> 2);
          if (y >= OH || x >= OW) continue;
#pragma unroll
          for (int b = 0; b < NS / 8; ++b) {
            const int ch = nb * NS + 8 * b + 2 * q;
            float o0 = acc[k][4 * b + 2 * h] + acc[k][4 * b + 2 * h + NS / 2];
            float o1 = acc[k][4 * b + 2 * h + 1] + acc[k][4 * b + 2 * h + 1 + NS / 2];
            if constexpr (Dst::BIAS) {
              o0 += __ldg(bias + ch);
              o1 += __ldg(bias + ch + 1);
            }
            dst.store(n, OH, OW, y, x, ch, o0, o1);
          }
        }
    }
    __syncthreads();   // planes are free again
  }
}

// bytes of the packed weight tiles of a CI -> CO, KS x KS layer (all N blocks)
constexpr size_t conv2d_tc_bytes(int ci, int co, int ks) { return (size_t)ks * ks * (ci < 16 ? 1 : ci / 16) * 64 * co; }

// fp32 [KS*KS taps][CI][CO] -> the weight tiles of conv2d_tc_kernel, [N block][tap][group][2 kc][2 NS rows][8]
static __global__ void conv2d_pack_kernel(const float* __restrict__ w, __half* __restrict__ out, int CI, int CO, int KK,
                                          int NS) {
  const int NG = CI < 16 ? 1 : CI / 16;
  const long long total = (long long)KK * NG * 64 * CO / 2;   // halves
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i & 7);
    long long rest = i >> 3;
    const int row = (int)(rest % (2 * NS)); rest /= 2 * NS;
    const int kc = (int)(rest & 1); rest >>= 1;
    const int g = (int)(rest % NG); rest /= NG;
    const int tap = (int)(rest % KK), nb = (int)(rest / KK);
    const int part = row / NS, co = nb * NS + row % NS;
    const int ci = CI == 8 ? e : g * 16 + kc * 8 + e;
    const float wv = w[((size_t)tap * CI + ci) * CO + co];
    __half hi, lo;
    split_f16(wv, hi, lo);
    __half v;
    if (CI == 8) v = part == 0 ? hi : (kc == 0 ? lo : __float2half_rn(0.f));
    else v = part == 0 ? hi : lo;
    out[i] = v;
  }
}

static inline int pack_conv2d_tc(const float* w, void* out, int ci, int co, int ks, int ns, cudaStream_t s) {
  conv2d_pack_kernel<<<cdiv(conv2d_tc_bytes(ci, co, ks) / 2, 256), 256, 0, s>>>(w, static_cast<__half*>(out), ci, co,
                                                                                 ks * ks, ns);
  MVSF_LAUNCH_CHECK("conv2d_pack");
  return MVSF_OK;
}

// persistent launch: the N blocks of the layer on grid.y, tiles strided over at most (resident CTAs / N blocks) CTAs
template <class L, class Src, class Dst>
static int launch_conv(const Src& src, const Dst& dst, const void* wtc, const float* bias, int N, int OH, int OW,
                       cudaStream_t s) {
  constexpr uint32_t smem = L::SMEM + Src::EXTRA;
  static_assert(smem <= 227 * 1024, "conv2d_tc: shared memory");
  auto kern = conv2d_tc_kernel<L, Src, Dst>;
  static DeviceOnce once;
  static int per_sm = 1;
  const int dev = current_device();
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MVSF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
    if (per_sm < 1) per_sm = 1;
    once.done(dev);
  }
  const int tiles_x = cdiv(OW, 32), tiles_y = cdiv(OH, L::TR);
  const long long ntiles = (long long)tiles_x * tiles_y * N;
  MVSF_REQUIRE(ntiles < (1ll << 30), "conv2d_tc: image too large");
  long long cap = (long long)per_sm * device_sm_count(dev) / L::NB;
  if (cap < 1) cap = 1;
  dim3 grid((unsigned)(ntiles < cap ? ntiles : cap), L::NB);
  kern<<<grid, 256, smem, s>>>(src, dst, reinterpret_cast<const __half*>(wtc), bias, OH, OW, tiles_x, tiles_y, (int)ntiles);
  MVSF_LAUNCH_CHECK("conv2d_tc");
  return MVSF_OK;
}

}  // namespace c2d
}  // namespace mvsf
