// FMT pathway level (models/FMT.py:154-162,195-197):  out = smooth( bilinear_up2(red) + lateral )  with smooth = Conv2d(C, C, 3,
// padding=1, bias=False), fused into one persistent kernel.  Included by fmt.cu (inside namespace mvsf).
//   phase 1 (SIMT)   pre = lateral (NCHW) + bilinear_up2(red) (NHWC, F.interpolate align_corners=False) on the 18 x 34 halo
//                    of a 16 x 32 output tile, written as fp16 hi|lo voxel-octet planes in shared memory (zero outside the
//                    image = the conv padding) - the upsampled + added tensor never goes to HBM
//   phase 2 (wgmma)  3x3 conv as implicit GEMM: four 16 x 8 M-tiles (two m64 halves each, two M-tiles per warpgroup, one
//                    after the other), a tap = a descriptor start address (conv3d_tc.cu);
//                    C = 8: one MMA per tap  [x_hi | x_lo] x [[w_hi;w_hi] | [w_lo;0]]  (N = 32);
//                    C >= 16: per 16 channels  x_hi x [w_hi | w_lo] (N = 2C) and x_lo x w_hi (N = C) onto the first half
//   phase 3          accumulator registers: add the two halves, fp32 NHWC store
#pragma once

namespace sm2 {
using namespace gmma;
constexpr int PR = 18, PC = 34;
constexpr uint32_t PLANE = PR * PC * 16, PITCH = PC * 16;
template <int C>
struct Cfg {
  static constexpr int NO = C / 8;                       // channel octets
  static constexpr int NPAD = C < 16 ? 16 : C;           // rows of one weight part
  static constexpr int NG = C < 16 ? 1 : C / 16;         // K = 16 groups
  static constexpr uint32_t BT = 2 * 2 * NPAD * 16;      // one (tap, group) weight tile: 2 k-chunks x 2 NPAD rows x 16 B
  static constexpr uint32_t OFF_PL = 0, OFF_BT = 2 * NO * PLANE, SMEM = OFF_BT + 9 * NG * BT;
};
}  // namespace sm2

template <int C>
__global__ void __launch_bounds__(256)
fmt_smooth_tc_kernel(const float* __restrict__ red, const float* __restrict__ lat, const float* __restrict__ wts,
                     float* __restrict__ out, int h, int w, int tiles_x, int tiles_y, int ntiles) {
  using namespace sm2;
  using K = Cfg<C>;
  constexpr int NO = K::NO, NPAD = K::NPAD, NG = K::NG;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = 2 * h, W = 2 * w;
  const uint32_t sb = smem_u32(smem);

  // ---- once per CTA: weight tiles.  wts = [tap][ci][co] fp32.  Tile (tap, g) = [2 k-chunks][2 NPAD rows][8 halves]:
  //      C >= 16: rows [0, NPAD) = w_hi, [NPAD, 2 NPAD) = w_lo, k-chunk kc = input channels 16 g + 8 kc + e
  //      C == 8 : K = [x_hi | x_lo] of the single octet: rows [0,16) = w_hi in BOTH k-chunks; rows [16,32) = w_lo in k-chunk 0, 0 in 1
  for (int i = tid; i < 9 * NG * 2 * 2 * NPAD * 8; i += 256) {
    const int e = i & 7;
    int q = i >> 3;
    const int row = q % (2 * NPAD); q /= 2 * NPAD;
    const int kc = q & 1; q >>= 1;
    const int g = q % NG, tap = q / NG;
    const int part = row / NPAD, n = row % NPAD;
    const int ci = C < 16 ? e : g * 16 + kc * 8 + e;
    float wv = 0.f;
    if (n < C) wv = __ldg(wts + ((size_t)tap * C + ci) * C + n);
    const __half hi = __float2half_rn(wv), lo = __float2half_rn(wv - __half2float(hi));
    __half v;
    if (C < 16) v = part == 0 ? hi : (kc == 0 ? lo : __float2half_rn(0.f));
    else v = part == 0 ? hi : lo;
    reinterpret_cast<__half*>(smem + K::OFF_BT)[i] = v;
  }
  fence_proxy_async();
  __syncthreads();
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  float acc[2][NPAD];   // one M-tile: [m64 half][accumulator of N = 2 NPAD columns: first | second part]

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, v = tile / (tiles_x * tiles_y);
    const int x0 = tx * 32, y0 = ty * 16;
    const float* lv = lat + (size_t)v * C * H * W;
    const float* rv = red + (size_t)v * h * w * C;
    // ---- phase 1: pre = lateral + bilinear_up2(red) on the halo region -> planes [octet][hi|lo]
    for (int i = tid; i < NO * PR * PC; i += 256) {
      const int o = i / (PR * PC), pix = i - o * (PR * PC);
      const int r = pix / PC, c = pix - r * PC;
      const int y = y0 - 1 + r, x = x0 - 1 + c;
      float pre[8];
      if (y >= 0 && y < H && x >= 0 && x < W) {
        // ATen area_pixel_compute_source_index(scale=0.5, align_corners=False): src = 0.5*(dst+0.5)-0.5, clamped at 0
        const float sy = fmaxf(0.5f * ((float)y + 0.5f) - 0.5f, 0.0f);
        const int ya = (int)sy, yb = ya + ((ya < h - 1) ? 1 : 0);
        const float ly1 = sy - (float)ya, ly0 = 1.0f - ly1;
        const float sx = fmaxf(0.5f * ((float)x + 0.5f) - 0.5f, 0.0f);
        const int xa = (int)sx, xb = xa + ((xa < w - 1) ? 1 : 0);
        const float lx1 = sx - (float)xa, lx0 = 1.0f - lx1;
        const float* p00 = rv + ((size_t)ya * w + xa) * C + o * 8;
        const float* p01 = rv + ((size_t)ya * w + xb) * C + o * 8;
        const float* p10 = rv + ((size_t)yb * w + xa) * C + o * 8;
        const float* p11 = rv + ((size_t)yb * w + xb) * C + o * 8;
#pragma unroll
        for (int q4 = 0; q4 < 2; ++q4) {
          const float4 v00 = ldg4(p00 + q4 * 4), v01 = ldg4(p01 + q4 * 4), v10 = ldg4(p10 + q4 * 4), v11 = ldg4(p11 + q4 * 4);
          const float a00[4] = {v00.x, v00.y, v00.z, v00.w}, a01[4] = {v01.x, v01.y, v01.z, v01.w};
          const float a10[4] = {v10.x, v10.y, v10.z, v10.w}, a11[4] = {v11.x, v11.y, v11.z, v11.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float up = ly0 * (lx0 * a00[e] + lx1 * a01[e]) + ly1 * (lx0 * a10[e] + lx1 * a11[e]);
            pre[q4 * 4 + e] = up + __ldg(lv + ((size_t)(o * 8 + q4 * 4 + e) * H + y) * W + x);
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) pre[e] = 0.f;
      }
      __half* p = reinterpret_cast<__half*>(smem + K::OFF_PL + (uint32_t)(2 * o) * PLANE + (uint32_t)pix * 16u);
      split_store8(p, p + PLANE / 2, pre);     // hi plane of octet o, then its lo plane (+ PLANE bytes)
    }
    fence_proxy_async();
    __syncthreads();
#pragma unroll 1
    for (int k = 0; k < 2; ++k) {
      const int ct = 2 * wg + k;
      // ---- phase 2: MMAs of M-tile ct
      wg_fence();
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const uint32_t aoff = (uint32_t)(kh * PC + kw) * 16u + (uint32_t)ct * 128u;
#pragma unroll
          for (int g = 0; g < NG; ++g) {
            const uint64_t wb = make_desc(sb + K::OFF_BT + (uint32_t)((kh * 3 + kw) * NG + g) * K::BT, 2 * NPAD * 16, 128);
            const uint32_t first = (kh | kw | g) ? 1u : 0u;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
              const uint32_t arow = aoff + (uint32_t)hf * 8u * PITCH;
              if (C < 16) {   // K = [hi | lo] planes of the octet
                mma_ss<2 * NPAD>(acc[hf], make_desc(sb + K::OFF_PL + arow, PLANE, PITCH), wb, first);
              } else {
                // planes of group g: [hi o(2g) | lo o(2g) | hi o(2g+1) | lo o(2g+1)]: K chunks = the two hi (or lo) planes
                const uint32_t ah = sb + K::OFF_PL + (uint32_t)(4 * g) * PLANE + arow;
                mma_ss<2 * NPAD>(acc[hf], make_desc(ah, 2 * PLANE, PITCH), wb, first);
                mma_ss<NPAD>(acc[hf], make_desc(ah + PLANE, 2 * PLANE, PITCH), wb, 1u);
              }
            }
          }
        }
      }
      wg_commit();
      wg_wait<0>();
      fence_regs<NPAD>(acc[0]);
      fence_regs<NPAD>(acc[1]);
      // ---- phase 3: epilogue (channels 8 b + 2 q, + 1 of rows 8 hf + 2 wq + h, column 8 ct + lane / 4)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int y = y0 + 8 * hf + 2 * wq + h, x = x0 + 8 * ct + (lane >> 2);
          if (y >= H || x >= W) continue;
          float* op = out + (((size_t)v * H + y) * W + x) * C;
#pragma unroll
          for (int b = 0; b < NPAD / 8; ++b) {
            if (8 * b >= C) continue;
            const float o0 = acc[hf][4 * b + 2 * h] + acc[hf][4 * (b + NPAD / 8) + 2 * h];
            const float o1 = acc[hf][4 * b + 2 * h + 1] + acc[hf][4 * (b + NPAD / 8) + 2 * h + 1];
            *reinterpret_cast<float2*>(op + 8 * b + 2 * q) = make_float2(o0, o1);
          }
        }
    }
    __syncthreads();   // planes are free again
  }
}

template <int C>
static int launch_fmt_smooth_tc(const float* red, const float* lat, const float* wts, float* out, int V, int h, int w,
                                cudaStream_t s) {
  using K = sm2::Cfg<C>;
  static DeviceOnce once;
  static int per_sm = 1;   // a function of the kernel's compile-time footprint only
  const int dev = current_device();
  const int num_sms = device_sm_count(dev);
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(fmt_smooth_tc_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K::SMEM));
    MVSF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fmt_smooth_tc_kernel<C>, 256, K::SMEM));
    if (per_sm < 1) per_sm = 1;
    once.done(dev);
  }
  const int H = 2 * h, W = 2 * w;
  const int tiles_x = cdiv(W, 32), tiles_y = cdiv(H, 16);
  const long long ntiles = (long long)tiles_x * tiles_y * V;
  MVSF_REQUIRE(ntiles < (1ll << 30), "fmt pathway: image too large");
  const long long cap = (long long)per_sm * num_sms;
  fmt_smooth_tc_kernel<C><<<(int)(ntiles < cap ? ntiles : cap), 256, K::SMEM, s>>>(red, lat, wts, out, h, w, tiles_x, tiles_y,
                                                                                       (int)ntiles);
  MVSF_LAUNCH_CHECK("fmt_smooth_tc");
  return MVSF_OK;
}
