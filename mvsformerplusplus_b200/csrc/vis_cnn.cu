// W4 visibility CNN: models/cost_volume.py:37,93
//   ConvBnReLU(1,16) -> ConvBnReLU(16,16) -> ConvBnReLU(16,8) -> Conv1x1(8,1) -> Sigmoid      (BN folded, fp32-class)
// One fused, persistent kernel; a CTA works on 14 x 30 output tiles and never writes the 16-channel intermediates to HBM
// (HBM traffic = 4 B in + 4 B out per pixel).
//   layer 1 (1 -> 16, 144 FMA / pixel)  SIMT over the 18 x 34 halo region; the result is stored as fp16 hi|lo VOXEL-OCTET
//                                       PLANES in shared memory (plane[row][col] = 8 channels = 16 B), the layout in
//                                       which a 3x3 tap is just another UMMA descriptor start address (see conv3d_tc.cu)
//   layer 2 (16 -> 16) and 3 (16 -> 8)  implicit GEMMs on wgmma: M-tile = 16 rows x 8 columns of pixels (two m64 halves of
//                                       8 rows), N = 16, K = 16 channels; per tap two MMAs: x_hi x [w_hi | w_lo] (N = 32,
//                                       both products side by side) and x_lo x w_hi (N = 16, accumulated onto the first
//                                       16 columns), fp32 accumulators in registers; each warpgroup owns two M-tiles; the
//                                       layer-2 epilogue (bias, ReLU, zero outside the image = layer 3's padding) writes
//                                       the planes of layer 3's input
//   layer 4 + sigmoid                   in the layer-3 epilogue (the 8 channels of a pixel sit in the 4 threads of a quad)
// The 16 x 32 region of layer 2 and the 14 x 30 tile of layer 3 are both covered by four 16 x 8 M-tiles; rows / columns of
// an M-tile that fall outside the useful region read the zero border of the plane buffers and are discarded.
// Two CTAs per SM (101 KB of shared memory each) overlap one CTA's SIMT phases with the other's MMAs.
// The fp32 SIMT version this replaces ran at 48 % of the FMA peak (1.9 ms per DTU depth map).
#include "common.cuh"
#include "linear_tc.cuh"
#include "wgmma.cuh"

namespace mvsf {

using namespace gmma;

namespace vc {
constexpr int TH = 14, TW = 30;                 // output tile
constexpr int PR = 18, PC = 34;                 // plane rows / columns (a1: all valid; a2: 16 x 32 valid, rest zero)
constexpr uint32_t PLANE = PR * PC * 16;        // 9792 B: one octet of channels, hi or lo
constexpr uint32_t PITCH = PC * 16;
constexpr int IN_R = 20, IN_C = 36;             // input region (3-pixel halo)
// packed weights (floats): w1[9][16] b1[16] w2[16][9][16] b2[16] w3[16][9][8] b3[8] w4[8] b4[1]
constexpr int OFF_W2 = 160, OFF_B2 = 160 + 2304, OFF_W3 = OFF_B2 + 16,
              OFF_B3 = OFF_W3 + 1152, OFF_W4 = OFF_B3 + 8, OFF_B4 = OFF_W4 + 8;
// shared memory (bytes): planes a1 [hi o0 | hi o1 | lo o0 | lo o1], planes a2, weight tiles, input, small params, barrier
constexpr uint32_t OFF_A1 = 0, OFF_A2 = 4 * PLANE, OFF_B2T = 8 * PLANE, BT_LAYER = 9 * 1024,      // [tap][2 kc][32 rows: w_hi | w_lo][8]
                   OFF_B3T = OFF_B2T + BT_LAYER, OFF_IN = OFF_B3T + BT_LAYER, OFF_PAR = OFF_IN + IN_R * IN_C * 4,
                   SMEM = OFF_PAR + 1024;
// small parameter block (floats): w1[144] b1[16] b2[16] b3[8] w4[8] b4[1]
constexpr int P_W1 = 0, P_B1 = 144, P_B2 = 160, P_B3 = 176, P_W4 = 184, P_B4 = 192;
}  // namespace vc

__global__ void __launch_bounds__(256, 2)
vis_cnn_kernel(const float* __restrict__ entropy, const float* __restrict__ wts, float* __restrict__ vis, int H, int W,
               int tiles_x, int tiles_y, int ntiles) {
  using namespace vc;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sb = smem_u32(smem);
  float* in_s = reinterpret_cast<float*>(smem + OFF_IN);
  float* par = reinterpret_cast<float*>(smem + OFF_PAR);
  // ---- once per CTA: parameters, fp16 hi|lo weight tiles in the canonical K-major B layout, zero border of a2
  for (int i = tid; i < 160; i += 256) par[i] = __ldg(wts + i);                      // w1, b1
  if (tid < 16) par[P_B2 + tid] = __ldg(wts + OFF_B2 + tid);
  if (tid < 8) { par[P_B3 + tid] = __ldg(wts + OFF_B3 + tid); par[P_W4 + tid] = __ldg(wts + OFF_W4 + tid); }
  if (tid == 0) par[P_B4] = __ldg(wts + OFF_B4);
  for (int i = tid; i < 2 * 9 * 2 * 16 * 8; i += 256) {   // (layer, tap, k-chunk, row n, e) -> hi and lo tiles
    const int e = i & 7, n = (i >> 3) & 15, kc = (i >> 7) & 1, tap = (i >> 8) % 9, layer = i / (9 * 256);
    const int ci = kc * 8 + e;
    float w = 0.f;
    if (layer == 0) w = __ldg(wts + OFF_W2 + (ci * 9 + tap) * 16 + n);
    else if (n < 8) w = __ldg(wts + OFF_W3 + (ci * 9 + tap) * 8 + n);
    __half hi, lo;
    split_f16(w, hi, lo);
    __half* t = reinterpret_cast<__half*>(smem + (layer ? OFF_B3T : OFF_B2T) + tap * 1024);
    t[kc * 256 + n * 8 + e] = hi;
    t[kc * 256 + (16 + n) * 8 + e] = lo;
  }
  for (int i = tid; i < (int)(4 * PLANE / 16); i += 256) reinterpret_cast<uint4*>(smem + OFF_A2)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();
  const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
  float acc[2][2][16];   // [M-tile 2 wg + k][m64 half][accumulator]

  // MMAs of one 3x3 layer over this warpgroup's two M-tiles: planes at `pl`, weight tiles at `bt`
  // accumulator columns: [0, 16) = x_hi w_hi + x_lo w_hi, [16, 32) = x_hi w_lo
  auto issue_layer = [&](uint32_t pl, uint32_t bt) {
    wg_fence();
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const uint32_t aoff = (uint32_t)(kh * PC + kw) * 16u;
        const uint64_t wb = make_desc(bt + (kh * 3 + kw) * 1024, 512, 128);
        const uint32_t first = (kh | kw) ? 1u : 0u;
#pragma unroll
        for (int k = 0; k < 2; ++k)
#pragma unroll
          for (int hf = 0; hf < 2; ++hf)
            mma_ss<32>(acc[k][hf], make_desc(pl + aoff + (2 * wg + k) * 128 + hf * 8 * PITCH, PLANE, PITCH), wb, first);
#pragma unroll
        for (int k = 0; k < 2; ++k)
#pragma unroll
          for (int hf = 0; hf < 2; ++hf)
            mma_ss<16>(acc[k][hf], make_desc(pl + 2 * PLANE + aoff + (2 * wg + k) * 128 + hf * 8 * PITCH, PLANE, PITCH), wb, 1u);
      }
    }
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) fence_regs<16>(acc[k][hf]);
  };

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, n = tile / (tiles_x * tiles_y);
    const int x0 = tx * TW, y0 = ty * TH;
    const float* __restrict__ E = entropy + (size_t)n * H * W;
    // ---- input region (zero outside the image: layer 1's padding)
    for (int i = tid; i < IN_R * IN_C; i += 256) {
      const int r = i / IN_C, c = i - r * IN_C;
      const int gy = y0 - 3 + r, gx = x0 - 3 + c;
      in_s[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(E + (size_t)gy * W + gx) : 0.0f;
    }
    __syncthreads();
    // ---- layer 1 on the 18 x 34 region -> planes a1 (zero outside the image: layer 2's padding)
    for (int i = tid; i < PR * PC; i += 256) {
      const int r = i / PC, c = i - r * PC;
      const int gy = y0 - 2 + r, gx = x0 - 2 + c;
      const bool inside = gy >= 0 && gy < H && gx >= 0 && gx < W;
      float acc[16];
#pragma unroll
      for (int oc = 0; oc < 16; ++oc) acc[oc] = par[P_B1 + oc];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float v = in_s[(r + ky) * IN_C + c + kx];
          const float* wp = par + P_W1 + (ky * 3 + kx) * 16;
#pragma unroll
          for (int oc = 0; oc < 16; ++oc) acc[oc] = fmaf(v, wp[oc], acc[oc]);
        }
#pragma unroll
      for (int oc = 0; oc < 16; ++oc) acc[oc] = inside ? fmaxf(acc[oc], 0.0f) : 0.0f;
      __half* p = reinterpret_cast<__half*>(smem + OFF_A1 + (uint32_t)i * 16u);
      const float (&lo8)[8] = reinterpret_cast<const float (&)[8]>(acc[0]);
      const float (&hi8)[8] = reinterpret_cast<const float (&)[8]>(acc[8]);
      // p is a __half*: + PLANE / 2 elements = + PLANE bytes.  Planes: [hi o0 | hi o1 | lo o0 | lo o1]
      split_store8(p, p + PLANE, lo8);                           // channels 0-7 : hi -> plane 0, lo -> plane 2
      split_store8(p + PLANE / 2, p + PLANE / 2 + PLANE, hi8);   // channels 8-15: hi -> plane 1, lo -> plane 3
    }
    fence_proxy_async();
    __syncthreads();
    issue_layer(sb + OFF_A1, sb + OFF_B2T);
    // ---- layer-2 epilogue: bias, ReLU, zero outside the image -> planes a2 (16 x 32 region anchored at row 0, column 0)
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int er = 8 * hf + 2 * wq + h, c = 16 * wg + 8 * k + (lane >> 2);
          const int gy = y0 - 1 + er, gx = x0 - 1 + c;
          const bool inside = gy >= 0 && gy < H && gx >= 0 && gx < W;
          __half* p = reinterpret_cast<__half*>(smem + OFF_A2 + (uint32_t)(er * PC + c) * 16u) + 2 * q;
#pragma unroll
          for (int b = 0; b < 2; ++b) {   // channel octet b: channels 8 b + 2 q, + 1
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float x = acc[k][hf][4 * b + 2 * h + e] + acc[k][hf][4 * (b + 2) + 2 * h + e];
              v[e] = inside ? fmaxf(x + par[P_B2 + 8 * b + 2 * q + e], 0.0f) : 0.0f;
            }
            // p is a __half*: + PLANE / 2 elements = + PLANE bytes.  Planes: [hi o0 | hi o1 | lo o0 | lo o1]
            split_store2(p + b * (PLANE / 2), p + b * (PLANE / 2) + PLANE, v[0], v[1]);
          }
        }
    fence_proxy_async();
    __syncthreads();
    issue_layer(sb + OFF_A2, sb + OFF_B3T);
    // ---- layer-3 epilogue: bias, ReLU, 1x1 conv, sigmoid (channels 2 q, 2 q + 1 here, the quad adds the rest)
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = 0.f;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int oc = 2 * q + e;
            const float x = acc[k][hf][2 * h + e] + acc[k][hf][8 + 2 * h + e];
            s = fmaf(fmaxf(x + par[P_B3 + oc], 0.f), par[P_W4 + oc], s);
          }
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          const int er = 8 * hf + 2 * wq + h, ox = 16 * wg + 8 * k + (lane >> 2);
          const int gy = y0 + er, gx = x0 + ox;
          if (q == 0 && er < TH && ox < TW && gy < H && gx < W)
            vis[((size_t)n * H + gy) * W + gx] = __fdiv_rn(1.0f, 1.0f + expf(-(s + par[P_B4])));
        }
    __syncthreads();   // a1, a2 and the input tile are free again
  }
}

}  // namespace mvsf

using namespace mvsf;

extern "C" int mvsf_vis_cnn(const float* entropy, const float* wts, float* vis, int N, int H, int W,
                            mvsf_stream_t stream) {
  MVSF_REQUIRE(entropy && wts && vis && N > 0 && N <= 65535 && H > 0 && W > 0, "vis_cnn: bad arguments");
  static DeviceOnce once;
  const int dev = current_device();
  const int num_sms = device_sm_count(dev);
  if (once.need(dev)) {
    MVSF_CUDA_OK(cudaFuncSetAttribute(vis_cnn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vc::SMEM));
    once.done(dev);
  }
  const int tiles_x = cdiv(W, vc::TW), tiles_y = cdiv(H, vc::TH);
  const long long ntiles = (long long)tiles_x * tiles_y * N;
  MVSF_REQUIRE(ntiles < (1ll << 30), "vis_cnn: image too large");
  const int grid = (int)(ntiles < 2 * num_sms ? ntiles : 2 * num_sms);
  vis_cnn_kernel<<<grid, 256, vc::SMEM, (cudaStream_t)stream>>>(entropy, wts, vis, H, W, tiles_x, tiles_y, (int)ntiles);
  MVSF_LAUNCH_CHECK("vis_cnn");
  return MVSF_OK;
}
