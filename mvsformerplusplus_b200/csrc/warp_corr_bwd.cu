// Adjoint of the view aggregation (pass B, warp_corr.cu): the gradients of the cost volume
//   vm[g,d] = sum_v w_v c_v[g,d] / (S + 1e-6),   c_v[g,d] = (1/Cg) sum_{c in g} ref[c] s_v[c,d],   S = sum_v w_v
// with respect to the features (reference and source views) and the visibility weights w_v (models/cost_volume.py:72-101
// under autograd).  With U = dL/dvm and u = U / (S + 1e-6):
//   dL/dw_v    = sum_{g,d} u c_v  -  sum_{g,d} u vm
//   dL/dref[c] = sum_v sum_d u[g(c),d] w_v s_v[c,d] / Cg
//   dL/dsrc_v  = u[g(c),d] w_v ref[c] / Cg scattered to the four corners of tap (p, d) with the tap's bilinear weights.
// The warped samples s_v are recomputed here with the forward's own tap set-up (warp_coord_fast + make_tap_fast through
// build_taps), so every corner and weight equals the one the forward used: a corner the forward weights 0 receives
// nothing, and a tap with non-finite coordinates (weights all 0) contributes nothing anywhere.
//
// Organisation: pass B run backwards.  LPP = C/4 lanes per reference pixel, each holding 4 channels of ref and of its
// gradient in registers; the warp's taps are built once per (view, chunk) into the shared tap table; the per-view weight
// gradient is summed over the pixel's lanes with a butterfly.  The reference-view gradient and dL/dw are each written once
// per element (bit-reproducible); the source-view gradient is accumulated with one red.global.add.v4.f32 per corner and
// lane, so its bits depend on the order the atomics land (as torch's grid_sample backward).
#include "warp_geom.cuh"

namespace mvsf {

__device__ __forceinline__ void red_add4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// GENERIC: D > DCH, the upstream gradient of each chunk is reloaded per view (the shipped stages have D == DCH: it stays in
// registers for the whole view loop)
template <int C, bool GENERIC>
__global__ void __launch_bounds__(256)
warp_corr_aggregate_bwd_kernel(const float* __restrict__ feat, const float* __restrict__ homs,
                               const float* __restrict__ depth, const float* __restrict__ vis,
                               const float* __restrict__ volume, const float* __restrict__ gvol,
                               float* __restrict__ gfeat, float* __restrict__ gvis, int V, int D, int H, int W) {
  constexpr int LPP = WC<C>::LPP, P = WC<C>::P, DCH = WC<C>::DCH;
  constexpr int G = 8, CPG = C / G;
  constexpr int NGL = (CPG >= 4) ? 1 : 4 / CPG;   // groups per lane
  constexpr int LPG = (CPG >= 4) ? CPG / 4 : 1;   // lanes per group (1 or 2)
  constexpr float inv_cpg = 1.0f / (float)CPG;
  __shared__ TapTable tables[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  TapTable& tb = tables[warp];
  const int HW = H * W;
  const int pix0 = (blockIdx.x * 8 + warp) * P;
  if (pix0 >= HW) return;
  const int p1 = min(pix0 + lane % P, HW - 1);
  const int p2raw = pix0 + lane / LPP;
  const bool active = p2raw < HW;
  const int p2 = active ? p2raw : HW - 1;
  const int lip = lane % LPP, pi = lane / LPP;
  const int g0 = lip * 4 / CPG;   // first group of this lane's 4 channels
  const CoordConst cc = make_coord_const(W, H);
  const int y1 = p1 / W, x1 = p1 - y1 * W;
  const float fx = (float)x1, fy = (float)y1;
  const float4 r = ldg4(feat + (size_t)p2 * C + lip * 4);
  const float rr[4] = {r.x, r.y, r.z, r.w};

  // S in the forward's order, and its denominator
  float wsum = 0.f;
  for (int v = 0; v < V - 1; ++v) wsum = __fadd_rn(wsum, __ldg(vis + (size_t)v * HW + p2));
  const float den = __fadd_rn(wsum, 1e-6f);

  // u = U / den for this lane's groups and hypotheses [d0, d0 + DCH); zero beyond D
  float u[DCH][NGL];
  auto load_u = [&](int d0) {
#pragma unroll
    for (int di = 0; di < DCH; ++di)
#pragma unroll
      for (int j = 0; j < NGL; ++j)
        u[di][j] = (d0 + di < D) ? __fdiv_rn(__ldg(gvol + ((size_t)(d0 + di) * HW + p2) * G + g0 + j), den) : 0.f;
  };
  // T = sum_{g,d} u vm (the view-independent term of dL/dw); with two lanes per group the even lane counts it
  float T = 0.f;
  for (int d0 = 0; d0 < D; d0 += DCH) {
    load_u(d0);
    if (lip % LPG == 0) {
#pragma unroll
      for (int di = 0; di < DCH; ++di)
#pragma unroll
        for (int j = 0; j < NGL; ++j)
          if (d0 + di < D) T = fmaf(u[di][j], __ldg(volume + ((size_t)(d0 + di) * HW + p2) * G + g0 + j), T);
    }
  }
#pragma unroll
  for (int o = LPP / 2; o > 0; o >>= 1) T += __shfl_xor_sync(0xffffffffu, T, o);   // u now holds chunk 0

  float gr[4] = {0.f, 0.f, 0.f, 0.f};
  for (int v = 0; v < V - 1; ++v) {
    const Hom m = load_hom(homs + (size_t)v * 12);
    const float3 ray = ref_ray(m, fx, fy);
    const float w = __ldg(vis + (size_t)v * HW + p2);
    const float ws = w * inv_cpg;   // exact: Cg is a power of two
    const float* __restrict__ src = feat + (size_t)(v + 1) * HW * C + lip * 4;
    float* gsrc = gfeat + (size_t)(v + 1) * HW * C + lip * 4;
    float gw = 0.f;   // this lane's part of sum_{g,d} u c_v, before the 1/Cg
    for (int d0 = 0; d0 < D; d0 += DCH) {
      if (GENERIC) load_u(d0);
      build_taps<C>(tb, depth, m, ray, cc, p1, d0, D, HW, H, W, lane);
      __syncwarp();
#pragma unroll
      for (int di = 0; di < DCH; ++di) {
        const int4 o = tb.off[di * P + pi];
        const float4 wt = tb.wt[di * P + pi];
        const float4 s4 = gather4(src, o, wt);
        const float s[4] = {s4.x, s4.y, s4.z, s4.w};
        float e[4];   // dL/dsrc of each channel before the corner weights
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float uc = u[di][c * NGL / 4];
          gw = fmaf(uc, rr[c] * s[c], gw);
          const float a = uc * ws;
          gr[c] = fmaf(a, s[c], gr[c]);
          e[c] = a * rr[c];
        }
        if (active && d0 + di < D) {
          if (wt.x != 0.f) red_add4(gsrc + o.x, e[0] * wt.x, e[1] * wt.x, e[2] * wt.x, e[3] * wt.x);
          if (wt.y != 0.f) red_add4(gsrc + o.y, e[0] * wt.y, e[1] * wt.y, e[2] * wt.y, e[3] * wt.y);
          if (wt.z != 0.f) red_add4(gsrc + o.z, e[0] * wt.z, e[1] * wt.z, e[2] * wt.z, e[3] * wt.z);
          if (wt.w != 0.f) red_add4(gsrc + o.w, e[0] * wt.w, e[1] * wt.w, e[2] * wt.w, e[3] * wt.w);
        }
      }
      __syncwarp();
    }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1) gw += __shfl_xor_sync(0xffffffffu, gw, o);
    if (active && lip == 0) gvis[(size_t)v * HW + p2] = __fsub_rn(gw * inv_cpg, T);
  }
  if (active) *reinterpret_cast<float4*>(gfeat + (size_t)p2 * C + lip * 4) = make_float4(gr[0], gr[1], gr[2], gr[3]);
}

template <int C>
static void launch_aggregate_bwd(const float* feat, const float* homs, const float* depth, const float* vis,
                                 const float* volume, const float* gvol, float* gfeat, float* gvis, int V, int D, int H, int W,
                                 cudaStream_t s) {
  dim3 grid(cdiv((long long)H * W, 8 * WC<C>::P));
  if (D <= WC<C>::DCH)
    warp_corr_aggregate_bwd_kernel<C, false><<<grid, 256, 0, s>>>(feat, homs, depth, vis, volume, gvol, gfeat, gvis, V, D, H, W);
  else
    warp_corr_aggregate_bwd_kernel<C, true><<<grid, 256, 0, s>>>(feat, homs, depth, vis, volume, gvol, gfeat, gvis, V, D, H, W);
}

}  // namespace mvsf

using namespace mvsf;

extern "C" int mvsf_warp_corr_aggregate_backward(const float* feat, const float* homs, const float* depth, const float* vis,
                                                 const float* volume, const float* grad_volume, float* grad_feat,
                                                 float* grad_vis, int V, int C, int G, int D, int H, int W,
                                                 mvsf_stream_t stream) {
  MVSF_REQUIRE(feat && homs && depth && vis && volume && grad_volume && grad_feat && grad_vis,
               "warp_corr_aggregate_backward: null pointer");
  MVSF_REQUIRE(V >= 2 && H > 0 && W > 0 && D >= 1, "warp_corr_aggregate_backward: bad shape");
  MVSF_REQUIRE(G <= C, "G must <= C!");
  MVSF_REQUIRE(G == 8 && (C == 8 || C == 16 || C == 32 || C == 64),
               "warp_corr_aggregate_backward: G must be 8 and C in 8/16/32/64");
  MVSF_REQUIRE(((uintptr_t)feat & 15) == 0 && ((uintptr_t)grad_feat & 15) == 0,
               "warp_corr_aggregate_backward: feat and grad_feat must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t view = (size_t)H * W * C;
  MVSF_CUDA_OK(cudaMemsetAsync(grad_feat + view, 0, sizeof(float) * view * (V - 1), s));
  switch (C) {
    case 8: launch_aggregate_bwd<8>(feat, homs, depth, vis, volume, grad_volume, grad_feat, grad_vis, V, D, H, W, s); break;
    case 16: launch_aggregate_bwd<16>(feat, homs, depth, vis, volume, grad_volume, grad_feat, grad_vis, V, D, H, W, s); break;
    case 32: launch_aggregate_bwd<32>(feat, homs, depth, vis, volume, grad_volume, grad_feat, grad_vis, V, D, H, W, s); break;
    default: launch_aggregate_bwd<64>(feat, homs, depth, vis, volume, grad_volume, grad_feat, grad_vis, V, D, H, W, s); break;
  }
  MVSF_LAUNCH_CHECK("warp_corr_aggregate_backward");
  return MVSF_OK;
}
