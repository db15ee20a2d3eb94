// W1 projection prep, F5/F6 hypothesis scheduling, F7 3-D positions, S1 soft-argmax, S2 confidence glue.
// All HBM-bound element-wise kernels: one thread per output pixel, depth-major planes so that a warp reads /
// writes 128 contiguous bytes per plane.
#include <float.h>

#include "common.cuh"

namespace mvsf {

// ------------------------------------------------------------------------------------------------
// W1: models/cost_volume.py:68-71 (P = E; P[:3,:4] = K @ E[:3,:4]) and models/warping.py:80-82
// (proj = P_src @ inverse(P_ref)).  Evaluated in fp64 (the reference uses fp32 LAPACK; the difference is
// ~1e-5 px, below the fp32 noise of the per-pixel coordinates themselves - DESIGN.md "Numerics").
// ------------------------------------------------------------------------------------------------
__device__ void compose_P(const float* pm, double P[16]) {
  const float* E = pm;        // [4][4]
  const float* K = pm + 16;   // [4][4], [:3,:3] used
  for (int i = 0; i < 16; ++i) P[i] = (double)E[i];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += (double)K[r * 4 + k] * (double)E[k * 4 + c];
      P[r * 4 + c] = s;
    }
}
__global__ void compose_geometry_kernel(const float* __restrict__ proj, int V, float* __restrict__ homs,
                                        float* __restrict__ kinv) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;  // 0 .. V-1 ; thread 0 also writes kinv
  if (v >= V) return;
  double Pref[16], Pinv[16];
  compose_P(proj, Pref);
  bool ok = invert4(Pref, Pinv);
  if (v == 0) {
    // inverse of the reference intrinsic K (3x3) by cofactors, fp64
    const float* K = proj + 16;
    double k[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) k[r * 3 + c] = (double)K[r * 4 + c];
    double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6]);
    double id = 1.0 / det;
    kinv[0] = (float)((k[4] * k[8] - k[5] * k[7]) * id);
    kinv[1] = (float)((k[2] * k[7] - k[1] * k[8]) * id);
    kinv[2] = (float)((k[1] * k[5] - k[2] * k[4]) * id);
    kinv[3] = (float)((k[5] * k[6] - k[3] * k[8]) * id);
    kinv[4] = (float)((k[0] * k[8] - k[2] * k[6]) * id);
    kinv[5] = (float)((k[2] * k[3] - k[0] * k[5]) * id);
    kinv[6] = (float)((k[3] * k[7] - k[4] * k[6]) * id);
    kinv[7] = (float)((k[1] * k[6] - k[0] * k[7]) * id);
    kinv[8] = (float)((k[0] * k[4] - k[1] * k[3]) * id);
    return;
  }
  double Ps[16];
  compose_P(proj + (size_t)v * 32, Ps);
  float* h = homs + (size_t)(v - 1) * 12;
  const double nanv = __longlong_as_double(0x7ff8000000000000LL);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += Ps[r * 4 + k] * Pinv[k * 4 + c];
      if (!ok) s = nanv;  // singular reference projection: torch.inverse raises; we propagate NaN
      if (c < 3) h[r * 3 + c] = (float)s; else h[9 + r] = (float)s;
    }
  }
}

// models/warping.py:80-82 for already composed 4x4 projections (the warp seam's own arguments):
// hom = rot (9, row-major) | trans (3) of src_proj @ inverse(ref_proj), one thread per batch item
__global__ void homography_from_proj_kernel(const float* __restrict__ src_proj, const float* __restrict__ ref_proj, int B,
                                            float* __restrict__ homs) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double Pr[16], Pi[16], Ps[16];
  for (int i = 0; i < 16; ++i) { Pr[i] = (double)ref_proj[b * 16 + i]; Ps[i] = (double)src_proj[b * 16 + i]; }
  const bool ok = invert4(Pr, Pi);
  const double nanv = __longlong_as_double(0x7ff8000000000000LL);
  float* h = homs + (size_t)b * 12;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += Ps[r * 4 + k] * Pi[k * 4 + c];
      if (!ok) s = nanv;
      if (c < 3) h[r * 3 + c] = (float)s; else h[9 + r] = (float)s;
    }
}

// ------------------------------------------------------------------------------------------------
// F5: models/module.py:692-704
// ------------------------------------------------------------------------------------------------
__global__ void init_inverse_range_kernel(const float* __restrict__ dv, int Dn, float* __restrict__ out, int D, int HW) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  float inv_min = __fdiv_rn(1.0f, __ldg(dv));
  float inv_max = __fdiv_rn(1.0f, __ldg(dv + Dn - 1));
  float diff = __fsub_rn(inv_min, inv_max);
  for (int k = 0; k < D; ++k) {
    float itv = __fdiv_rn((float)k, (float)(D - 1));
    float hypo = __fadd_rn(inv_max, __fmul_rn(diff, itv));
    out[(size_t)k * HW + p] = __fdiv_rn(1.0f, hypo);
  }
}

// ------------------------------------------------------------------------------------------------
// F6: models/module.py:707-724.  The trilinear x2 upsample (align_corners=True) has scale 1 along D, so it
// is a bilinear blend of the 4 half-resolution neighbours; hypotheses at the 4 neighbours are formed
// exactly as the reference forms them at half resolution.
// ------------------------------------------------------------------------------------------------
__global__ void schedule_inverse_range_kernel(const float* __restrict__ depth, const float* __restrict__ hypo,
                                              float split, float* __restrict__ out, int D, int H, int W) {
  const int h = H / 2, w = W / 2, hw = h * w;
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  if (x >= W) return;
  float sh = (H > 1) ? __fdiv_rn((float)(h - 1), (float)(H - 1)) : 0.0f;
  float sw = (W > 1) ? __fdiv_rn((float)(w - 1), (float)(W - 1)) : 0.0f;
  float fy = __fmul_rn(sh, (float)y), fx = __fmul_rn(sw, (float)x);
  int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
  int y1 = y0 + ((y0 < h - 1) ? 1 : 0), x1 = x0 + ((x0 < w - 1) ? 1 : 0);
  float ly1 = fy - (float)y0, lx1 = fx - (float)x0;
  float ly0 = 1.0f - ly1, lx0 = 1.0f - lx1;
  int idx[4] = {y0 * w + x0, y0 * w + x1, y1 * w + x0, y1 * w + x1};
  float imax[4], idiff[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float itv = __fsub_rn(__fdiv_rn(1.0f, __ldg(hypo + 2 * (size_t)hw + idx[c])),
                          __fdiv_rn(1.0f, __ldg(hypo + 1 * (size_t)hw + idx[c])));
    float invd = __fdiv_rn(1.0f, __ldg(depth + idx[c]));
    float s = __fmul_rn(split, itv);
    float imin = __fadd_rn(invd, s);
    imax[c] = __fsub_rn(invd, s);
    idiff[c] = __fsub_rn(imin, imax[c]);
  }
  size_t HW = (size_t)H * W;
  size_t o = (size_t)y * W + x;
  for (int k = 0; k < D; ++k) {
    float itv = __fdiv_rn((float)k, (float)(D - 1));
    float v00 = __fadd_rn(imax[0], __fmul_rn(idiff[0], itv));
    float v01 = __fadd_rn(imax[1], __fmul_rn(idiff[1], itv));
    float v10 = __fadd_rn(imax[2], __fmul_rn(idiff[2], itv));
    float v11 = __fadd_rn(imax[3], __fmul_rn(idiff[3], itv));
    float top = lx0 * v00 + lx1 * v01;
    float bot = lx0 * v10 + lx1 * v11;
    float v = ly0 * top + ly1 * bot;
    out[(size_t)k * HW + o] = __fdiv_rn(1.0f, v);
  }
}

// ------------------------------------------------------------------------------------------------
// F7: models/position_encoding.py:138-161
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned enc_f(float f) {
  unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__global__ void pos3d_init_kernel(unsigned* stats_u) {
  stats_u[0] = enc_f(FLT_MAX);   // width_min
  stats_u[1] = enc_f(-FLT_MAX);  // width_max
  stats_u[2] = enc_f(FLT_MAX);   // height_min
  stats_u[3] = enc_f(-FLT_MAX);  // height_max
}
__global__ void pos3d_minmax_kernel(const float* __restrict__ kinv, const float* __restrict__ depth, unsigned* stats_u,
                                    int D, int H, int W) {
  const int HW = H * W;
  float k00 = kinv[0], k01 = kinv[1], k02 = kinv[2], k10 = kinv[3], k11 = kinv[4], k12 = kinv[5];
  float xmin = FLT_MAX, xmax = -FLT_MAX, ymin = FLT_MAX, ymax = -FLT_MAX;
  size_t total = (size_t)D * HW;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int p = (int)(i % HW);
    int y = p / W, x = p - y * W;
    float d = __ldg(depth + i);
    float ax = __fadd_rn(fmaf(k01, (float)y, __fmul_rn(k00, (float)x)), k02);
    float ay = __fadd_rn(fmaf(k11, (float)y, __fmul_rn(k10, (float)x)), k12);
    float px = __fmul_rn(ax, d), py = __fmul_rn(ay, d);
    xmin = fminf(xmin, px); xmax = fmaxf(xmax, px);
    ymin = fminf(ymin, py); ymax = fmaxf(ymax, py);
  }
  for (int o = 16; o > 0; o >>= 1) {
    xmin = fminf(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
    xmax = fmaxf(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
    ymin = fminf(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    ymax = fmaxf(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(stats_u + 0, enc_f(xmin));
    atomicMax(stats_u + 1, enc_f(xmax));
    atomicMin(stats_u + 2, enc_f(ymin));
    atomicMax(stats_u + 3, enc_f(ymax));
  }
}
__global__ void pos3d_finalize_kernel(float* stats, const float* __restrict__ dv, int Dn, int decode) {
  // single warp: decode the 4 extents in place, and depth_values.min()/max() (DINOv2_mvsformer_model.py:156)
  if (decode && threadIdx.x < 4) {
    unsigned u = reinterpret_cast<unsigned*>(stats)[threadIdx.x];
    stats[threadIdx.x] = dec_f(u);
  }
  float mn = FLT_MAX, mx = -FLT_MAX;
  for (int i = threadIdx.x; i < Dn; i += 32) { float v = dv[i]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (threadIdx.x == 0) { stats[4] = mn; stats[5] = mx; }
}
__global__ void pos3d_normalize_kernel(const float* __restrict__ kinv, const float* __restrict__ depth,
                                       const float* __restrict__ stats, float* __restrict__ pos, int D, int H, int W) {
  const int HW = H * W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  int y = p / W, x = p - y * W;
  float wmin = stats[0], wmax = stats[1], hmin = stats[2], hmax = stats[3], dmin = stats[4], dmax = stats[5];
  float ax = __fadd_rn(fmaf(kinv[1], (float)y, __fmul_rn(kinv[0], (float)x)), kinv[2]);
  float ay = __fadd_rn(fmaf(kinv[4], (float)y, __fmul_rn(kinv[3], (float)x)), kinv[5]);
  float az = __fadd_rn(fmaf(kinv[7], (float)y, __fmul_rn(kinv[6], (float)x)), kinv[8]);
  float wden = __fadd_rn(__fsub_rn(wmax, wmin), 1e-5f);
  float hden = __fadd_rn(__fsub_rn(hmax, hmin), 1e-5f);
  float dden = __fadd_rn(__fsub_rn(dmax, dmin), 1e-5f);
  size_t DHW = (size_t)D * HW;
  for (int d = 0; d < D; ++d) {
    float dv = __ldg(depth + (size_t)d * HW + p);
    float px = __fmul_rn(ax, dv), py = __fmul_rn(ay, dv), pz = __fmul_rn(az, dv);
    size_t o = (size_t)d * HW + p;
    pos[o] = __fdiv_rn(__fsub_rn(px, wmin), wden);
    pos[DHW + o] = __fdiv_rn(__fsub_rn(py, hmin), hden);
    float zc = fminf(fmaxf(pz, dmin), dmax);
    pos[2 * DHW + o] = __fdiv_rn(__fsub_rn(zc, dmin), dden);
  }
}

// ------------------------------------------------------------------------------------------------
// S1: models/cost_volume.py:105-117, models/module.py:649-655
// ------------------------------------------------------------------------------------------------
template <int DT>
__global__ void softargmax_kernel(const float* __restrict__ logits, const float* __restrict__ hypo, float tmp,
                                  float* __restrict__ prob, float* __restrict__ depth, float* __restrict__ conf, int D,
                                  int HW) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  if (DT > 0) {
    float z[DT > 0 ? DT : 1];
    float m = -FLT_MAX;
#pragma unroll
    for (int d = 0; d < DT; ++d) { z[d] = __ldg(logits + (size_t)d * HW + p); m = fmaxf(m, z[d]); }
    float s = 0.f, st = 0.f, mt = m * tmp;
    if (tmp < 0.f) {  // max of z*tmp is min(z)*tmp for negative temperature; handle generally
      mt = -FLT_MAX;
#pragma unroll
      for (int d = 0; d < DT; ++d) mt = fmaxf(mt, z[d] * tmp);
    }
    float e[DT > 0 ? DT : 1];
#pragma unroll
    for (int d = 0; d < DT; ++d) { e[d] = expf(z[d] - m); s += e[d]; }
    float pm = 0.f, acc = 0.f;
    float et[DT > 0 ? DT : 1];
#pragma unroll
    for (int d = 0; d < DT; ++d) { et[d] = expf(__fmul_rn(z[d], tmp) - mt); st += et[d]; }
#pragma unroll
    for (int d = 0; d < DT; ++d) {
      float pr = __fdiv_rn(e[d], s);
      prob[(size_t)d * HW + p] = pr;
      pm = fmaxf(pm, pr);
      acc += __fdiv_rn(et[d], st) * __ldg(hypo + (size_t)d * HW + p);
    }
    depth[p] = acc;
    conf[p] = pm;
  } else {
    float m = -FLT_MAX, mt = -FLT_MAX;
    for (int d = 0; d < D; ++d) {
      float z = __ldg(logits + (size_t)d * HW + p);
      m = fmaxf(m, z);
      mt = fmaxf(mt, __fmul_rn(z, tmp));
    }
    float s = 0.f, st = 0.f;
    for (int d = 0; d < D; ++d) {
      float z = __ldg(logits + (size_t)d * HW + p);
      s += expf(z - m);
      st += expf(__fmul_rn(z, tmp) - mt);
    }
    float pm = 0.f, acc = 0.f;
    for (int d = 0; d < D; ++d) {
      float z = __ldg(logits + (size_t)d * HW + p);
      float pr = __fdiv_rn(expf(z - m), s);
      prob[(size_t)d * HW + p] = pr;
      pm = fmaxf(pm, pr);
      acc += __fdiv_rn(expf(__fmul_rn(z, tmp) - mt), st) * __ldg(hypo + (size_t)d * HW + p);
    }
    depth[p] = acc;
    conf[p] = pm;
  }
}

// S2: DINOv2_mvsformer_model.py:167-172 (nearest upsample: src = floor(dst * in/out))
__global__ void conf_accumulate_kernel(const float* __restrict__ conf, int h, int w, float* __restrict__ acc, int H,
                                       int W, float scale, int init) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y;
  if (x >= W) return;
  float sy = (float)h / (float)H, sx = (float)w / (float)W;
  int yy = min((int)floorf((float)y * sy), h - 1), xx = min((int)floorf((float)x * sx), w - 1);
  float v = __ldg(conf + (size_t)yy * w + xx) * scale;
  size_t o = (size_t)y * W + x;
  acc[o] = init ? v : acc[o] + v;
}

}  // namespace mvsf

using namespace mvsf;

extern "C" {

int mvsf_compose_geometry(const float* proj, int V, float* homs, float* kinv_ref, mvsf_stream_t stream) {
  MVSF_REQUIRE(proj && homs && kinv_ref && V >= 2 && V <= 64, "compose_geometry: need 2 <= V <= 64 views");
  compose_geometry_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(proj, V, homs, kinv_ref);
  MVSF_LAUNCH_CHECK("compose_geometry");
  return MVSF_OK;
}

int mvsf_homography_from_proj(const float* src_proj, const float* ref_proj, int B, float* homs, mvsf_stream_t stream) {
  MVSF_REQUIRE(src_proj && ref_proj && homs && B > 0, "homography_from_proj: bad arguments");
  homography_from_proj_kernel<<<cdiv(B, 32), 32, 0, (cudaStream_t)stream>>>(src_proj, ref_proj, B, homs);
  MVSF_LAUNCH_CHECK("homography_from_proj");
  return MVSF_OK;
}

int mvsf_init_inverse_range(const float* depth_values, int Dn, float* out, int D, int H, int W, mvsf_stream_t stream) {
  MVSF_REQUIRE(depth_values && out && Dn >= 2 && D >= 2 && H > 0 && W > 0, "init_inverse_range: bad arguments");
  int HW = H * W;
  init_inverse_range_kernel<<<cdiv(HW, 256), 256, 0, (cudaStream_t)stream>>>(depth_values, Dn, out, D, HW);
  MVSF_LAUNCH_CHECK("init_inverse_range");
  return MVSF_OK;
}

int mvsf_schedule_inverse_range(const float* prev_depth, const float* prev_hypo, int Dp, float split_itv, float* out,
                                int D, int H, int W, mvsf_stream_t stream) {
  MVSF_REQUIRE(prev_depth && prev_hypo && out && D >= 2 && H >= 2 && W >= 2 && (H % 2 == 0) && (W % 2 == 0),
               "schedule_inverse_range: H, W must be even and D >= 2");
  MVSF_REQUIRE(Dp >= 3, "schedule_inverse_range: previous stage needs >= 3 hypotheses (reference reads [:,1] and [:,2])");
  dim3 grid(cdiv(W, 128), H);
  schedule_inverse_range_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(prev_depth, prev_hypo, split_itv, out, D, H, W);
  MVSF_LAUNCH_CHECK("schedule_inverse_range");
  return MVSF_OK;
}

int mvsf_position3d(const float* kinv_ref, const float* depth, const float* depth_values, int Dn, float* stats,
                    int compute_minmax, float* pos, int D, int H, int W, mvsf_stream_t stream) {
  // compute_minmax: 1 = extents of this sample + depth range, then normalise (B == 1, first stage that uses the PE)
  //                 0 = reuse the decoded extents in `stats`, refresh the depth range from depth_values, normalise
  //   batched callers (the reference reduces the extents and depth_values.min()/max() over the whole batch,
  //   position_encoding.py:152-157, DINOv2_mvsformer_model.py:156): 2 = reset + accumulate extents, 3 = accumulate,
  //   4 = decode extents + depth range of depth_values[0..Dn) (pass the whole [B,Dn] block), 5 = normalise only
  const int mode = compute_minmax;
  MVSF_REQUIRE(mode >= 0 && mode <= 5 && stats && D >= 1 && H > 0 && W > 0, "position3d: bad arguments");
  MVSF_REQUIRE(mode == 4 || (kinv_ref && depth), "position3d: null kinv / depth");
  MVSF_REQUIRE((mode != 0 && mode != 1 && mode != 4) || (depth_values && Dn >= 1), "position3d: null depth_values");
  MVSF_REQUIRE((mode != 0 && mode != 1 && mode != 5) || pos, "position3d: null output");
  cudaStream_t s = (cudaStream_t)stream;
  if (mode == 1 || mode == 2) {
    pos3d_init_kernel<<<1, 1, 0, s>>>(reinterpret_cast<unsigned*>(stats));
    MVSF_LAUNCH_CHECK("pos3d_init");
  }
  if (mode == 1 || mode == 2 || mode == 3) {
    size_t total = (size_t)D * H * W;
    int blocks = (int)((total + 255) / 256);
    const int cap = device_sm_count(current_device()) * 8;
    if (blocks > cap) blocks = cap;
    pos3d_minmax_kernel<<<blocks, 256, 0, s>>>(kinv_ref, depth, reinterpret_cast<unsigned*>(stats), D, H, W);
    MVSF_LAUNCH_CHECK("pos3d_minmax");
  }
  if (mode == 0 || mode == 1 || mode == 4) {
    pos3d_finalize_kernel<<<1, 32, 0, s>>>(stats, depth_values, Dn, mode != 0);
    MVSF_LAUNCH_CHECK("pos3d_finalize");
  }
  if (mode == 0 || mode == 1 || mode == 5) {
    pos3d_normalize_kernel<<<cdiv(H * W, 256), 256, 0, s>>>(kinv_ref, depth, stats, pos, D, H, W);
    MVSF_LAUNCH_CHECK("pos3d_normalize");
  }
  return MVSF_OK;
}

int mvsf_softargmax(const float* logits, const float* depth_hypo, float tmp, float* prob, float* depth, float* conf,
                    int D, int H, int W, mvsf_stream_t stream) {
  MVSF_REQUIRE(logits && depth_hypo && prob && depth && conf && D >= 1 && H > 0 && W > 0, "softargmax: bad arguments");
  int HW = H * W;
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid(cdiv(HW, 256));
  switch (D) {
    case 4: softargmax_kernel<4><<<grid, 256, 0, s>>>(logits, depth_hypo, tmp, prob, depth, conf, D, HW); break;
    case 8: softargmax_kernel<8><<<grid, 256, 0, s>>>(logits, depth_hypo, tmp, prob, depth, conf, D, HW); break;
    case 16: softargmax_kernel<16><<<grid, 256, 0, s>>>(logits, depth_hypo, tmp, prob, depth, conf, D, HW); break;
    case 32: softargmax_kernel<32><<<grid, 256, 0, s>>>(logits, depth_hypo, tmp, prob, depth, conf, D, HW); break;
    default: softargmax_kernel<0><<<grid, 256, 0, s>>>(logits, depth_hypo, tmp, prob, depth, conf, D, HW); break;
  }
  MVSF_LAUNCH_CHECK("softargmax");
  return MVSF_OK;
}

int mvsf_conf_accumulate(const float* conf, int h, int w, float* acc, int H, int W, float scale, int init,
                         mvsf_stream_t stream) {
  MVSF_REQUIRE(conf && acc && h > 0 && w > 0 && H > 0 && W > 0, "conf_accumulate: bad arguments");
  dim3 grid(cdiv(W, 128), H);
  conf_accumulate_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(conf, h, w, acc, H, W, scale, init);
  MVSF_LAUNCH_CHECK("conf_accumulate");
  return MVSF_OK;
}
}
