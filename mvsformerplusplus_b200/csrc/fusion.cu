// Depth-map fusion: the pcd and dpcd consistency filters of the reference's test.py:387-517 over misc/fusion.py:79-165,
// and the ordered extraction of the surviving pixels as a coloured point cloud.
//
// One thread per reference pixel, a loop over the source views of that reference view, every intermediate in registers.
// The arithmetic is the reference's fp32 chain operation by operation (each product, sum and quotient rounded on its own:
// the __f*_rn intrinsics keep the compiler from contracting a product and a sum into an FMA), so a comparison against a
// threshold falls on the same side as in the torch restatement oracle/fusion.py, which spells out the same order.
// NaN and Inf propagate to "comparison false", as the reference relies on.
#include "common.cuh"

namespace mvsf {

constexpr int FUSION_MAX_SRC = 16;   // the dpcd vote counters of a pixel live in registers
constexpr int FUSION_BLOCK = 256;    // pixels per block = granularity of the survivor counts
constexpr int FUSION_SCAN_THREADS = 1024;

struct FusionSrc { int idx[FUSION_MAX_SRC]; };

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
constexpr float FUSION_EPS = 1e-9f;   // the "+ 1e-9" of every homogeneous divide (fusion.py:25,33,39,44,46)

// ------------------------------------------------------------------------------------------------
// fusion_prepare: per camera E^-1 (slot 0) and K^-1 (slot 1 [:3,:3]) in the layout of the cameras themselves, computed
// in fp64 and rounded once (the reference inverts in fp32 per pixel batch, fusion.py:24,32).  Singular: NaN.
// ------------------------------------------------------------------------------------------------
__global__ void fusion_prepare_kernel(const float* __restrict__ cams, int N, float* __restrict__ inv) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* E = cams + (size_t)n * 32;
  const float* K = E + 16;
  float* Ei = inv + (size_t)n * 32;
  float* Ki = Ei + 16;
  const double nanv = __longlong_as_double(0x7ff8000000000000LL);
  double A[16], B[16];
  for (int i = 0; i < 16; ++i) A[i] = (double)E[i];
  bool ok = invert4(A, B);
  for (int i = 0; i < 16; ++i) Ei[i] = (float)(ok ? B[i] : nanv);
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) A[r * 4 + c] = (r < 3 && c < 3) ? (double)K[r * 4 + c] : (r == c ? 1.0 : 0.0);
  ok = invert4(A, B);
  for (int i = 0; i < 16; ++i) Ki[i] = (float)(ok ? B[i] : nanv);
}

// ------------------------------------------------------------------------------------------------
// The reprojection chain: pixel (u, v) of camera a at depth d -> its image position (x, y) in camera b and its depth z
// there.  idx_img2cam, idx_cam2world (fusion.py:23-34) with a's inverses, idx_world2cam, idx_cam2img (:37-47) with b.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void img2world(const float* __restrict__ inv_a, float u, float v, float d, float w[4]) {
  const float* Ei = inv_a;
  const float* Ki = inv_a + 16;
  float c[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = add(add(mul(__ldg(Ki + i * 4), u), mul(__ldg(Ki + i * 4 + 1), v)), __ldg(Ki + i * 4 + 2));
  const float dc = add(c[2], FUSION_EPS);
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = mul(dvd(c[i], dc), d);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] = add(add(add(mul(__ldg(Ei + i * 4), c[0]), mul(__ldg(Ei + i * 4 + 1), c[1])), mul(__ldg(Ei + i * 4 + 2), c[2])),
               __ldg(Ei + i * 4 + 3));
  const float dw = add(w[3], FUSION_EPS);
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = dvd(w[i], dw);
}

__device__ __forceinline__ void reproject(const float* __restrict__ inv_a, const float* __restrict__ cam_b, float u, float v,
                                          float d, float& x, float& y, float& z) {
  float w[4], q[4], r[3], im[3];
  img2world(inv_a, u, v, d, w);
  const float* E = cam_b;
  const float* K = cam_b + 16;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    q[i] = add(add(add(mul(__ldg(E + i * 4), w[0]), mul(__ldg(E + i * 4 + 1), w[1])), mul(__ldg(E + i * 4 + 2), w[2])),
               mul(__ldg(E + i * 4 + 3), w[3]));
  const float dq = add(q[3], FUSION_EPS);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = dvd(q[i], dq);
  const float dr = add(q[3], FUSION_EPS);
#pragma unroll
  for (int i = 0; i < 3; ++i) r[i] = dvd(q[i], dr);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    im[i] = add(add(mul(__ldg(K + i * 4), r[0]), mul(__ldg(K + i * 4 + 1), r[1])), mul(__ldg(K + i * 4 + 2), r[2]));
  const float di = add(im[2], FUSION_EPS);
  x = dvd(im[0], di);
  y = dvd(im[1], di);
  z = q[2];
}

// grid_sample(align_corners=True) un-normalisation and the bilinear corner weights (NaN stays NaN)
struct Bilinear {
  float x0, y0, wx0, wx1, wy0, wy1;
  __device__ __forceinline__ Bilinear(float gx, float gy, int H, int W) {
    const float ix = mul(dvd(add(gx, 1.0f), 2.0f), (float)(W - 1));
    const float iy = mul(dvd(add(gy, 1.0f), 2.0f), (float)(H - 1));
    x0 = floorf(ix);
    y0 = floorf(iy);
    wx1 = sub(ix, x0);
    wx0 = sub(add(x0, 1.0f), ix);
    wy1 = sub(iy, y0);
    wy0 = sub(add(y0, 1.0f), iy);
  }
  // corner k = 0 nw, 1 ne, 2 sw, 3 se: its pixel, whether it lies in the map (zero padding otherwise), its weight
  __device__ __forceinline__ bool corner(int k, int H, int W, int& cx, int& cy, float& wgt) const {
    const float fx = (k & 1) ? add(x0, 1.0f) : x0, fy = (k & 2) ? add(y0, 1.0f) : y0;
    wgt = mul((k & 1) ? wx1 : wx0, (k & 2) ? wy1 : wy0);
    const bool in = fx >= 0.0f && fx <= (float)(W - 1) && fy >= 0.0f && fy <= (float)(H - 1);
    cx = in ? (int)fx : 0;
    cy = in ? (int)fy : 0;
    return in;
  }
};

__device__ __forceinline__ float clamp_keep_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

// mask, averaged depth and the block's survivor count
__device__ __forceinline__ void fusion_store(bool inside, bool keep, float avg, int p, unsigned char* __restrict__ mask,
                                             float* __restrict__ depth_avg, int* __restrict__ block_counts) {
  if (inside) {
    mask[p] = keep ? 1 : 0;
    depth_avg[p] = avg;
  }
  const int n = __syncthreads_count(inside && keep);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = n;
}

// ------------------------------------------------------------------------------------------------
// pcd: filter_depth, test.py:395-412 (get_reproj + vis_filter + ave_fusion, fusion.py:79-112).  The reference stages the
// source -> reference reprojection of every source pixel as a 3-channel map and samples it; here it is evaluated at the
// four corners the sample touches.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FUSION_BLOCK)
fusion_pcd_kernel(const float* __restrict__ depths, const float* __restrict__ confs, const float* __restrict__ cams,
                  const float* __restrict__ cams_inv, int ref, const __grid_constant__ FusionSrc src, int V, int H, int W, float conf,
                  float thres_view, float thres_disp, unsigned char* __restrict__ mask, float* __restrict__ depth_avg,
                  int* __restrict__ block_counts) {
  const int HW = H * W;
  const int p = blockIdx.x * FUSION_BLOCK + threadIdx.x;
  const bool inside = p < HW;
  bool keep = false;
  float avg = 0.0f;
  if (inside) {
    const int py = p / W, px = p - py * W;
    const float u = add((float)px, 0.5f), v = add((float)py, 0.5f);
    const float d_ref = __ldg(depths + (size_t)ref * HW + p);
    float sum = 0.0f, cnt = 0.0f;
    for (int s = 0; s < V; ++s) {
      const int sv = src.idx[s];
      const float* ds = depths + (size_t)sv * HW;
      const float* cs = confs + (size_t)sv * HW;
      float wx, wy, wz;
      reproject(cams_inv + (size_t)ref * 32, cams + (size_t)sv * 32, u, v, d_ref, wx, wy, wz);
      // project_img, fusion.py:58-64: normalised by the size, sampled with align_corners=True (the reference's mismatch)
      const float gx = clamp_keep_nan(sub(mul(dvd(wx, (float)W), 2.0f), 1.0f), -1.1f, 1.1f);
      const float gy = clamp_keep_nan(sub(mul(dvd(wy, (float)H), 2.0f), 1.0f), -1.1f, 1.1f);
      const bool in_range = -1.0f <= gx && gx <= 1.0f && -1.0f <= gy && gy <= 1.0f;
      const Bilinear b(gx, gy, H, W);
      float bx = 0.0f, by = 0.0f, bd = 0.0f;
#pragma unroll 1
      for (int k = 0; k < 4; ++k) {
        int cx, cy;
        float wgt;
        if (!b.corner(k, H, W, cx, cy, wgt)) continue;
        const int q = cy * W + cx;
        // test.py:397-400: source depths are zeroed where the source confidence does not exceed the threshold
        const float d = mul(__ldg(ds + q), __ldg(cs + q) > conf ? 1.0f : 0.0f);
        float rx, ry, rz;
        reproject(cams_inv + (size_t)sv * 32, cams + (size_t)ref * 32, add((float)cx, 0.5f), add((float)cy, 0.5f), d, rx, ry, rz);
        bx = add(bx, mul(rx, wgt));
        by = add(by, mul(ry, wgt));
        bd = add(bd, mul(rz, wgt));
      }
      const float dx = sub(bx, u), dy = sub(by, v);
      const bool close_xy = sqrtf(add(mul(dx, dx), mul(dy, dy))) < thres_disp;
      const bool same = fabsf(sub(d_ref, bd)) < mul(fmaxf(d_ref, bd), 0.01f);   // a NaN depth fails on the left side
      const float m = (in_range && close_xy && same) ? 1.0f : 0.0f;
      sum = add(sum, mul(bd, m));   // ave_fusion multiplies by the mask: a NaN depth poisons the average as it does there
      cnt = add(cnt, m);
    }
    const bool vis = (double)cnt >= (double)thres_view - 1.1;   // fusion.py:106
    avg = dvd(add(sum, d_ref), add(cnt, 1.0f));
    keep = vis && __ldg(confs + (size_t)ref * HW + p) > conf;
  }
  fusion_store(inside, keep, avg, p, mask, depth_avg, block_counts);
}

// ------------------------------------------------------------------------------------------------
// dpcd: dynamic_filter_depth, test.py:453-483 (get_reproj_dynamic + vis_filter_dynamic, fusion.py:114-165).  The
// [V][V-1][H][W] threshold masks are V-1 counters per pixel.  With one source view there is no threshold (the reference
// fails on the empty mask): no pixel is accepted and the averaged depth is the reference depth.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FUSION_BLOCK)
fusion_dpcd_kernel(const float* __restrict__ depths, const float* __restrict__ confs, const float* __restrict__ cams,
                   const float* __restrict__ cams_inv, int ref, const __grid_constant__ FusionSrc src, int V, int H, int W, float conf,
                   float dist_base, float rel_diff_base, unsigned char* __restrict__ mask, float* __restrict__ depth_avg,
                   int* __restrict__ block_counts) {
  const int HW = H * W;
  const int p = blockIdx.x * FUSION_BLOCK + threadIdx.x;
  const bool inside = p < HW;
  bool keep = false;
  float avg = 0.0f;
  if (inside) {
    const int py = p / W, px = p - py * W;
    const float u = add((float)px, 0.5f), v = add((float)py, 0.5f);
    const float d_ref = __ldg(depths + (size_t)ref * HW + p);
    const float half_w = dvd((float)(W - 1), 2.0f), half_h = dvd((float)(H - 1), 2.0f);
    int votes[FUSION_MAX_SRC - 1];
#pragma unroll
    for (int j = 0; j < FUSION_MAX_SRC - 1; ++j) votes[j] = 0;
    float sum = 0.0f;
    int cnt_last = 0;
    for (int s = 0; s < V; ++s) {
      const int sv = src.idx[s];
      const float* ds = depths + (size_t)sv * HW;
      float wx, wy, wz;
      reproject(cams_inv + (size_t)ref * 32, cams + (size_t)sv * 32, u, v, d_ref, wx, wy, wz);
      const Bilinear b(sub(dvd(wx, half_w), 1.0f), sub(dvd(wy, half_h), 1.0f), H, W);
      float d = 0.0f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        int cx, cy;
        float wgt;
        if (b.corner(k, H, W, cx, cy, wgt)) d = add(d, mul(__ldg(ds + cy * W + cx), wgt));
      }
      float rx, ry, rz;
      reproject(cams_inv + (size_t)sv * 32, cams + (size_t)ref * 32, wx, wy, d, rx, ry, rz);
      const float dx = sub(rx, u), dy = sub(ry, v);
      const float dist = sqrtf(add(mul(dx, dx), mul(dy, dy)));
      const float rel = dvd(fabsf(sub(d_ref, rz)), d_ref);
#pragma unroll
      for (int j = 0; j < FUSION_MAX_SRC - 1; ++j) {
        const float i = (float)(j + 2);
        const bool ok = j < V - 1 && dist < dvd(i, dist_base) && rel < dvd(i, rel_diff_base);
        votes[j] += ok ? 1 : 0;
        if (j == V - 2 && ok) {   // the loosest threshold selects what is averaged (test.py:471-475)
          sum = add(sum, rz);
          cnt_last += 1;
        }
      }
    }
    bool geo = false;   // test.py:476's "sum >= V + 1" can never hold
#pragma unroll
    for (int j = 0; j < FUSION_MAX_SRC - 1; ++j) geo = geo || (j < V - 1 && votes[j] >= j + 2);
    avg = dvd(add(sum, d_ref), (float)(cnt_last + 1));
    keep = geo && __ldg(confs + (size_t)ref * HW + p) > conf;
  }
  fusion_store(inside, keep, avg, p, mask, depth_avg, block_counts);
}

// ------------------------------------------------------------------------------------------------
// Ordered extraction: exclusive scan of the block counts (one CTA; in place, the total goes to counts[n]), then every
// block writes its survivors at offset[block] + rank within the block, so points come out in row-major pixel order.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FUSION_SCAN_THREADS) fusion_scan_kernel(int* __restrict__ counts, int n) {
  __shared__ int warp_sums[FUSION_SCAN_THREADS / 32];
  const int t = threadIdx.x, per = (n + FUSION_SCAN_THREADS - 1) / FUSION_SCAN_THREADS;
  const int lo = min(t * per, n), hi = min(lo + per, n);
  int mine = 0;
  for (int i = lo; i < hi; ++i) mine += counts[i];
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += y;
  }
  if ((t & 31) == 31) warp_sums[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    int ws = warp_sums[t];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, ws, o);
      if (t >= o) ws += y;
    }
    warp_sums[t] = ws;
  }
  __syncthreads();
  int run = incl - mine + ((t >> 5) ? warp_sums[(t >> 5) - 1] : 0);
  for (int i = lo; i < hi; ++i) {
    const int c = counts[i];
    counts[i] = run;
    run += c;
  }
  if (t == FUSION_SCAN_THREADS - 1) counts[n] = warp_sums[FUSION_SCAN_THREADS / 32 - 1];
}

__global__ void __launch_bounds__(FUSION_BLOCK)
fusion_extract_kernel(const unsigned char* __restrict__ mask, const float* __restrict__ depth_avg,
                      const int* __restrict__ offsets, const float* __restrict__ cam_inv, const float* __restrict__ image,
                      float* __restrict__ xyz, unsigned char* __restrict__ rgb, long long capacity, int H, int W) {
  __shared__ int warp_base[FUSION_BLOCK / 32];
  const int HW = H * W;
  const int p = blockIdx.x * FUSION_BLOCK + threadIdx.x;
  const bool keep = p < HW && mask[p] != 0;
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_base[warp] = __popc(bal);
  __syncthreads();
  if (!keep) return;
  long long pos = offsets[blockIdx.x] + __popc(bal & ((1u << lane) - 1u));
  for (int w = 0; w < warp; ++w) pos += warp_base[w];
  if (pos >= capacity) return;
  const int py = p / W, px = p - py * W;
  float w[4];
  img2world(cam_inv, add((float)px, 0.5f), add((float)py, 0.5f), depth_avg[p], w);   // test.py:410-412
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    xyz[pos * 3 + k] = w[k];
    rgb[pos * 3 + k] = (unsigned char)mul(__ldg(image + (size_t)k * HW + p), 255.0f);   // astype(np.uint8), test.py:422-424
  }
}

static size_t fusion_ws_bytes(int H, int W) { return ((size_t)cdiv((long long)H * W, FUSION_BLOCK) + 1) * sizeof(int); }

// ------------------------------------------------------------------------------------------------
// gipuma: the cross-view voting and point averaging of fusibile, the fusion misc/gipuma.py:208-228 runs as an external
// binary (probability_filter, P = [K|0] E, fusibile at normal_thresh = 360 with constant normals, which makes the
// normal test vacuous).  Reference views are processed one at a time in index order; a view's step reads only its own
// used marks and sets only other views' marks, so every step is race-free and deterministic.
//
// Camera table: GIPUMA_CAM floats per view (128 bytes, 64-bit offsets, read through the L1 from global memory, so the
// number of views is bounded only by int N and memory): [0, 12) P = K E[:3, :] row-major, [12, 21) M^-1 (M = P[:, :3])
// row-major, [21] f b with f = K[0][0] / K[2][2] and b = 0.54; all computed in fp64 and rounded once.
// ------------------------------------------------------------------------------------------------
constexpr int GIPUMA_CAM = 32;
constexpr double GIPUMA_BASELINE = 0.54;   // fusibile's fixed baseline

__global__ void gipuma_cameras_kernel(const float* __restrict__ cams, int N, float* __restrict__ table) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* E = cams + (size_t)n * 32;
  const float* K = E + 16;
  float* t = table + (size_t)n * GIPUMA_CAM;
  const double nanv = __longlong_as_double(0x7ff8000000000000LL);
  double P[12], A[16], B[16];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      P[r * 4 + c] = __dadd_rn(__dadd_rn(__dmul_rn(K[r * 4], E[c]), __dmul_rn(K[r * 4 + 1], E[4 + c])), __dmul_rn(K[r * 4 + 2], E[8 + c]));
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) A[r * 4 + c] = (r < 3 && c < 3) ? P[r * 4 + c] : (r == c ? 1.0 : 0.0);
  const bool ok = invert4(A, B);
  for (int i = 0; i < 12; ++i) t[i] = (float)P[i];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) t[12 + r * 3 + c] = (float)(ok ? B[r * 4 + c] : nanv);
  t[21] = (float)__dmul_rn(__ddiv_rn(K[0], K[10]), GIPUMA_BASELINE);
  for (int i = 22; i < GIPUMA_CAM; ++i) t[i] = 0.0f;
}

// probability_filter (misc/gipuma.py:160-177) and fusibile's depth range: depth where conf > prob_threshold and
// depth_min <= depth <= depth_max, else 0 (a NaN fails every comparison)
__global__ void gipuma_depth_kernel(const float* __restrict__ depths, const float* __restrict__ confs, long long n, float prob,
                                    float dmin, float dmax, float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float d = __ldg(depths + i);
    out[i] = (__ldg(confs + i) > prob && d >= dmin && d <= dmax) ? d : 0.0f;
  }
}

// pixel (x, y) at depth d -> world point X = M^-1 (d x - p4.x, d y - p4.y, d - p4.z)
__device__ __forceinline__ void gipuma_unproject(const float* __restrict__ cam, float x, float y, float d, float X[3]) {
  const float a0 = sub(mul(d, x), __ldg(cam + 3)), a1 = sub(mul(d, y), __ldg(cam + 7)), a2 = sub(d, __ldg(cam + 11));
#pragma unroll
  for (int i = 0; i < 3; ++i)
    X[i] = add(add(mul(__ldg(cam + 12 + i * 3), a0), mul(__ldg(cam + 13 + i * 3), a1)), mul(__ldg(cam + 14 + i * 3), a2));
}

// One probe: world point X of the reference pixel into source view s.  True iff it lands in the image on a valid source
// pixel q whose disparity f_r b / D_s(q) is within disp of f_r b / z; q and D_s(q) are returned.
__device__ __forceinline__ bool gipuma_probe(const float* __restrict__ cam_s, const float* __restrict__ depth_s, const float X[3],
                                             float fb, float disp, int H, int W, int& q, float& ds) {
  float t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    t[i] = add(add(add(mul(__ldg(cam_s + i * 4), X[0]), mul(__ldg(cam_s + i * 4 + 1), X[1])), mul(__ldg(cam_s + i * 4 + 2), X[2])),
               __ldg(cam_s + i * 4 + 3));
  const float xs = dvd(t[0], t[2]), ys = dvd(t[1], t[2]);
  if (!(xs >= 0.0f && xs < (float)W && ys >= 0.0f && ys < (float)H)) return false;
  q = (int)floorf(ys) * W + (int)floorf(xs);
  ds = __ldg(depth_s + q);
  return ds > 0.0f && fabsf(sub(dvd(fb, t[2]), dvd(fb, ds))) < disp;
}

// vote: the number of consistent source views of every valid, unused pixel of reference view r -> mask (n >= num_consistent)
// and the block survivor counts
__global__ void __launch_bounds__(FUSION_BLOCK)
gipuma_vote_kernel(const float* __restrict__ depth, const unsigned char* __restrict__ used, const float* __restrict__ table, int N,
                   int ref, int H, int W, float disp, int num_consistent, unsigned char* __restrict__ mask,
                   int* __restrict__ block_counts) {
  const int HW = H * W;
  const int p = blockIdx.x * FUSION_BLOCK + threadIdx.x;
  const bool inside = p < HW;
  bool keep = false;
  if (inside) {
    const float d = __ldg(depth + (size_t)ref * HW + p);
    if (d > 0.0f && __ldg(used + (size_t)ref * HW + p) == 0) {
      const float* cam_r = table + (size_t)ref * GIPUMA_CAM;
      const int py = p / W, px = p - py * W;
      float X[3];
      gipuma_unproject(cam_r, (float)px, (float)py, d, X);
      const float fb = __ldg(cam_r + 21);
      int n = 0;
      for (int s = 0; s < N; ++s) {
        if (s == ref) continue;
        int q;
        float ds;
        n += gipuma_probe(table + (size_t)s * GIPUMA_CAM, depth + (size_t)s * HW, X, fb, disp, H, W, q, ds) ? 1 : 0;
      }
      keep = n >= num_consistent;
    }
    mask[p] = keep ? 1 : 0;
  }
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// emit: the survivors of the vote again, now averaging the world points and colours of the consistent source pixels and
// marking those pixels used; the point goes to offsets[block] + rank, so a view's points are in row-major pixel order.
// Survivors beyond capacity set their used marks but write no point.
__global__ void __launch_bounds__(FUSION_BLOCK)
gipuma_emit_kernel(const float* __restrict__ depth, const float* __restrict__ table, const float* __restrict__ images, int N,
                   int ref, int H, int W, float disp, const unsigned char* __restrict__ mask, const int* __restrict__ offsets,
                   unsigned char* __restrict__ used, float* __restrict__ xyz, unsigned char* __restrict__ rgb,
                   long long capacity) {
  __shared__ int warp_base[FUSION_BLOCK / 32];
  const int HW = H * W;
  const int p = blockIdx.x * FUSION_BLOCK + threadIdx.x;
  const bool keep = p < HW && mask[p] != 0;
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_base[warp] = __popc(bal);
  __syncthreads();
  if (!keep) return;
  long long pos = offsets[blockIdx.x] + __popc(bal & ((1u << lane) - 1u));
  for (int w = 0; w < warp; ++w) pos += warp_base[w];
  const float* cam_r = table + (size_t)ref * GIPUMA_CAM;
  const int py = p / W, px = p - py * W;
  float X[3], sum[3];
  gipuma_unproject(cam_r, (float)px, (float)py, __ldg(depth + (size_t)ref * HW + p), X);
  const float fb = __ldg(cam_r + 21);
  int col[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    sum[k] = X[k];
    col[k] = __float2int_rn(mul(__ldg(images + ((size_t)ref * 3 + k) * HW + p), 255.0f));
  }
  int n = 0;
  for (int s = 0; s < N; ++s) {
    if (s == ref) continue;
    const float* cam_s = table + (size_t)s * GIPUMA_CAM;
    int q;
    float ds;
    if (!gipuma_probe(cam_s, depth + (size_t)s * HW, X, fb, disp, H, W, q, ds)) continue;
    const int qy = q / W, qx = q - qy * W;
    float Xs[3];
    gipuma_unproject(cam_s, (float)qx, (float)qy, ds, Xs);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      sum[k] = add(sum[k], Xs[k]);
      col[k] += __float2int_rn(mul(__ldg(images + ((size_t)s * 3 + k) * HW + q), 255.0f));
    }
    used[(size_t)s * HW + q] = 1;
    ++n;
  }
  if (pos >= capacity) return;
  const float cnt = (float)(n + 1);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    xyz[pos * 3 + k] = dvd(sum[k], cnt);
    rgb[pos * 3 + k] = (unsigned char)(col[k] / (n + 1));
  }
}

}  // namespace mvsf

extern "C" {

int mvsf_fusion_workspace_bytes(int H, int W, size_t* bytes) {
  MVSF_REQUIRE(bytes, "fusion_workspace_bytes: null pointer");
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_workspace_bytes: H x W = %d x %d outside [1, 2^31)", H, W);
  *bytes = mvsf::fusion_ws_bytes(H, W);
  return MVSF_OK;
}

int mvsf_fusion_prepare_cameras(const float* cams, int N, float* cams_inv, mvsf_stream_t stream) {
  MVSF_REQUIRE(cams && cams_inv && N > 0, "fusion_prepare_cameras: null pointer or N = %d < 1", N);
  mvsf::fusion_prepare_kernel<<<mvsf::cdiv(N, 64), 64, 0, (cudaStream_t)stream>>>(cams, N, cams_inv);
  MVSF_LAUNCH_CHECK("fusion_prepare_cameras");
  return MVSF_OK;
}

int mvsf_fusion_filter(int method, const float* depths, const float* confs, const float* cams, const float* cams_inv, int N,
                       int ref, const int* src, int V, int H, int W, float conf, float thres_view, float thres_disp,
                       float dist_base, float rel_diff_base, unsigned char* mask, float* depth_avg, void* workspace,
                       size_t workspace_bytes, mvsf_stream_t stream) {
  MVSF_REQUIRE(method == 0 || method == 1, "fusion_filter: method %d is neither 0 (pcd) nor 1 (dpcd)", method);
  MVSF_REQUIRE(depths && confs && cams && cams_inv && src && mask && depth_avg && workspace, "fusion_filter: null pointer");
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_filter: H x W = %d x %d outside [1, 2^31)", H, W);
  MVSF_REQUIRE(V >= 1 && V <= mvsf::FUSION_MAX_SRC, "fusion_filter: %d source views outside [1, %d]", V, mvsf::FUSION_MAX_SRC);
  MVSF_REQUIRE(N > 0 && ref >= 0 && ref < N, "fusion_filter: reference view %d outside the scene's %d views", ref, N);
  mvsf::FusionSrc s;
  for (int i = 0; i < mvsf::FUSION_MAX_SRC; ++i) s.idx[i] = 0;
  for (int i = 0; i < V; ++i) {
    MVSF_REQUIRE(src[i] >= 0 && src[i] < N, "fusion_filter: source view %d outside the scene's %d views", src[i], N);
    s.idx[i] = src[i];
  }
  if (workspace_bytes < mvsf::fusion_ws_bytes(H, W))
    return mvsf::fail(MVSF_ERR_WORKSPACE, "fusion_filter: workspace %zu < %zu bytes", workspace_bytes, mvsf::fusion_ws_bytes(H, W));
  const int blocks = mvsf::cdiv((long long)H * W, mvsf::FUSION_BLOCK);
  int* counts = (int*)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  if (method == 0)
    mvsf::fusion_pcd_kernel<<<blocks, mvsf::FUSION_BLOCK, 0, st>>>(depths, confs, cams, cams_inv, ref, s, V, H, W, conf,
                                                                  thres_view, thres_disp, mask, depth_avg, counts);
  else
    mvsf::fusion_dpcd_kernel<<<blocks, mvsf::FUSION_BLOCK, 0, st>>>(depths, confs, cams, cams_inv, ref, s, V, H, W, conf,
                                                                   dist_base, rel_diff_base, mask, depth_avg, counts);
  MVSF_LAUNCH_CHECK("fusion_filter");
  mvsf::fusion_scan_kernel<<<1, mvsf::FUSION_SCAN_THREADS, 0, st>>>(counts, blocks);
  MVSF_LAUNCH_CHECK("fusion_scan");
  return MVSF_OK;
}

int mvsf_fusion_extract(const unsigned char* mask, const float* depth_avg, const void* workspace, size_t workspace_bytes,
                        const float* cam_inv, const float* image, float* xyz, unsigned char* rgb, long long capacity, int H,
                        int W, mvsf_stream_t stream) {
  MVSF_REQUIRE(mask && depth_avg && workspace && cam_inv && image, "fusion_extract: null pointer");
  MVSF_REQUIRE(capacity >= 0 && (capacity == 0 || (xyz && rgb)), "fusion_extract: no output for %lld points", capacity);
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_extract: H x W = %d x %d outside [1, 2^31)", H, W);
  if (workspace_bytes < mvsf::fusion_ws_bytes(H, W))
    return mvsf::fail(MVSF_ERR_WORKSPACE, "fusion_extract: workspace %zu < %zu bytes", workspace_bytes, mvsf::fusion_ws_bytes(H, W));
  if (capacity == 0) return MVSF_OK;
  mvsf::fusion_extract_kernel<<<mvsf::cdiv((long long)H * W, mvsf::FUSION_BLOCK), mvsf::FUSION_BLOCK, 0, (cudaStream_t)stream>>>(
      mask, depth_avg, (const int*)workspace, cam_inv, image, xyz, rgb, capacity, H, W);
  MVSF_LAUNCH_CHECK("fusion_extract");
  return MVSF_OK;
}

int mvsf_fusion_gipuma_prepare(const float* depths, const float* confs, const float* cams, int N, int H, int W,
                               float prob_threshold, float depth_min, float depth_max, float* depth, float* cam_table,
                               mvsf_stream_t stream) {
  MVSF_REQUIRE(depths && confs && cams && depth && cam_table, "fusion_gipuma_prepare: null pointer");
  MVSF_REQUIRE(N > 0, "fusion_gipuma_prepare: N = %d < 1", N);
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_gipuma_prepare: H x W = %d x %d outside [1, 2^31)", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)N * H * W;
  const int blocks = mvsf::cdiv(n, 256) < 65536 ? mvsf::cdiv(n, 256) : 65536;   // grid-stride beyond
  mvsf::gipuma_depth_kernel<<<blocks, 256, 0, st>>>(
      depths, confs, n, prob_threshold, depth_min, depth_max, depth);
  MVSF_LAUNCH_CHECK("fusion_gipuma_prepare (depth)");
  mvsf::gipuma_cameras_kernel<<<mvsf::cdiv(N, 64), 64, 0, st>>>(cams, N, cam_table);
  MVSF_LAUNCH_CHECK("fusion_gipuma_prepare (cameras)");
  return MVSF_OK;
}

int mvsf_fusion_gipuma_vote(const float* depth, const unsigned char* used, const float* cam_table, int N, int ref, int H, int W,
                            float disp_threshold, int num_consistent, unsigned char* mask, void* workspace,
                            size_t workspace_bytes, mvsf_stream_t stream) {
  MVSF_REQUIRE(depth && used && cam_table && mask && workspace, "fusion_gipuma_vote: null pointer");
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_gipuma_vote: H x W = %d x %d outside [1, 2^31)", H, W);
  MVSF_REQUIRE(N > 0 && ref >= 0 && ref < N, "fusion_gipuma_vote: reference view %d outside the scene's %d views", ref, N);
  MVSF_REQUIRE(num_consistent >= 0, "fusion_gipuma_vote: num_consistent = %d < 0", num_consistent);
  if (workspace_bytes < mvsf::fusion_ws_bytes(H, W))
    return mvsf::fail(MVSF_ERR_WORKSPACE, "fusion_gipuma_vote: workspace %zu < %zu bytes", workspace_bytes, mvsf::fusion_ws_bytes(H, W));
  const int blocks = mvsf::cdiv((long long)H * W, mvsf::FUSION_BLOCK);
  int* counts = (int*)workspace;
  cudaStream_t st = (cudaStream_t)stream;
  mvsf::gipuma_vote_kernel<<<blocks, mvsf::FUSION_BLOCK, 0, st>>>(depth, used, cam_table, N, ref, H, W, disp_threshold,
                                                                  num_consistent, mask, counts);
  MVSF_LAUNCH_CHECK("fusion_gipuma_vote");
  mvsf::fusion_scan_kernel<<<1, mvsf::FUSION_SCAN_THREADS, 0, st>>>(counts, blocks);
  MVSF_LAUNCH_CHECK("fusion_scan");
  return MVSF_OK;
}

int mvsf_fusion_gipuma_emit(const float* depth, const float* cam_table, const float* images, int N, int ref, int H, int W,
                            float disp_threshold, const unsigned char* mask, const void* workspace, size_t workspace_bytes,
                            unsigned char* used, float* xyz, unsigned char* rgb, long long capacity, mvsf_stream_t stream) {
  MVSF_REQUIRE(depth && cam_table && images && mask && workspace && used, "fusion_gipuma_emit: null pointer");
  MVSF_REQUIRE(capacity >= 0 && (capacity == 0 || (xyz && rgb)), "fusion_gipuma_emit: no output for %lld points", capacity);
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "fusion_gipuma_emit: H x W = %d x %d outside [1, 2^31)", H, W);
  MVSF_REQUIRE(N > 0 && ref >= 0 && ref < N, "fusion_gipuma_emit: reference view %d outside the scene's %d views", ref, N);
  if (workspace_bytes < mvsf::fusion_ws_bytes(H, W))
    return mvsf::fail(MVSF_ERR_WORKSPACE, "fusion_gipuma_emit: workspace %zu < %zu bytes", workspace_bytes, mvsf::fusion_ws_bytes(H, W));
  mvsf::gipuma_emit_kernel<<<mvsf::cdiv((long long)H * W, mvsf::FUSION_BLOCK), mvsf::FUSION_BLOCK, 0, (cudaStream_t)stream>>>(
      depth, cam_table, images, N, ref, H, W, disp_threshold, mask, (const int*)workspace, used, xyz, rgb, capacity);
  MVSF_LAUNCH_CHECK("fusion_gipuma_emit");
  return MVSF_OK;
}
}
