// Linear attention (attention.py:261-291) and row LayerNorms on token rows, templated on the head geometry / width so
// that FMT (4 heads of 16, d_model 64: fmt.cu) and the ViT decoder (12 heads of 64, d_model 768: vit_decoder.cu) share
// them.  The LayerNorms emit the fp16 hi|lo split [hi(C) | lo(C)] the tensor-core GEMMs consume.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace mvsf {

// K/V summary of NH heads of HD: KV[h][m][d] = sum_s k[s,h,d] v[s,h,m], then ksum[h][d] = sum_s k[s,h,d]
template <int NH, int HD>
struct LinAttn {
  static constexpr int KVSZ = NH * HD * HD + NH * HD;
  static constexpr int HG = HD * HD >= 1024 ? 1 : 1024 / (HD * HD);   // heads per kv_partial block (256 threads x 4 d)
  static constexpr int ITEMS = HG * HD * HD / 1024;                    // (h, m, 4 d) strips per thread
  static_assert(NH % HG == 0 && ITEMS >= 1 && HD % 16 == 0, "head geometry");
};

// partial[view][blk][KVSZ] over a KV_CHUNK-token chunk; grid (chunks, views, NH / HG)
constexpr int KV_CHUNK = 256, KV_TILE = 64;
template <int NH, int HD>
__global__ void __launch_bounds__(256)
kv_partial_kernel(const float* __restrict__ kv, int ld, int koff, int voff, int L, float* __restrict__ partial) {
  using G = LinAttn<NH, HD>;
  constexpr int CW = G::HG * HD;   // columns of the head group
  __shared__ __align__(16) float ks[KV_TILE][CW];
  __shared__ __align__(16) float vs[KV_TILE][CW];
  const int view = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x, c0 = blockIdx.z * CW;
  const float* base = kv + (size_t)view * L * ld;
  float acc[G::ITEMS][4], ksum[G::ITEMS][4];
#pragma unroll
  for (int it = 0; it < G::ITEMS; ++it)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[it][e] = ksum[it][e] = 0.f;
  const int s_begin = blk * KV_CHUNK, s_end = min(L, s_begin + KV_CHUNK);
  for (int s0 = s_begin; s0 < s_end; s0 += KV_TILE) {
    __syncthreads();
    for (int i = tid; i < KV_TILE * CW / 4; i += 256) {
      int r = i / (CW / 4), c = (i % (CW / 4)) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (s0 + r < s_end) {
        a = ldg4(base + (size_t)(s0 + r) * ld + koff + c0 + c);
        b = ldg4(base + (size_t)(s0 + r) * ld + voff + c0 + c);
      }
      *reinterpret_cast<float4*>(&ks[r][c]) = a;
      *reinterpret_cast<float4*>(&vs[r][c]) = b;
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < G::ITEMS; ++it) {
      const int item = tid + 256 * it;
      const int h = item / (HD * HD / 4), m = (item / (HD / 4)) % HD, d0 = (item % (HD / 4)) * 4;
#pragma unroll 8
      for (int r = 0; r < KV_TILE; ++r) {
        float4 k4 = *reinterpret_cast<const float4*>(&ks[r][h * HD + d0]);
        float vv = vs[r][h * HD + m];
        acc[it][0] = fmaf(k4.x, vv, acc[it][0]); acc[it][1] = fmaf(k4.y, vv, acc[it][1]);
        acc[it][2] = fmaf(k4.z, vv, acc[it][2]); acc[it][3] = fmaf(k4.w, vv, acc[it][3]);
        ksum[it][0] += k4.x; ksum[it][1] += k4.y; ksum[it][2] += k4.z; ksum[it][3] += k4.w;
      }
    }
  }
  float* o = partial + ((size_t)view * gridDim.x + blk) * G::KVSZ;
#pragma unroll
  for (int it = 0; it < G::ITEMS; ++it) {
    const int item = tid + 256 * it;
    const int h = blockIdx.z * G::HG + item / (HD * HD / 4), m = (item / (HD / 4)) % HD, d0 = (item % (HD / 4)) * 4;
    *reinterpret_cast<float4*>(o + (h * HD + m) * HD + d0) = make_float4(acc[it][0], acc[it][1], acc[it][2], acc[it][3]);
    if (m == 0)
      *reinterpret_cast<float4*>(o + NH * HD * HD + h * HD + d0) =
          make_float4(ksum[it][0], ksum[it][1], ksum[it][2], ksum[it][3]);
  }
}
template <int NH, int HD>
__global__ void kv_final_kernel(const float* __restrict__ partial, int nblk, float* __restrict__ fin) {
  constexpr int KVSZ = LinAttn<NH, HD>::KVSZ;
  const int view = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KVSZ) return;
  float s = 0.f;
  for (int b = 0; b < nblk; ++b) s += partial[((size_t)view * nblk + b) * KVSZ + i];
  fin[(size_t)view * KVSZ + i] = s;
}
// both passes over L tokens of `views` views: kv rows of width ld, k at column koff, v at voff
template <int NH, int HD>
static int launch_kv_summary(const float* kv, int ld, int koff, int voff, int L, int views, float* partial, float* fin,
                             cudaStream_t s) {
  using G = LinAttn<NH, HD>;
  const int nblk = cdiv(L, KV_CHUNK);
  kv_partial_kernel<NH, HD><<<dim3(nblk, views, NH / G::HG), 256, 0, s>>>(kv, ld, koff, voff, L, partial);
  MVSF_LAUNCH_CHECK("kv_partial");
  kv_final_kernel<NH, HD><<<dim3(cdiv(G::KVSZ, 256), views), 256, 0, s>>>(partial, nblk, fin);
  MVSF_LAUNCH_CHECK("kv_final");
  return MVSF_OK;
}

// out[s][h*HD+m] = (sum_d q[s,h,d] KV[h][m][d]) / (q[s,h,:] . ksum[h,:] + 1e-6)     (attention.py:281-284)
// grid (tokens / 128, NH); out2 rows are the fp16 hi|lo split [hi(NH*HD) | lo(NH*HD)]
template <int NH, int HD>
__global__ void __launch_bounds__(128)
linattn_apply_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ kvfin, size_t kv_view_stride,
                     __half* __restrict__ out2, int L, int M) {
  constexpr int C = NH * HD;
  __shared__ __align__(16) float kvs[HD * HD + HD];
  const int h = blockIdx.y;
  const int s = blockIdx.x * 128 + threadIdx.x;
  const int view = (blockIdx.x * 128) / L;  // host guarantees L % 128 == 0 or a single view per launch
  const float* kvp = kvfin + (size_t)view * kv_view_stride;
  for (int i = threadIdx.x; i < HD * HD; i += 128) kvs[i] = __ldg(kvp + h * HD * HD + i);
  if (threadIdx.x < HD) kvs[HD * HD + threadIdx.x] = __ldg(kvp + NH * HD * HD + h * HD + threadIdx.x);
  __syncthreads();
  if (s >= M) return;
  float qv[HD];
  const float* qp = q + (size_t)s * ldq + h * HD;
#pragma unroll
  for (int c = 0; c < HD / 4; ++c) {
    float4 t = ldg4(qp + c * 4);
    qv[c * 4] = t.x; qv[c * 4 + 1] = t.y; qv[c * 4 + 2] = t.z; qv[c * 4 + 3] = t.w;
  }
  float den = 0.f;
#pragma unroll
  for (int d = 0; d < HD; ++d) den = fmaf(qv[d], kvs[HD * HD + d], den);
  const float z = __fdiv_rn(1.0f, den + 1e-6f);
  __half* op = out2 + (size_t)s * (2 * C) + h * HD;
#pragma unroll
  for (int mq = 0; mq < HD / 4; ++mq) {
    float r[4];
#pragma unroll
    for (int mm = 0; mm < 4; ++mm) {
      const float4* kp = reinterpret_cast<const float4*>(&kvs[(mq * 4 + mm) * HD]);
      float4 a = kp[0];
      float t = qv[0] * a.x;
      t = fmaf(qv[1], a.y, t); t = fmaf(qv[2], a.z, t); t = fmaf(qv[3], a.w, t);
#pragma unroll
      for (int d4 = 1; d4 < HD / 4; ++d4) {
        a = kp[d4];
        t = fmaf(qv[4 * d4], a.x, t); t = fmaf(qv[4 * d4 + 1], a.y, t);
        t = fmaf(qv[4 * d4 + 2], a.z, t); t = fmaf(qv[4 * d4 + 3], a.w, t);
      }
      r[mm] = t * z;
    }
    split_store2(op + mq * 4, op + C + mq * 4, r[0], r[1]);
    split_store2(op + mq * 4 + 2, op + C + mq * 4 + 2, r[2], r[3]);
  }
}

// ---- row LayerNorm over C channels, one warp per row: lane owns C / 32 values (C == 64: a float2 at 2 lane; else float4s
// at 4 lane + 128 i)
template <int C>
struct RowVec {
  static constexpr int E = C / 32;
  static_assert(C == 64 || C % 128 == 0, "row width");
  float v[E];
  __device__ __forceinline__ static int col(int lane, int e) { return C == 64 ? 2 * lane + e : 4 * lane + 128 * (e / 4) + e % 4; }
  __device__ __forceinline__ void load(const float* row, int lane) {
    if constexpr (C == 64) {
      const float2 t = ldg2(row + lane * 2);
      v[0] = t.x; v[1] = t.y;
    } else {
#pragma unroll
      for (int i = 0; i < E / 4; ++i) {
        const float4 t = ldg4(row + 4 * lane + 128 * i);
        v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
      }
    }
  }
  __device__ __forceinline__ void store(float* row, int lane) const {
#pragma unroll
    for (int i = 0; i < E / 4; ++i)
      *reinterpret_cast<float4*>(row + 4 * lane + 128 * i) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  }
  // v <- LN(v) with weight w, bias b (two-pass mean / variance over the row, IEEE division by the deviation)
  __device__ __forceinline__ void layernorm(const float* __restrict__ w, const float* __restrict__ b, float eps, int lane) {
    float s = v[0];
#pragma unroll
    for (int e = 1; e < E; ++e) s += v[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.0f / C);
    float d[E];
#pragma unroll
    for (int e = 0; e < E; ++e) d[e] = v[e] - mean;
    float q = d[0] * d[0];
#pragma unroll
    for (int e = 1; e < E; ++e) q += d[e] * d[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float sd = sqrtf(q * (1.0f / C) + eps);
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = col(lane, e);
      v[e] = __fdiv_rn(d[e], sd) * __ldg(w + c) + __ldg(b + c);
    }
  }
  __device__ __forceinline__ void store_split(__half* y2, int lane) const {   // [hi(C) | lo(C)]
#pragma unroll
    for (int e = 0; e < E; e += 2) {
      const int c = col(lane, e);
      split_store2(y2 + c, y2 + C + c, v[e], v[e + 1]);
    }
  }
};

// y2[row] = split(LN(x[row]))
template <int C>
__global__ void __launch_bounds__(256)
layernorm_split_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                       __half* __restrict__ y2, int M, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  RowVec<C> r;
  r.load(x + (size_t)row * C, lane);
  r.layernorm(w, b, eps, lane);
  r.store_split(y2 + (size_t)row * 2 * C, lane);
}

}  // namespace mvsf
