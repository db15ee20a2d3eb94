// Host-side interface of the wgmma linear layers (linear_tc.cu).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace mvsf {

struct TcLinArgs {
  const __half* Ah; const __half* Al; int lda;  // activations [M][K] as fp16 hi and lo parts (x ~= hi + lo), row stride lda
  const __half* Bh; const __half* Bl; int ldb;  // weights [N][K] (nn.Linear layout) as fp16 hi and lo parts, row stride ldb
  int M, N, K;
  const float* bias;            // [N] or nullptr
  const float* res; int ldres;  // residual (LIN_RES / LIN_RES_LN)
  const float* gamma;           // [N]
  const float* ln_w; const float* ln_b; float ln_eps;
  int elu_cols;
  float* C; int ldc;            // fp32 result (may be nullptr when only the split result is needed)
  float* Cpre; int ldcpre;      // LayerNorm epilogues only, optional: the value BEFORE the LayerNorm (the residual stream of a
                                // pre-norm block: x_new = res + gamma * (acc + bias)), may alias `res`
  __half* C2; int ldc2;         // optional fp16 hi|lo split of the result: row m = [hi(0..N) | lo(0..N)]
};

int launch_linear_tc(const TcLinArgs& a, int epi, cudaStream_t s);
// out row m = [hi(0..K) | lo(0..K)] (ldo >= 2K)
int launch_split_f16(const float* x, int ldx, __half* out, int ldo, int M, int K, cudaStream_t s);
// element-wise split of a flat fp32 blob into two fp16 blobs with the same indexing (weights, done once at install time)
int launch_split_blob_f16(const float* x, __half* hi, __half* lo, size_t n, cudaStream_t s);
__device__ __forceinline__ void split_store8(__half* hi_dst, __half* lo_dst, const float (&v)[8]) {
  __align__(16) __half h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    h[e] = __float2half_rn(v[e]);
    l[e] = __float2half_rn(v[e] - __half2float(h[e]));
  }
  *reinterpret_cast<uint4*>(hi_dst) = *reinterpret_cast<uint4*>(h);
  *reinterpret_cast<uint4*>(lo_dst) = *reinterpret_cast<uint4*>(l);
}

}  // namespace mvsf
