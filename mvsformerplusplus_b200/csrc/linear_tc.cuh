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

// Streamed-weight GEMM (weights too large to stay resident: N, K in the thousands).  N % 64 == 0, K = taps * cin.
// Row m of A is an implicit-GEMM row: m = (img * H + y) * W + x enumerates an H x W grid per image, and K-block kb reads
// channels [c, c + 64) of tap t = kb / (cin / 64) at input pixel (y + dy_t, x + dx_t) of the same grid, zero outside it:
// A element (m, t * cin + c) = Ah[(m + dy_t * W + dx_t) * lda + c].  A token linear is one tap (0, 0) on a 1 x 1 grid.
// Row m is stored at output pixel (img, sy * y + py, sx * x + px) of an (sy H) x (sx W) map (the parity classes of a
// stride-2 transposed convolution); C / C2 / res rows are indexed by that pixel.  Epilogues: LIN_BIAS, LIN_GELU,
// LIN_ELU1, LIN_RES, LIN_SILU; the C2 split of row p is [hi(0..N) | lo(0..N)].
struct TcsArgs : TcLinArgs {
  int H, W, cin, ntaps;
  unsigned long long taps;   // tap t: bits [4t, 4t+2) = dy + 1, [4t+2, 4t+4) = dx + 1  (dy, dx in {-1, 0, 1})
  int sy, sx, py, px;
};
void tcs_token_rows(TcsArgs& a);   // one tap (0, 0) on a 1 x 1 grid: plain rows of A, stored in place
// token linear of M rows: A rows [hi(K) | lo(K)] of stride lda, weights [N][K] at Bh / Bl (rows of stride K)
inline TcsArgs tcs_rows(const __half* A, int lda, int K, const __half* Bh, const __half* Bl, int N, int M) {
  TcsArgs a{};
  a.Ah = A; a.Al = A + K; a.lda = lda;
  a.Bh = Bh; a.Bl = Bl; a.ldb = K;
  a.M = M; a.N = N; a.K = K;
  tcs_token_rows(a);
  return a;
}
int launch_linear_tcs(const TcsArgs& a, int epi, cudaStream_t s);
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
