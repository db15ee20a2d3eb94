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

// Token MLP of a transformer block in one kernel: proj (64 -> 64) and its residual + LayerNorm epilogue, FFN1
// (64 -> 256, GELU), FFN2 (256 -> 64) and its residual epilogue.  With p = proj(A) + proj_b, f = FFN(input):
//   MLP_PRE_NORM       (FMT block, block.py:344-345):  x = res + gamma1 p;  x += gamma2 f(LN_mid(x));  C = x, C2 = split(LN_out(x))
//   MLP_PRE_NORM_LAST  (last FMT block):               the same, C = x only
//   MLP_POST_NORM      (transformer layer, module.py:575-576):  y = LN_mid(res + gamma1 p);  C = LN_out(y + gamma2 f(y)),
//                                                               C2 = split(C)
// Rows are dense: A [M][hi(64) | lo(64)] fp16, res and C [M][64] fp32 (C may alias res), C2 [M][hi(64) | lo(64)].
// Weights (nn.Linear layout, hi and lo parts with rows of stride K): proj [64][64], FFN1 [256][64], FFN2 [64][256].
enum MlpForm { MLP_PRE_NORM = 0, MLP_PRE_NORM_LAST = 1, MLP_POST_NORM = 2 };
struct TokenMlpArgs {
  const __half* A;
  const float* res;
  float* C;
  __half* C2;
  const __half *pw_h, *pw_l, *f1w_h, *f1w_l, *f2w_h, *f2w_l;
  const float *proj_b, *gamma1, *f1_b, *f2_b, *gamma2;
  const float *mid_w, *mid_b, *out_w, *out_b;   // LN_mid, LN_out (out_* unused by MLP_PRE_NORM_LAST)
  float mid_eps, out_eps;
  int M;
};
int launch_token_mlp(const TokenMlpArgs& a, int form, cudaStream_t s);

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

}  // namespace mvsf
