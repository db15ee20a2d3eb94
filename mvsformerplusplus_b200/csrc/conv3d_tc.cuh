// Host-side interface of the wgmma implicit-GEMM 3-D convolutions (conv3d_tc.cu) used by the U-Net regularisers.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace mvsf {

enum ConvTcMode { CONV_S1 = 0, CONV_S2 = 1, DECONV_S2 = 2 };   // stride (1,1,1) | (SD,2,2) | transposed (SD,2,2)
enum ConvTcOut { OUT_SPLIT = 0, OUT_F32 = 1, OUT_PROB = 2 };   // fp16 hi|lo activations | fp32 (+fp32 skip) | fused 1x1x1 prob

struct ConvTcArgs {
  const __half* in_hi; const __half* in_lo;      // input activations [ID][IH][IW][CIN], x ~= hi + lo
  const __half* wtc;                             // packed weight slabs (conv3d_tc_pack)
  const float* bias;                             // [COUT] (BatchNorm shift)
  const __half* skip_hi; const __half* skip_lo;  // OUT_SPLIT: optional skip tensor [OD][OH][OW][COUT], added after the ReLU
  const float* skip32;                           // OUT_F32 / OUT_PROB: fp32 skip tensor
  __half* out_hi; __half* out_lo;                // OUT_SPLIT
  float* out32;                                  // OUT_F32: [OD][OH][OW][COUT]; OUT_PROB: logits [OD][OH][OW]
  const float* probw;                            // OUT_PROB: w[COUT], b
  int CIN, COUT, SD, ID, IH, IW;                 // the output extent follows from mode and SD
  int KG;                                        // channel octets per pipeline unit = conv3d_tc_kg(mode, CIN)
  int col;                                       // weight slab layout / kernel = conv3d_tc_col(mode, SD, COUT)
};

int conv3d_tc_kg(int mode, int cin);                           // 2 (16 channels per unit) for cin >= 16 except strided convs
size_t conv3d_tc_packed_halves(int mode, int cin, int cout);   // number of fp16 elements of one layer's packed slabs
// w32: [27][cin][cout] fp32 (BN folded) -> slabs [kd][channel group][9 (transposed: 16) weight blocks x 2 MMA variants x
// 2 k-chunks x NPAD x 8]
int conv3d_tc_col(int mode, int sd, int cout);                 // 1: depth-streaming kernel (depth stride 1, Cout <= 32)
int conv3d_tc_pack(const float* w32, __half* out, int mode, int sd, int cin, int cout, cudaStream_t s);
int launch_conv3d_tc(const ConvTcArgs& a, int mode, int out_mode, cudaStream_t s);
// hi[n], lo[n] fp16 -> x [n] fp32 (n % 8 == 0), the inverse of launch_split_f16
int launch_merge_vec8(const __half* hi, const __half* lo, float* x, size_t n, cudaStream_t s);

}  // namespace mvsf
