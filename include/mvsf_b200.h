/*
 * libmvsf_b200 - C ABI of the CUDA-native (sm_90a) MVSFormer++ depth-inference hot path.
 *
 * The reference (maybeLx/MVSFormerPlusPlus) has no FFI layer: its seams are Python callables
 * (SURVEY.md §8b).  Each entry point below states the reference callable (file:line, relative to the
 * reference repo root) whose arithmetic it replaces.  Conventions:
 *   - every pointer is a DEVICE pointer to fp32 data unless marked "host"; buffers are owned by the
 *     caller and borrowed for the duration of the call (the reference's torch tensors play this role);
 *   - one sample per call (the reference's eval path is batch-1: DINOv2_mvsformer_model.py:88);
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); calls never synchronise;
 *   - return 0 on success, a negative mvsf_status otherwise; mvsf_last_error() gives the message
 *     (the Python host raises RuntimeError, mirroring the reference's Python exceptions);
 *   - there is no CPU fallback and no dispatch: a missing/failed CUDA path is an error.
 *
 * Layouts (HBM):  feature maps are channels-last  [V][H][W][C];  hypothesis / probability volumes are
 * depth-major [D][H][W] (the reference's [B,D,H,W] with B=1);  cost volumes are [D][H][W][G] (NDHWC);
 * tokens are [L][C].  Packed-weight layouts are documented per function and produced by
 * mvsformerplusplus_b200/packing.py from a reference state_dict (BatchNorm folded, eval mode).
 */
#ifndef MVSF_B200_H
#define MVSF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mvsf_stream_t; /* cudaStream_t */

enum mvsf_status {
  MVSF_OK = 0,
  MVSF_ERR_INVALID = -1,     /* bad argument / unsupported shape (reference: AssertionError / NotImplementedError) */
  MVSF_ERR_CUDA = -2,        /* CUDA launch or runtime error */
  MVSF_ERR_WORKSPACE = -3    /* workspace too small */
};

const char* mvsf_last_error(void);
int mvsf_abi_version(void);
/* number of kernel launches issued by this library on the calling thread since the last reset (bench.py's gpu_launches) */
long long mvsf_launch_count(int reset);
/* opt-in device timers around single kernels launched from inside a multi-kernel entry point ("attention_tc"):
 * CUDA events on the launching stream; read = device ms + launches since the last read (synchronises, resets). */
int mvsf_ktimer_enable(int on);
int mvsf_ktimer_read(const char* name, double* ms, long long* launches);

/* ---- layout helpers at the boundary (reference tensors are NCHW: DINOv2_mvsformer_model.py:95-98) */
int mvsf_nchw_to_nhwc(const float* src, float* dst, int N, int C, int HW, mvsf_stream_t stream);
int mvsf_nhwc_to_nchw(const float* src, float* dst, int N, int C, int HW, mvsf_stream_t stream);

/* ---- W1: projection prep.  models/cost_volume.py:68-71 + models/warping.py:80-82 (src@inv(ref), rot/trans)
 *      and torch.inverse(K) of models/position_encoding.py:146.
 * proj [V][2][4][4] (slot 0 extrinsic, slot 1[:3,:3] intrinsic; view 0 = reference view).
 * homs [(V-1)][12]: rot row-major (9) then trans (3) of  P_src * P_ref^-1.   kinv_ref [9] row-major. */
int mvsf_compose_geometry(const float* proj, int V, float* homs, float* kinv_ref, mvsf_stream_t stream);

/* ---- W2 prep for the warp seam: models/warping.py:80-82  proj = src_proj @ inverse(ref_proj) on composed 4x4
 * projections [B][4][4] (fp64 on device) -> homs [B][12] = rot row-major (9) then trans (3). */
int mvsf_homography_from_proj(const float* src_proj, const float* ref_proj, int B, float* homs, mvsf_stream_t stream);

/* ---- F5: models/module.py:692-704 init_inverse_range.  depth_values [Dn] -> out [D][H][W] */
int mvsf_init_inverse_range(const float* depth_values, int Dn, float* out, int D, int H, int W, mvsf_stream_t stream);
/* ---- F6: models/module.py:707-724 schedule_inverse_range (shift=False).
 * prev_depth [H/2][W/2], prev_hypo [Dp][H/2][W/2] (only planes 1 and 2 are read) -> out [D][H][W] */
int mvsf_schedule_inverse_range(const float* prev_depth, const float* prev_hypo, int Dp, float split_itv, float* out,
                                int D, int H, int W, mvsf_stream_t stream);
/* ---- F7: models/position_encoding.py:138-161 get_position_3d(normalize=True).
 * stats [6] = {width_min,width_max,height_min,height_max,depth_min,depth_max}.  pos [3][D][H][W].
 * compute_minmax: 1 = extents from this call's positions + depth range of depth_values, then normalise (B == 1);
 *                 0 = reuse the extents, refresh the depth range, normalise.
 * Batched callers (the reference reduces extents and depth_values.min()/max() over the whole batch,
 * position_encoding.py:152-157, DINOv2_mvsformer_model.py:156):  2 = reset + accumulate this sample's extents,
 * 3 = accumulate, 4 = finalise (decode extents, depth range over depth_values[0..Dn), Dn = B * numdepth),
 * 5 = normalise only.  Unused pointers may be NULL in modes 2-5. */
int mvsf_position3d(const float* kinv_ref, const float* depth, const float* depth_values, int Dn, float* stats,
                    int compute_minmax, float* pos, int D, int H, int W, mvsf_stream_t stream);

/* ---- W2 (finest seam): models/warping.py:69-109 homo_warping_3D_with_mask.
 * src [H][W][C], hom [12], depth [D][H][W] -> warped [C][D][H][W] (reference layout), mask [D][H][W] u8 or NULL */
int mvsf_homo_warp(const float* src_nhwc, const float* hom, const float* depth, float* warped, uint8_t* mask, int C,
                   int D, int H, int W, mvsf_stream_t stream);

/* ---- test seam: the cost-volume passes have two organisations computing the same function - L1 gathers
 * from global memory (warp_corr.cu, any C in 8/16/32/64) and TMA-staged shared-memory windows (warp_tile.cu, C = 8/16, even H).
 * mode 0: force the L1 organisation everywhere (the tests' same-input reference); 1 (default): adaptive - the window kernels
 * of the two-gather plan where they apply, and for mvsf_warp_corr_entropy_store at C = 8, D = 4 a per-call choice made ON
 * THE DEVICE from the call's own geometry (share of sampled taps that miss the pipeline kernel's predicted windows <= 60 per
 * mille -> pipeline kernel, else L1 kernel; both are launched, the one not chosen returns at once); 2: force the window /
 * pipeline kernels wherever they exist (the only way a wide-baseline call reaches the pipeline kernel's out-of-window
 * fallback).  mvsf_warp_corr_last_selection reads the most recent decision back (synchronises). */
int mvsf_warp_corr_set_tile_path(int mode);
int mvsf_warp_corr_last_selection(int* used_pipeline, int* miss_permille);

/* ---- which of the two cost-volume plans to run for a stage shape: 1 = two gathers (mvsf_warp_corr_entropy, mvsf_vis_cnn,
 * mvsf_warp_corr_aggregate; no intermediate buffer), 0 = spill plan (mvsf_warp_corr_entropy_store, mvsf_vis_cnn,
 * mvsf_corr_aggregate; needs a [(V-1)][D][H][W][8] fp32 buffer).  Both give the same volume. */
int mvsf_warp_corr_plan(int C, int G, int D, int H, int W, int V, size_t spill_budget_bytes);

/* ---- W2+W3+W4 pass A: warp + group correlation summed over groups + softmax-entropy over D.
 * models/cost_volume.py:72-92.  feat [V][H][W][C] (view 0 = reference), homs [(V-1)][12], depth [D][H][W]
 * -> entropy [(V-1)][H][W].   The (V-1,C,D,H,W) warped volume is never written. */
int mvsf_warp_corr_entropy(const float* feat, const float* homs, const float* depth, float* entropy, int V, int C,
                           int G, int D, int H, int W, mvsf_stream_t stream);
/* ---- W4 visibility CNN: models/cost_volume.py:37,93.  entropy [N][H][W] -> vis [N][H][W].
 * wts: packed, BN folded: w1[9][16] b1[16] w2[16 ic][9][16 oc] b2[16] w3[16 ic][9][8 oc] b3[8] w4[8] b4[1] (=3649 floats) */
int mvsf_vis_cnn(const float* entropy, const float* wts, float* vis, int N, int H, int W, mvsf_stream_t stream);
/* ---- W2+W3+W4 pass B: recompute warp + group correlation, weight by vis, reduce over views.
 * models/cost_volume.py:72-101 -> volume [D][H][W][G] = sum_v w_v*inprod_v / (sum_v w_v + 1e-6) */
int mvsf_warp_corr_aggregate(const float* feat, const float* homs, const float* depth, const float* vis,
                             float* volume, int V, int C, int G, int D, int H, int W, mvsf_stream_t stream);
/* Faster variant of the two calls above (the one hotpath.py uses): pass A additionally stores the per-view group
 * correlations corr [V-1][D][H*W][G] (G must be 8; 4*G*D*H*W*(V-1) bytes), the view aggregation then streams them
 * instead of gathering the source features a second time (the gather is L1-request bound, HBM has headroom). */
int mvsf_warp_corr_entropy_store(const float* feat, const float* homs, const float* depth, float* entropy, float* corr,
                                 int V, int C, int G, int D, int H, int W, mvsf_stream_t stream);
int mvsf_corr_aggregate(const float* corr, const float* vis, float* volume, int V, int G, int D, int H, int W,
                        mvsf_stream_t stream);

/* ---- R2-R4: models/module.py:367-408 (kind 0: CostRegNet, stride 2, 3^3 prob no bias) and
 *      :453-504 (kind 1: CostRegNet3D, stride (1,2,2), 1^3 prob + bias).  volume [D][H][W][C] -> logits [D][H][W].
 * wts: the small fp32 parameters (small part of packing.pack_costreg_unet: per layer the folded bias[Cout], then the
 * prob conv; 496 floats for kind 0, 292 for kind 1); wts_tc = mvsf_costreg_unet_pack_tc(conv part of
 * packing.pack_costreg_unet: per layer [27][Cin][Cout] with BN scale folded, 290 304 floats). */
int mvsf_costreg_unet_workspace_bytes(int kind, int C, int D, int H, int W, size_t* bytes);
/* install time: conv part -> wts_tc, the fp16 hi/lo weight slabs of the wgmma implicit-GEMM convolutions
 * (csrc/conv3d_tc.cu) */
int mvsf_costreg_unet_tc_bytes(size_t* bytes);
int mvsf_costreg_unet_pack_tc(int kind, const float* conv, void* wts_tc, size_t wts_tc_bytes, mvsf_stream_t stream);
int mvsf_costreg_unet_forward(int kind, const float* volume, const float* wts, const void* wts_tc, float* logits,
                              void* workspace, size_t workspace_bytes, int C, int D, int H, int W, mvsf_stream_t stream);
/* test seam: ONE 3x3x3 layer of the U-Nets on the wgmma implicit-GEMM path, fp32 in / out (module.py:367-504:
 * Conv3d / strided Conv3d / ConvTranspose3d(output_padding = stride - 1) + folded BN + ReLU, optional skip added after the
 * ReLU).  mode 0: stride 1, 1: stride (sd,2,2), 2: transposed (sd,2,2).  in [ID][IH][IW][cin]; w32 = [27][cin][cout] then
 * bias[cout]; skip (or NULL) and out [OD][OH][OW][cout]; workspace >= 4*(nin + 2*nout) + 216*cin*max(cout,16) + 512 bytes. */
int mvsf_conv3d_tc_layer(int mode, int sd, const float* in, const float* w32, const float* skip, float* out,
                         void* workspace, size_t workspace_bytes, int cin, int cout, int ID, int IH, int IW,
                         mvsf_stream_t stream);

/* ---- R1: models/module.py:602-646 PureTransformerCostReg (+ position_encoding.py:164-189 PositionEncoding3D).
 * volume [D][H][W][C] is modified in place by the PE add; pos [3][D][H][W] or NULL.
 * Fixed by the shipped config: down_rate (2,4,4), mid 64, heads 4, mlp 256.  softmax_scale = hd^-0.5*log_tal(N).
 * wts: the small fp32 parameters (small part of packing.pack_costreg_tr, layout in csrc/costreg_tr.cu: pe_proj, biases,
 * LayerNorms, gammas and prob; 672 + 768 layers floats); wts16 = mvsf_split_weights_f16(GEMM part of
 * packing.pack_costreg_tr: the down, qkv, proj, FFN and up weights as [N][K] rows), n_wts = the floats of that GEMM part,
 * 32 768 + 49 152 layers (any other value: -1, nothing launched). */
int mvsf_costreg_tr_workspace_bytes(int C, int D, int H, int W, size_t* bytes);
int mvsf_costreg_tr_forward(float* volume, const float* pos, const float* wts, const void* wts16, size_t n_wts,
                            float* logits, void* workspace, size_t workspace_bytes, int C, int D, int H, int W,
                            int layers, float softmax_scale, mvsf_stream_t stream);
/* install-time helper: fp32 weight blob (n floats, n % 8 == 0) -> out16 = [n fp16 hi parts | n fp16 lo parts] (4n bytes);
 * wts and out16 16-byte aligned */
int mvsf_split_weights_f16(const float* wts, void* out16, size_t n, mvsf_stream_t stream);

/* softmax attention of R1 alone: models/dino/layers/attention.py:141-170 (FlashAttention2.forward after the qkv linear).
 * qkv [N][3][4][16] fp32 -> out [N][64]; workspace >= (N+128)*896 bytes.  wgmma tensor cores, 3-term split-fp16 operands,
 * fp32 accumulation in registers; |q*scale|, |k|, |v| must be < 65504. */
int mvsf_attention_forward(const float* qkv, float* out, void* workspace, size_t workspace_bytes, int N,
                           float softmax_scale, mvsf_stream_t stream);

/* how mvsf_attention_forward (and each layer of mvsf_costreg_tr_forward) covers num_sms SMs at N tokens: the last
 * *split_items (head, 192-query) items of the grid run as *parts key ranges each, merged by a second kernel; 0 and 1
 * when every item runs whole.  Host only. */
int mvsf_attention_split_plan(int N, int num_sms, int* split_items, int* parts);

/* test seam: a token-wise linear layer (nn.Linear) with one of its fused epilogues, as FMT and the transformer regulariser
 * call it: C[M,N] = epi(A[M,K] W[N,K]^T + bias) on the wgmma tensor cores with fp16 hi/lo split operands (fp32-class
 * accuracy), weights resident in shared memory, K % 64 == 0.
 * epi: 0 C = acc + bias, 1 C = gelu(acc + bias) (exact erf), 2 C = col < elu_cols ? elu(acc + bias) + 1 : acc + bias,
 * 3 C = res + gamma * (acc + bias), 4 C = LN(res + gamma * (acc + bias)), 5 C = LN(acc + bias); LN = LayerNorm over
 * the row with ln_w, ln_b, ln_eps.  Only the (N, epi) pairs that FMT and the transformer regulariser run, and the single
 * GEMMs mvsf_token_mlp_forward is compared against, are built (kTcPairs in csrc/linear_tc.cu); any other pair is -1.
 * A [M][lda] and W [N][K] are fp32 and split into fp16 hi/lo parts inside the call.  bias [N] may be NULL;
 * res [M][ldres] and gamma [N] are read by epilogues 3 and 4.
 * Outputs, each optional (C or C2 required): C [M][ldc] fp32; Cpre [M][ldcpre] = the value before the LayerNorm
 * (epilogues 4 and 5 only, may alias res); C2 [M][ldc2] fp16 = [hi(N) | lo(N)] split of C per row.
 * Operands and outputs 16-byte aligned.  workspace >= (M+N)*2K*2 + 256 bytes. */
int mvsf_linear_tc_epilogue(int epi, const float* A, int lda, const float* W, const float* bias, const float* res,
                            int ldres, const float* gamma, const float* ln_w, const float* ln_b, float ln_eps,
                            int elu_cols, float* C, int ldc, float* Cpre, int ldcpre, void* C2, int ldc2,
                            void* workspace, size_t workspace_bytes, int M, int N, int K, mvsf_stream_t stream);
/* test seam: the token MLP of an FMT block or a transformer-regulariser layer in the one kernel they run it on: proj,
 * its residual + LayerNorm epilogue, FFN1 (GELU), FFN2 and its residual epilogue.  With p = A proj_w^T + proj_b and
 * f(z) = gelu(z f1_w^T + f1_b) f2_w^T + f2_b:
 *   form 0 (pre-norm block): x = res + gamma1 p; x += gamma2 f(LN_mid(x)); C = x, C2 = split(LN_out(x))
 *   form 1 (last pre-norm block): the same, C = x only (C2, out_w, out_b unused)
 *   form 2 (post-norm layer): y = LN_mid(res + gamma1 p); C = LN_out(y + gamma2 f(y)), C2 = split(C)
 * LN_mid / LN_out: LayerNorm over the row with mid_w, mid_b, mid_eps / out_w, out_b, out_eps.  Dense fp32 rows: A, res
 * and C [M][64] (C may alias res); C2 [M][128] fp16 = [hi(64) | lo(64)].  Weights fp32 in nn.Linear layout: proj_w
 * [64][64], f1_w [256][64], f2_w [64][256]; A and the weights are split into fp16 hi/lo parts inside the call.  The
 * outputs equal those of the three mvsf_linear_tc_epilogue calls (proj: epilogue 4, FFN1: epilogue 1, FFN2: epilogue 4
 * or 3) bit for bit.  Operands and outputs 16-byte aligned.  workspace >= (M*128 + 73728)*2 bytes. */
int mvsf_token_mlp_forward(int form, const float* A, const float* res, const float* proj_w, const float* proj_b,
                           const float* gamma1, const float* mid_w, const float* mid_b, float mid_eps, const float* f1_w,
                           const float* f1_b, const float* f2_w, const float* f2_b, const float* gamma2,
                           const float* out_w, const float* out_b, float out_eps, float* C, void* C2, void* workspace,
                           size_t workspace_bytes, int M, mvsf_stream_t stream);
/* test seam: the streamed-weight GEMM the ViT decoder runs on (models/module.py:273-364: its q/k/v, proj, fc1, fc2
 * linears and conv head), for token rows.  Weights stream through the pipeline with A, so N and K are limited only by
 * N % 64 == 0 and K % 64 == 0.  epi: 0 bias, 1 gelu, 2 elu+1 on columns < elu_cols, 3 C = res + gamma * (acc + bias),
 * 6 C = silu(acc + bias); no LayerNorm epilogues.  Arguments and outputs as mvsf_linear_tc_epilogue (no Cpre). */
int mvsf_linear_tc_streamed_epilogue(int epi, const float* A, int lda, const float* W, const float* bias,
                                     const float* res, int ldres, const float* gamma, int elu_cols, float* C, int ldc,
                                     void* C2, int ldc2, void* workspace, size_t workspace_bytes, int M, int N, int K,
                                     mvsf_stream_t stream);

/* ---- S1: models/cost_volume.py:105-117 + models/module.py:649-655 (eval, depth_type 'ce').
 * logits [D][H][W], depth hypotheses [D][H][W] -> prob [D][H][W], depth [H][W], conf [H][W] */
int mvsf_softargmax(const float* logits, const float* depth_hypo, float tmp, float* prob, float* depth, float* conf,
                    int D, int H, int W, mvsf_stream_t stream);
/* ---- S2: DINOv2_mvsformer_model.py:167-177: acc (+)= scale * nearest_upsample(conf) ; init!=0 overwrites */
int mvsf_conf_accumulate(const float* conf, int h, int w, float* acc, int H, int W, float scale, int init,
                         mvsf_stream_t stream);

/* ---- F1-F4: models/FMT.py:164-206 FMT_with_pathway.forward.
 * Inputs are the reference's NCHW pyramids: f1 [V][64][H1][W1], f2 [V][32][2H1][2W1], f3 [V][16][4H1][4W1],
 * f4 [V][8][8H1][8W1]; pe [H1*W1][64] is the PositionEncodingSineNorm table (position_encoding.py:61-74).
 * Outputs are channels-last: o1 [V][H1][W1][64] ... o4 [V][8H1][8W1][8].  wts: the small fp32 parameters (small part
 * of packing.pack_fmt, layout in csrc/fmt.cu: norms, biases, LayerScales, dim_reduction and smooth weights; 17 856
 * floats); wts16 = mvsf_split_weights_f16(GEMM part of packing.pack_fmt: the qkv, proj and MLP weights as [N][K] rows),
 * n_wts = the floats of that GEMM part, 196 608 (any other value: -1, nothing launched). */
int mvsf_fmt_workspace_bytes(int V, int H1, int W1, size_t* bytes);
int mvsf_fmt_forward(const float* f1, const float* f2, const float* f3, const float* f4, const float* pe,
                     const float* wts, const void* wts16, size_t n_wts, float* o1, float* o2, float* o3, float* o4,
                     void* workspace, size_t workspace_bytes, int V, int H1, int W1, mvsf_stream_t stream);

/* ---- P1: models/module.py:208-239 FPNEncoder.forward (feat_chs [8,16,32,64], norm_type 'BN', eval; every layer
 *      Conv2d(bias=False) -> BatchNorm folded -> LeakyReLU(0.1), module.py:61-80).
 * x [N][3][H][W] (H, W positive multiples of 8) -> c01 [N][H][W][8], c11 [N][H/2][W/2][16], c21 [N][H/4][W/4][32],
 * c31 [N][H/8][W/8][64] (NHWC).  Layers conv00, conv01, downsample1, conv10, conv11, downsample2, conv20, conv21,
 * downsample3, conv30, conv31, each w [KS*KS][CI][CO] with BN scale folded and the folded shift [CO].  wts: the small
 * fp32 parameters (small part of packing.pack_fpn_encoder: conv00's w and shift, then the shifts of the other layers;
 * 1 528 floats); wts_tc = mvsf_fpn_pack_tc(0, conv part of packing.pack_fpn_encoder: w of every layer after conv00,
 * 132 800 floats).  Bad shapes: -1, nothing launched. */
int mvsf_fpn_encoder_workspace_bytes(int N, int H, int W, size_t* bytes);
int mvsf_fpn_encoder_forward(const float* x, const float* wts, const void* wts_tc, float* c01, float* c11, float* c21,
                             float* c31, void* workspace, size_t workspace_bytes, int N, int H, int W, mvsf_stream_t stream);
/* The encoder as DINOv2MVSNet.forward uses it (DINOv2_mvsformer_model.py:85-88): c31 receives LeakyReLU(conv31) +
 * vit_feat[n % V] (one fp32 add in the last layer's epilogue), vit_feat [V][H/8][W/8][64] (NHWC, what
 * mvsf_vit_decoder_forward writes for one batch item).  Image n = b V + v thus gets view v of batch item 0's ViT
 * features, as the reference's eval forward adds vit_feat[vi] for every batch item. */
int mvsf_fpn_encoder_vit_forward(const float* x, const float* vit_feat, int V, const float* wts, const void* wts_tc,
                                 float* c01, float* c11, float* c21, float* c31, void* workspace, size_t workspace_bytes,
                                 int N, int H, int W, mvsf_stream_t stream);
/* ---- P2: models/module.py:242-270 FPNDecoder.forward (F.interpolate bilinear, align_corners=True; BN folded).
 * c01..c31 as the encoder writes them (NHWC, full-resolution H x W) -> o0 [N][64][H/8][W/8], o1 [N][32][H/4][W/4],
 * o2 [N][16][H/2][W/2], o3 [N][8][H][W] (NCHW: the layout mvsf_fmt_forward reads, DINOv2_mvsformer_model.py:95-98).
 * wts: the small fp32 parameters (small part of packing.pack_fpn_decoder: out0 [64 ci][64 co] + shift[64]; per level
 * k: inner_k [CL][64] + bias[64], then out_k's shift[C_k]; 7 992 floats); wts_tc = mvsf_fpn_pack_tc(1, conv part of
 * packing.pack_fpn_decoder: out_k [9][64][C_k], 32 256 floats).  The full-resolution intra feature never reaches HBM. */
int mvsf_fpn_decoder_workspace_bytes(int N, int H, int W, size_t* bytes);
int mvsf_fpn_decoder_forward(const float* c01, const float* c11, const float* c21, const float* c31, const float* wts,
                             const void* wts_tc, float* o0, float* o1, float* o2, float* o3, void* workspace,
                             size_t workspace_bytes, int N, int H, int W, mvsf_stream_t stream);
/* install time: fp32 conv part -> fp16 hi/lo weight tiles of the wgmma convolutions (csrc/fpn.cu); part 0 encoder,
 * 1 decoder */
int mvsf_fpn_tc_bytes(int part, size_t* bytes);
int mvsf_fpn_pack_tc(int part, const float* conv, void* wts_tc, size_t wts_tc_bytes, mvsf_stream_t stream);

/* ---- V1: models/module.py:273-364 CrossVITDecoder.forward, shipped config (d_model 768, 12 heads, linear attention,
 *      ffn 768 -> 3072, LayerScale, pre-norm CrossBlocks with pre_norm_query, 3 interval layers, eval-mode BN folded).
 * x0, x1, x2 [B][V][h*w][768] (the ViT tokens of dinov2.py:249-266 without the cls token, view 0 = reference)
 * -> out [B*V][4h][4w][64] (NHWC).  wts: the small fp32 parameters (small part of packing.pack_vit_decoder, layout in
 * csrc/vit_decoder.cu: norms, biases, LayerScales, prev_values and folded conv biases; 49 608 floats); wts_tc =
 * mvsf_split_weights_f16(GEMM part of packing.pack_vit_decoder: the GEMM and conv weights as [N][K] rows, 37 814 272
 * floats).  Bad shapes (B < 1, V < 2, h or w outside [1, 2048)): -1, nothing launched. */
int mvsf_vit_decoder_workspace_bytes(int B, int V, int h, int w, size_t* bytes);
int mvsf_vit_decoder_forward(const float* x0, const float* x1, const float* x2, const float* wts, const void* wts_tc,
                             float* out, void* workspace, size_t workspace_bytes, int B, int V, int h, int w,
                             mvsf_stream_t stream);

/* ---- V2: models/dino/dinov2.py:249-266 DinoVisionTransformer.forward_interval_features, shipped config (ViT-B/14 built
 *      by DINOv2_mvsformer_model.py:40-41: embed 768, 12 blocks of 12 heads x 64 softmax attention (attention.py:77-101,
 *      scale 1/8), mlp 3072 exact-erf GELU, LayerScale, LayerNorm eps 1e-6, cross_interval_layers 3).
 * img [n][3][14 gh][14 gw] fp32 (contiguous); pos [gh gw + 1][768] = interpolate_pos_encoding(pos_embed) for the grid
 * (dinov2.py:176-200, computed once per grid at pack time).  Outputs, cls token dropped: out0 = block 3, out1 = block 7,
 * out2 = norm(block 11), each [n][gh gw][768] in its first n gh gw rows; out0 and out1 also hold the residual stream and
 * need n (gh gw + 1) rows (the n cls rows come after the patch rows), out2 needs n gh gw rows.
 * wts: the small fp32 parameters (small part of packing.pack_vit, layout in csrc/vit.cu, 141 312 floats); wts_tc =
 * mvsf_split_weights_f16(GEMM part of packing.pack_vit: 85 426 176 floats).  Bad shapes (n outside [1, 65535], gh or
 * gw outside [1, 1024], n (gh gw + 1) > 2^21), null or misaligned pointers: -1; short workspace: -3; nothing launched. */
int mvsf_vit_workspace_bytes(int n, int gh, int gw, size_t* bytes);
int mvsf_vit_forward(const float* img, const float* pos, const float* wts, const void* wts_tc, float* out0, float* out1,
                     float* out2, void* workspace, size_t workspace_bytes, int n, int gh, int gw, mvsf_stream_t stream);
/* The same forward on images of any size: img [n][3][H][W] fp32 (contiguous) is resized to 14 gh x 14 gw as
 * F.interpolate(mode="bicubic", align_corners=False) does (DINOv2_mvsformer_model.py:76-77) inside the patch im2col; the
 * resized image is never stored.  H, W >= 1 and H W < 2^30. */
int mvsf_vit_forward_image(const float* img, int H, int W, const float* pos, const float* wts, const void* wts_tc,
                           float* out0, float* out1, float* out2, void* workspace, size_t workspace_bytes, int n, int gh,
                           int gw, mvsf_stream_t stream);
/* The ViT's softmax attention alone: qkv [n][N][2304] fp32 (row stride ldq, [q | k | v] x 12 heads x 64) -> out
 * [n][N][768] (row stride ldo).  workspace >= n * 12 * ceil(N / 128) * 100 352 bytes. */
int mvsf_vit_attention_forward(const float* qkv, int ldq, float* out, int ldo, void* workspace, size_t workspace_bytes,
                               int n, int N, mvsf_stream_t stream);

/* ---- P1: depth-map fusion, test.py:387-517 (filter_depth / dynamic_filter_depth) over misc/fusion.py:79-165, per
 *      reference view.  The scene is depths [N][H][W], confs [N][H][W] (fp32, contiguous) and cams [N][2][4][4] (slot 0
 *      extrinsic, slot 1 [:3][:3] intrinsic); the source views of a reference view are an index list into them.
 * workspace: (ceil(H W / 256) + 1) ints per reference view; mvsf_fusion_filter leaves in it the exclusive scan of the
 * survivor counts of the 256-pixel blocks and, in its last int, the view's survivor count, which mvsf_fusion_extract reads.
 * Bad arguments (null pointer, H W outside [1, 2^31), V outside [1, 16], a view index outside [0, N), method not 0 / 1):
 * -1; short workspace: -3; nothing launched. */
int mvsf_fusion_workspace_bytes(int H, int W, size_t* bytes);
/* The inverses the un-projections need (idx_img2cam / idx_cam2world, fusion.py:23-34, invert per call): cams_inv
 * [N][2][4][4], slot 0 = E^-1, slot 1 = K^-1 (4x4 with K in its [:3][:3]), fp64 rounded once; NaN if singular. */
int mvsf_fusion_prepare_cameras(const float* cams, int N, float* cams_inv, mvsf_stream_t stream);
/* method 0 = pcd: the source-confidence masking of test.py:397-400, get_reproj, vis_filter, ave_fusion (fusion.py:79-112)
 * and the masks of test.py:402-408 (uses conf, thres_view, thres_disp).  method 1 = dpcd: get_reproj_dynamic,
 * vis_filter_dynamic (fusion.py:114-165) and the voting of test.py:471-480 (uses conf, dist_base, rel_diff_base).
 * src: V view indices in HOST memory.  -> mask u8 [H][W] (0 / 1), depth_avg [H][W], workspace as above. */
int mvsf_fusion_filter(int method, const float* depths, const float* confs, const float* cams, const float* cams_inv, int N,
                       int ref, const int* src, int V, int H, int W, float conf, float thres_view, float thres_disp,
                       float dist_base, float rel_diff_base, unsigned char* mask, float* depth_avg, void* workspace,
                       size_t workspace_bytes, mvsf_stream_t stream);
/* test.py:410-424 (484-497): the world points of the averaged depth (idx_img2cam + idx_cam2world) and uint8(image * 255)
 * of the masked pixels, in row-major pixel order.  cam_inv: the reference view's [2][4][4] of cams_inv; image [3][H][W]
 * fp32 in [0, 1]; xyz [capacity][3], rgb [capacity][3]; survivors beyond capacity are not written. */
int mvsf_fusion_extract(const unsigned char* mask, const float* depth_avg, const void* workspace, size_t workspace_bytes,
                        const float* cam_inv, const float* image, float* xyz, unsigned char* rgb, long long capacity, int H,
                        int W, mvsf_stream_t stream);

/* ---- gipuma fusion: probability_filter (misc/gipuma.py:160-177) and fusibile's cross-view voting and point averaging
 *      at normal_thresh = 360 (test.py's default filter_method).  Reference views are stepped one at a time, in index
 *      order: mvsf_fusion_gipuma_vote then mvsf_fusion_gipuma_emit per view, with one used-mark map for the scene.
 * depth [N][H][W] (filtered), used [N][H][W] u8 (zero before view 0), cam_table [N][32] fp32; the workspace is that of
 * mvsf_fusion_workspace_bytes.  N is bounded only by memory: the table is read from global memory with 64-bit offsets.
 * Bad arguments (null pointer, H W outside [1, 2^31), ref outside [0, N), num_consistent < 0): -1; short workspace: -3;
 * nothing launched. */
/* depth = depths where conf > prob_threshold and depth_min <= depths <= depth_max, else 0; cam_table per view: P = K E[:3]
 * (12, row-major), M^-1 of M = P[:, :3] (9, row-major), f b (f = K[0][0] / K[2][2], b = 0.54), padding; fp64 rounded once. */
int mvsf_fusion_gipuma_prepare(const float* depths, const float* confs, const float* cams, int N, int H, int W,
                               float prob_threshold, float depth_min, float depth_max, float* depth, float* cam_table,
                               mvsf_stream_t stream);
/* Reference view ref: a valid, unused pixel survives when at least num_consistent other views are consistent with it
 * (the pixel's world point lands on a valid source pixel within disp_threshold in disparity).  -> mask u8 [H][W] and the
 * workspace's scanned survivor counts, the view's survivor count in its last int. */
int mvsf_fusion_gipuma_vote(const float* depth, const unsigned char* used, const float* cam_table, int N, int ref, int H, int W,
                            float disp_threshold, int num_consistent, unsigned char* mask, void* workspace,
                            size_t workspace_bytes, mvsf_stream_t stream);
/* The survivors of the vote, in row-major pixel order: xyz [capacity][3] the mean of the pixel's world point and those of
 * its consistent source pixels, rgb [capacity][3] the integer mean of round(255 image) over the same pixels (images
 * [N][3][H][W] fp32 in [0, 1]); each consistent source pixel is marked used.  Survivors beyond capacity write no point. */
int mvsf_fusion_gipuma_emit(const float* depth, const float* cam_table, const float* images, int N, int ref, int H, int W,
                            float disp_threshold, const unsigned char* mask, const void* workspace, size_t workspace_bytes,
                            unsigned char* used, float* xyz, unsigned char* rgb, long long capacity, mvsf_stream_t stream);

/* ---- image preparation of the eval loader, datasets/general_eval.py:112-131 (read_img's edge pad, scale_mvs_input's
 *      cv2.resize) and :210-211 (ToTensor + Normalize), bit-exact.  Images are uint8 RGB, channels-last [H][W][3].
 * src [N][h][w][3] (one source size) -> dst [N][H][W][3]: pad_rows rows repeated at the top and the bottom (the edge pad
 * of np.pad), then cv2.resize(img, (W, H)) with INTER_LINEAR as cv2 computes it for uint8 (equal sizes: a copy).
 * Bad arguments (null pointer, a size < 1, pad_rows < 0, 2^31 pixels or more per image): -1; nothing launched. */
int mvsf_image_resize_u8(const unsigned char* src, int N, int h, int w, int pad_rows, unsigned char* dst, int H, int W,
                         mvsf_stream_t stream);
/* The V images views[0..V) (indices in HOST memory, V in [1, 64]) of scene [N][H][W][3] -> norm [V][3][H][W] =
 * (u8 / 255 - mean) / std with the ImageNet mean and std, and colour [V][3][H][W] = trunc(clip((norm std + mean) 255, 0,
 * 255)) / 255, the colour test.py:287-292 saves for fusion before its JPEG encode.  Either output may be NULL, not both.
 * Bad arguments (null pointer, V outside [1, 64], a view outside [0, N), H W outside [1, 2^31)): -1; nothing launched. */
int mvsf_image_normalize(const unsigned char* scene, int N, const int* views, int V, int H, int W, float* norm,
                         float* colour, mvsf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MVSF_B200_H */
