/* dinounet_b200 — C-ABI of the H100-native Dino U-Net forward path.
 *
 * Plain pointers and sizes only (no torch types).  Every function launches hand-written sm_90a kernels on the
 * given CUDA stream, never allocates, never synchronises, and returns 0 on success or a negative error code
 * (message via b2u_last_error()).  All device tensors are channels-last ("token-major"): [rows, C] with C contiguous.
 *
 * Reference interface each entry replaces (paths relative to the reference repo root):
 *   - the reference's ONLY native FFI is the pybind11 module `MultiScaleDeformableAttention`
 *     (dinounet/dinov3/eval/segmentation/models/utils/ops/src/vision.cpp:18-21, ms_deform_attn.h:26-67);
 *     b2u_msda_forward is its drop-in (same tensor meaning, fused softmax/location prologue available).
 *   - every other entry replaces an ATen/cuDNN/cuBLAS library call that the reference's Python forward makes
 *     (SURVEY.md section 2.3); the call site is cited per function.
 */
#ifndef DINOUNET_B200_H_
#define DINOUNET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* b2u_stream_t; /* cudaStream_t */

enum { B2U_F16 = 0, B2U_BF16 = 1 };
enum { B2U_ACT_NONE = 0, B2U_ACT_GELU = 1, B2U_ACT_RELU = 2, B2U_ACT_LRELU = 3,
       /* act1 = B2U_ACT_SWIGLU (SwiGLUFFN.forward, ffn_layers.py:73-77): Wp rows (and bias) are packed in 32-row blocks
        * [w1 rows 32j..32j+31 | w2 rows 32j..32j+31], N = 2*hidden; out[:, j] = silu(x.w1_j + b1_j) * (x.w2_j + b2_j),
        * 16-bit [M, N/2] (ldc/col_off in output columns). */
       B2U_ACT_SWIGLU = 4 };
enum { B2U_CONV_NONE = 0, B2U_CONV3X3_S1 = 1, B2U_CONV3X3_S2 = 2 };

/* Epilogue applied to each fp32 accumulator element acc[m, n], in this order:
 *   v = acc + bias[n]; if (round16) v = round_to_dtype(v); v = act1(v); v = v * scale[n] + shift[n]; v = act2(v);
 *   v += residual[orow, ocol] (fp32) ; v += add16[orow, ocol] (16-bit) ; out[orow, ocol] = v
 * (orow, ocol) = output addressing: identity, batch row-remap, or 2x2 pixel-shuffle (ConvTranspose2d k2 s2). */
typedef struct b2u_epilogue {
  void* out;            /* 16-bit (dtype) or fp32 */
  int32_t out_fp32;     /* 1: out is float */
  int64_t ldc;          /* output row stride, elements */
  int32_t col_off;      /* output column offset (concat buffers) */
  int32_t rows_in;      /* row remap: orow = (m / rows_in) * rows_out + row_off + m % rows_in ; 0 = identity */
  int32_t rows_out;
  int32_t row_off;
  int32_t ps_cout;      /* >0: pixel-shuffle store, n = q*ps_cout + co, q = 2*a + b, input pixel grid ps_h x ps_w */
  int32_t ps_h;
  int32_t ps_w;
  const float* bias;    /* [N] or NULL */
  const float* scale;   /* [N] or NULL */
  const float* shift;   /* [N] or NULL */
  int32_t act1;
  int32_t act2;
  int32_t round16;
  const float* residual; /* fp32 [*, ldres], may alias out */
  int64_t ldres;
  const void* add16;     /* 16-bit [*, ldadd] */
  int64_t ldadd;
} b2u_epilogue;

/* wgmma tensor-core GEMM / implicit-GEMM 3x3 convolution:  acc[M, N] = A[M, K] * Wp[N, K]^T.
 * conv == NONE : A is [M, K] row-major (row stride lda).  Replaces F.linear / 1x1 Conv2d / ConvTranspose2d(k2,s2)
 *                (attention.py:88-90, ffn_layers.py:43-49, ms_deform_attn.py:183-215, dinov3_adapter.py:274-277,467,
 *                dinounet_training.py:419-441,255-264,613).
 * conv != NONE : A is an NHWC image [B, Hin, Win, C]; the kernel walks the 9 taps with TMA halo tiles (zero fill),
 *                no im2col buffer.  Wp is [N, 9*Cpad] with k = tap*Cpad + c, Cpad = ceil(C/64)*64.  Output pixel
 *                grid is Hin/stride x Win/stride.  Replaces Conv2d(3x3,pad 1) (dinov3_adapter.py:239-273,
 *                dynamic_network_architectures ConvDropoutNormReLU). */
typedef struct b2u_gemm_params {
  int32_t M, N, K;
  const void* A;
  int64_t lda;
  const void* Wp;       /* packed weights [N, ldw], 16-bit, zero padded */
  int64_t ldw;
  int32_t dtype;        /* B2U_F16 / B2U_BF16 for A, Wp and 16-bit outputs */
  int32_t conv;
  int32_t B, Hin, Win, C;
  b2u_epilogue epi;
} b2u_gemm_params;

int b2u_gemm(const b2u_gemm_params* p, b2u_stream_t stream);

/* QKV projection with masked bias + RoPE + head split fused in the epilogue (attention.py:30-40,66-92):
 *   qkv = A[M=B*ntok, D] * Wp[3D, D]^T + bias (already multiplied by bias_mask); rounded to dtype; q,k rows with
 *   token index >= prefix rotated with sin/cos[(tok - prefix), hd] (fp32); written as q,k,v [B, heads, ntok, hd],
 *   hd = D / heads = 64 (ViT-S/B/L) or 128 (ViT-7B). */
typedef struct b2u_qkv_params {
  int32_t B, ntok, D, heads, prefix;
  const void* A;
  int64_t lda;
  const void* Wp;
  int64_t ldw;
  const float* bias;    /* [3D] or NULL */
  const float* rope_sin;
  const float* rope_cos;
  void* q;
  void* k;
  void* v;
  int32_t dtype;
  int32_t v_transposed; /* 1: write V as V^T [B, heads, 64, npad] (keys contiguous) for b2u_attention_tc */
  int32_t npad;         /* row length of V^T: multiple of 8, >= ntok; columns >= ntok are never written (keep them 0) */
  int32_t rope_w;       /* > 0: the rope tables describe an (ntok-prefix)/rope_w x rope_w patch grid with separable angles
                           (rope_position_encoding.py:99-104: first 16 of 32 angles depend on the row, last 16 on the column,
                           tiled twice) -> the kernel keeps compact per-row / per-column tables in shared memory */
} b2u_qkv_params;

int b2u_qkv_rope(const b2u_qkv_params* p, b2u_stream_t stream);

/* wgmma flash attention, non-causal softmax attention (attention.py:106-118 -> F.scaled_dot_product_attention):
 * q,k [B, heads, ntok, 64], vt = V^T [B, heads, 64, npad]
 * with zero padding columns (see b2u_qkv_params.v_transposed) -> out [B, ntok, heads*64].  Only the query rows
 * [q_begin, ntok) are produced (128-row tiles, one per CTA); keys always span [0, ntok).  With q_begin = the
 * number of cls/storage tokens the ViT's 1024 patch rows fill whole tiles and b2u_attention_rows does the prefix. */
int b2u_attention_tc(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads, int32_t ntok,
                     int32_t npad, int32_t q_begin, float scale, int32_t dtype, b2u_stream_t stream);

/* Same kernel for head_dim 64 or 128 (ViT-7B: q,k [B, heads, ntok, 128], vt [B, heads, 128, npad]); all query rows. */
int b2u_attention_tc_hd(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads, int32_t ntok,
                        int32_t npad, int32_t head_dim, float scale, int32_t dtype, b2u_stream_t stream);

/* Few-row attention (same layouts as b2u_attention_tc): query rows [row_begin, row_begin + nrows), one warp per row,
 * fp32 softmax.  Meant for the handful of prefix-token rows. */
int b2u_attention_rows(const void* q, const void* k, const void* vt, void* out, int32_t B, int32_t heads, int32_t ntok,
                       int32_t npad, int32_t row_begin, int32_t nrows, float scale, int32_t dtype, b2u_stream_t stream);

/* LayerNorm over the last dim (block.py:193-194, vision_transformer.py:300, dinov3_adapter.py:142-148):
 *   in fp32 [rows_sel, D] -> out (16-bit or fp32).  Row selection: for output row r,
 *   input row = (r / rows_out) * rows_in + row_off + r % rows_out  (rows_out == 0: identity). */
int b2u_layernorm(const float* in, void* out, const float* gamma, const float* beta, int32_t rows, int32_t D,
                  float eps, int32_t rows_in, int32_t rows_out, int32_t row_off, int32_t out_fp32, int32_t dtype,
                  b2u_stream_t stream);
/* Same, for a 16-bit input stream `in` (element type = dtype). */
int b2u_layernorm16(const void* in, void* out, const float* gamma, const float* beta, int32_t rows, int32_t D,
                  float eps, int32_t rows_in, int32_t rows_out, int32_t row_off, int32_t out_fp32, int32_t dtype,
                  b2u_stream_t stream);

/* fp32 -> 16-bit cast of a [rows, D] matrix with the same row selection as b2u_layernorm. */
int b2u_cast_rows(const float* in, void* out, int32_t rows, int32_t D, int32_t rows_in, int32_t rows_out,
                  int32_t row_off, int32_t dtype, b2u_stream_t stream);
/* 16-bit -> 16-bit row gather with the same row selection (no conversion). */
int b2u_copy_rows16(const void* in, void* out, int32_t rows, int32_t D, int32_t rows_in, int32_t rows_out,
                    int32_t row_off, b2u_stream_t stream);

/* Patch-embed operand: x fp32 NCHW [B,3,S,S] -> [B*(S/16)^2, 768] 16-bit with k = c*256 + ky*16 + kx
 * (non-overlapping patches: a permutation + cast, no duplication)  (patch_embed.py:64-76). */
int b2u_patchify(const float* x, void* out, int32_t B, int32_t S, int32_t dtype, b2u_stream_t stream);

/* cls/storage prefix rows of the token stream: X[b, t, :] = prefix[t, :] for t < n_prefix (vision_transformer.py:207-214). */
int b2u_write_prefix(float* X, const float* prefix, int32_t B, int32_t ntok, int32_t n_prefix, int32_t D,
                     b2u_stream_t stream);

/* SPM stem conv0: Conv2d(3,64,3,s2,p1,no bias)+BN(eval)+ReLU reading fp32 NCHW, writing NHWC 16-bit
 * (dinov3_adapter.py:241-243).  w is [64,3,3,3] fp32; scale/shift = folded BN. */
int b2u_stem_conv0(const float* x, const float* w, const float* scale, const float* shift, void* out, int32_t B,
                   int32_t S, int32_t dtype, b2u_stream_t stream);

/* MaxPool2d(3, s2, p1) on NHWC 16-bit (dinov3_adapter.py:250). */
int b2u_maxpool3x3s2(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t dtype,
                     b2u_stream_t stream);

/* Depthwise 3x3 (pad 1) + bias (+GELU) on NHWC 16-bit.  `planes` > 1 processes the ConvFFN token stream
 * [B, 21n, C] as three planes (2h x 2w, h x w, h/2 x w/2) with shared weights (dinov3_adapter.py:99-109);
 * planes == 1 is a plain [B,H,W,C] image (dinounet_training.py:241-243).  w is tap-major [9, C] fp32. */
int b2u_dwconv3x3(const void* in, void* out, const float* w, const float* bias, int32_t B, int32_t H, int32_t W,
                  int32_t C, int32_t planes, int32_t act, int32_t dtype, b2u_stream_t stream);

/* MultiScaleDeformableAttention forward, single level, n_heads x n_points, fused prologue
 * (ms_deform_attn.py:185-213 + ms_deform_im2col_cuda.cuh:242-304):
 *   value  [B, Hv*Wv, heads, dh] 16-bit;  offaw fp32 [B*Lq, heads*points*3] = (offsets(x,y) | attention logits);
 *   reference point of query q = cell centre of q in the pyramid of (2Hv x 2Wv, Hv x Wv, Hv/2 x Wv/2) grids;
 *   loc = ref + off / (Wv, Hv); weights = softmax over points; bilinear, zero padding, align_corners=False.
 *   out [B*Lq, heads*dh] 16-bit. */
int b2u_msda_forward(const void* value, const float* offaw, void* out, int32_t B, int32_t Hv, int32_t Wv,
                     int32_t heads, int32_t dh, int32_t points, int32_t dtype, b2u_stream_t stream);

/* Drop-in for the reference pybind op `ms_deform_attn_forward` (ops/src/vision.cpp:18, ms_deform_attn.h:26-45):
 * value fp32 [B, S, heads, dh]; spatial_shapes int64 [levels, 2] (H, W) and level_start_index int64 [levels] on the
 * DEVICE (as in the reference); sampling locations fp32 [B, Lq, heads, levels, points, 2]; attention weights fp32
 * [B, Lq, heads, levels, points]; out fp32 [B, Lq, heads*dh].  (im2col_step is a launch-chunking detail of the
 * reference kernel and has no equivalent here.) */
int b2u_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                         const float* loc, const float* attw, float* out, int32_t B, int32_t S, int32_t Lq,
                         int32_t heads, int32_t dh, int32_t levels, int32_t points, b2u_stream_t stream);

/* Drop-in for the reference pybind op `ms_deform_attn_backward` (ops/src/vision.cpp:19, ms_deform_attn.h:48-67; the one
 * native kernel the reference's training step runs, ms_deform_attn.py:58-66).  Same inputs as the forward plus
 * grad_out fp32 [B, Lq, heads*dh]; writes grad_value [B, S, heads, dh] (zeroed here, then accumulated),
 * grad_loc [B, Lq, heads, levels, points, 2] and grad_attw [B, Lq, heads, levels, points], all fp32, caller-owned.
 * grad_value is accumulated with fp32 atomics (as in the reference kernel): summation order is not fixed. */
int b2u_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                          const float* loc, const float* attw, const float* grad_out, float* grad_value,
                          float* grad_loc, float* grad_attw, int32_t B, int32_t S, int32_t Lq, int32_t heads,
                          int32_t dh, int32_t levels, int32_t points, b2u_stream_t stream);

/* ---- Sliding-window prediction (inference/predict_from_raw_data.py:537-621, sliding_window_prediction.py:11-56).
 * tile_desc: DEVICE int32 [n_entries][4] = (slice d, y0, x0, flip bits: 1 = rows / tensor dim 2, 2 = cols / dim 3).
 * b2u_sw_gather_tiles: volume fp32 [Cin, D, H, W] -> batch fp32 [n_entries, 3, th, tw]; crops, mirrors and applies the
 *   1/2/>3 -> 3 channel rule of DINOv3EncoderAdapter.forward (dinounet_training.py:491-497).
 * b2u_sw_accumulate: one tile whose mirror variants are logits[first .. first+nvar) (fp32 [n, C, th, tw], variant 0
 *   unflipped, nvar in {1,2,4}): un-mirror, mean over variants, * gaussian (fp16 [th, tw], NULL = 1), accumulate into
 *   acc fp16 [C, D, H, W] and npred fp16 [D, H, W] with the reference's fp16 rounding sequence (:545-551, :598-599).
 *   Launches for overlapping tiles must be stream-ordered.
 * b2u_sw_finalize: acc /= npred (:601); *inf_flag |= 1 if any result is inf (:603-606 raises). */
int b2u_sw_gather_tiles(const float* volume, float* batch, const int32_t* tile_desc, int32_t n_entries, int32_t Cin,
                        int32_t D, int32_t H, int32_t W, int32_t th, int32_t tw, b2u_stream_t stream);
int b2u_sw_accumulate(const float* logits, const int32_t* tile_desc, int32_t first, int32_t nvar, const void* gaussian,
                      void* acc, void* npred, int32_t C, int32_t D, int32_t H, int32_t W, int32_t th, int32_t tw,
                      b2u_stream_t stream);
int b2u_sw_finalize(void* acc, const void* npred, int32_t C, int64_t plane, int32_t* inf_flag, b2u_stream_t stream);

/* ---- Prediction export (inference/export_prediction.py:15-68), the two device steps before the host paste.
 * b2u_export_resample_f16: fp16 [C, Z, h, w] -> fp16 [C, Z, H, W], Z unchanged: the 2D configuration's
 *   `resampling_fn_probabilities` (resample_data_or_seg_to_shape, order 1; default_resampling.py), i.e. scipy
 *   ndimage.zoom(order=1, mode='nearest', grid_mode=True) in fp64 with scipy's exact coordinate and weight arithmetic,
 *   rounded to fp16 to nearest even.  Bit-identical to the reference for finite logits; h == H && w == W copies `in`
 *   (the reference returns the array unchanged).  `in` and `out` must not overlap otherwise.
 * b2u_export_segment: fp16 logits [C, voxels], 1 <= C <= 32.  mode 0 (label maps): fp32 softmax over C, labels = index
 *   of the first maximum probability.  mode 1 (regions): fp32 sigmoid, labels = region_labels[i] (DEVICE int32 [C]) of
 *   the last channel i with p > 0.5, else 0 (label_handling.py:128-175).  labels: uint8 (label_bytes 1) or uint16 (2)
 *   [voxels]; probs: fp32 [C, voxels], written only when non-NULL.  No atomics: repeated launches give identical bits. */
int b2u_export_resample_f16(const void* in, void* out, int32_t C, int32_t Z, int32_t h, int32_t w, int32_t H, int32_t W,
                            b2u_stream_t stream);
int b2u_export_segment(const void* logits, int32_t C, int64_t voxels, int32_t mode, const int32_t* region_labels,
                       void* labels, int32_t label_bytes, float* probs, b2u_stream_t stream);

/* ---- Case preprocessing (preprocessing/preprocessors/default_preprocessor.py:40-118 `run_case_npy` of a 2D
 * configuration), fp32 channels in the caller's memory.  Bit-identical to numpy / scipy for finite input.
 * b2u_pre_minmax_f32: lo_hi[0..1] = exact min / max of x[n]; *nonfinite = 1 if x holds a NaN or an infinity (left
 *   untouched otherwise; may be NULL).  work: 2 * ceil(n / 65536) floats.
 * b2u_pre_zscore: ZScoreNormalization (default_normalization_schemes.py:27-50) in place on x[n]: numpy's float32 mean and
 *   std as ONE pairwise sum (numpy's pairwise_sum tree) over the elements in the order (i0, i1, i2) -> x[i0*s0 + i1*s1 +
 *   i2*s2], n = n0*n1*n2 (memory order: 1, 1, n, 0, 0, 1; use_mask_for_norm gathers in the transposed view's order);
 *   stats[0] = mean, stats[1] = max(std, 1e-8f), both left on the device.  work: ceil(n / 8) floats.
 * b2u_pre_normalize: scheme 1 CTNormalization x = (clip(x, a, b) - c) / d; 2 RescaleTo01 x = (x - stats[0]) /
 *   max(stats[1] - stats[0], 1e-8f) with stats the device [min, max] of x; 3 RGBTo01 x = x / 255.
 * b2u_pre_resample3: resample_data_or_seg_to_shape(order=3) of one channel (default_resampling.py:77-216), Z unchanged:
 *   x is the normalized channel as a [Z, h, w] view (element strides sz, sy, sx: the transpose is folded into the read),
 *   out fp32 [Z, H, W] contiguous.  three_d 0: separate z along axis 0, a 2-D resize per slice; 1: one 3-D resize.  Each
 *   is skimage resize(order=3, mode='edge') = scipy ndimage.zoom(order=3, mode='nearest', grid_mode=True) in fp64 with
 *   scipy's arithmetic, clipped to the slice's (0) or channel's (1) [min, max], rounded once to fp32.  consts: HOST
 *   array of 15 doubles, per axis (z, y, x) {pole, pole^n, gain, pole / (1 - pole^2n), pole / (pole - 1)} with n the
 *   padded length (Z + 24 or unused, h + 24, w + 24).  work: b2u_pre_resample3_work_doubles(Z, h, w, three_d) doubles.
 * b2u_pre_ensemble_f16: fold ensemble in fp16 as torch's CPU ops: acc = fp16(fp32(acc) + fp32(x)) when x != NULL, then
 *   acc = fp16(fp32(acc) / divisor) when divisor > 0.  acc, x: fp16 [n]. */
int b2u_pre_minmax_f32(const float* x, int64_t n, float* work, float* lo_hi, int32_t* nonfinite, b2u_stream_t stream);
int b2u_pre_zscore(float* x, int64_t n, int32_t n0, int32_t n1, int32_t n2, int64_t s0, int64_t s1, int64_t s2,
                   float* work, float* stats, b2u_stream_t stream);
int b2u_pre_normalize(float* x, int64_t n, int32_t scheme, const float* stats, float a, float b, float c, float d,
                      b2u_stream_t stream);
int64_t b2u_pre_resample3_work_doubles(int32_t Z, int32_t h, int32_t w, int32_t three_d);
int b2u_pre_resample3(const float* x, int32_t Z, int32_t h, int32_t w, int64_t sz, int64_t sy, int64_t sx, int32_t H,
                      int32_t W, int32_t three_d, const double* consts, double* work, float* out, b2u_stream_t stream);
int b2u_pre_ensemble_f16(void* acc, const void* x, int64_t n, int32_t divisor, b2u_stream_t stream);

/* ---- Evaluation of predictions against the ground truth (evaluation/evaluate_predictions.py:152-230
 * `compute_metrics`, HD95 / ASD as medpy's hd95 / asd).  Volumes are C-contiguous [Z, Y, X] (a mask of rank 1 or 2 is
 * padded with leading axes of size 1, and `ndim` names its true rank).
 * b2u_eval_masks: one label or region (labels: HOST int64 [n_labels], 1 <= n_labels <= B2U_EVAL_MAX_REGION_LABELS):
 *   mask = any(seg == labels[j]) with numpy's `==` (exact for the integer dtypes; float32 volumes compare with the
 *   label rounded to float32); border_* = mask ^ binary_erosion(mask) with face connectivity along the true axes and
 *   out-of-range neighbours 0 (uint8 0/1 [Z*Y*X]); counts (DEVICE int64 [6], zeroed by the call) = TP, FP, FN, TN over
 *   the voxels whose reference is not ignore_label (when has_ignore), then the populations of the reference and
 *   prediction masks over all voxels.  ref_dtype / pred_dtype: B2U_EVAL_* codes; the two may differ.
 * b2u_eval_edt: dt = scipy distance_transform_edt(border == 0, sampling=(s0, s1, s2)) in float64: the distance of every
 *   voxel to the nearest border voxel (+inf when the border is empty).  Bit-identical to scipy at integer spacings.
 *   tmp: double [Z*Y*X]; scratch: int32 [Z*Y*X].  Rows are staged in shared memory, 20 bytes per voxel: X is limited to
 *   the device's opt-in shared memory per block / 20 (11,622 on an H100).
 * b2u_eval_sum_f64: work[0] = numpy's pairwise float64 sum of x[n] (np.add.reduce of a contiguous array).  work:
 *   ceil(n / 8) doubles. */
enum { B2U_EVAL_U8 = 0, B2U_EVAL_I8 = 1, B2U_EVAL_I16 = 2, B2U_EVAL_U16 = 3, B2U_EVAL_I32 = 4, B2U_EVAL_F32 = 5 };
#define B2U_EVAL_MAX_REGION_LABELS 8
int b2u_eval_masks(const void* ref, int32_t ref_dtype, const void* pred, int32_t pred_dtype, int32_t ndim, int32_t Z,
                   int32_t Y, int32_t X, const int64_t* labels, int32_t n_labels, int32_t has_ignore,
                   int64_t ignore_label, uint8_t* border_ref, uint8_t* border_pred, int64_t* counts,
                   b2u_stream_t stream);
int b2u_eval_edt(const uint8_t* border, int32_t Z, int32_t Y, int32_t X, double s0, double s1, double s2, double* tmp,
                 int32_t* scratch, double* dt, b2u_stream_t stream);
int b2u_eval_sum_f64(const double* x, int64_t n, double* work, b2u_stream_t stream);

/* ---- Keep-the-largest-component postprocessing (postprocessing/remove_connected_components.py:22-34
 * `remove_all_but_largest_component_from_segmentation`, acvl-utils' `remove_all_but_largest_component`).
 * b2u_pp_largest_component: mask = any(seg == labels[j]) with evaluation's comparison rule (labels: DEVICE int64
 *   [n_labels], ascending and distinct, n_labels >= 0); its components with full connectivity (26 neighbours on the
 *   C-contiguous [Z, Y, X] volume, Z*Y*X < 2^31; a lower-rank mask padded with leading unit axes); out = seg with every
 *   masked voxel whose component is smaller than the largest set to `background` (the stored element's bits in the
 *   low 1, 2 or 4 bytes).  Every component of the largest size is kept; an empty mask leaves out == seg.  dtype:
 *   B2U_EVAL_* code.  work: int32 [2 * Z*Y*X + 1] (the component forest, the sizes, the largest size). */
int b2u_pp_largest_component(const void* seg, int32_t dtype, int32_t Z, int32_t Y, int32_t X, const int64_t* labels,
                             int32_t n_labels, int64_t background, void* out, int32_t* work, b2u_stream_t stream);

/* ---- Training augmentation of 2-D batches (nnUNetTrainer.get_training_transforms, nnUNetTrainer.py:684-775, as
 * batchgenerators 0.25 runs it; dinounet_b200/augmentation.py writes the record and restates the draws).
 * b2u_aug_apply: data fp32 [B, C, h, w] and seg int16 [B, 1, h, w] at the initial patch size -> out fp32 [B, C, H, W]
 *   and target fp32 ([B, 1, H, W] label map, or [B, R, H, W] regions), h >= H, w >= W, B*C <= 65535.  rec: DEVICE
 *   double [B*C, B2U_AUG_REC], every decision of every transform (field layout in csrc/augmentation.cu).  consts: HOST
 *   double[5] {pole, pole^(h-1), pole^(w-1), gain, pole^2 - 1} of the spatial transform's spline prefilter (mirror
 *   boundaries).  seed keys the Gaussian noise (b2u_aug_noise_field).  regions: DEVICE int32 [R + 1 offsets, labels],
 *   region q is labels[offsets[q] .. offsets[q+1]); R = 0 writes the label map.  work: b2u_aug_work_bytes bytes.  No
 *   host synchronisation; the launch sequence does not depend on the record.
 * b2u_aug_noise_field: the standard-normal field the noise step adds (times its std), fp64 [B, C, n]: Philox4x32-10
 *   keyed by seed, counter (pixel / 2, channel, sample), Box-Muller on two 53-bit uniforms. */
#define B2U_AUG_REC 40
int64_t b2u_aug_work_bytes(int32_t B, int32_t C, int32_t h, int32_t w, int32_t H, int32_t W);
int b2u_aug_apply(const float* data, const int16_t* seg, int32_t B, int32_t C, int32_t h, int32_t w, int32_t H,
                  int32_t W, const double* rec, const double* consts, uint64_t seed, const int32_t* regions, int32_t R,
                  void* work, float* out, float* target, b2u_stream_t stream);
int b2u_aug_noise_field(uint64_t seed, int32_t B, int32_t C, int64_t n, double* out, b2u_stream_t stream);

/* ---- Dice + cross-entropy loss and online-validation statistics on the logits of the forward path
 * (training/loss/compound_losses.py:31-56 `DC_and_CE_loss`, dice.py:72-119 `MemoryEfficientSoftDiceLoss`,
 * robust_ce_loss.py:12-16, built at nnUNetTrainer.py:363-365; consumer nnUNetTrainer.py:961-1005 `validation_step`).
 * logits fp32 [B, C, plane] (plane = H*W), 2 <= C <= 32; target [B, plane] labels, target_kind 0 = uint8, 1 = int32,
 * 2 = int64, 3 = float32 (nnU-Net hands float label maps).  has_ignore: a pixel labelled ignore_label (any integer;
 * nnU-Net uses C) counts for nothing (compound_losses.py:21-22, 38-53; validation_step's mask, nnUNetTrainer.py:982-986);
 * without it ignore_label is not read.  work: caller-owned, b2u_dice_ce_work_doubles(B, C, plane, has_ignore) doubles,
 * shared by the three calls.  Deterministic (fixed reduction order, fp64 partials).
 * stats: one pass over logits and target;  *bad_label = 1 if a (valid) label is outside [0, C) (torch raises a device
 *   assert there);  batch_sums (NULL: not needed) fp64 [C][3] = (intersect, sum_pred, sum_gt) of every class over the
 *   valid pixels of the local batch, for the caller to all-reduce across data-parallel ranks (dice.py:106-110,
 *   AllGatherGrad) before the finalisation.
 * finalize: out3[0] = weight_ce*CE + weight_dice*dice, out3[1] = CE (mean over the valid pixels; 0 when there are none,
 *   as the reference skips it), out3[2] = dice term (-mean_c (2*sum(p*y)+smooth)/max(sum(y)+sum(p)+smooth, 1e-8); over
 *   the batch if batch_dice, background class skipped unless do_bg);  tp_fp_fn (optional) int64 [3][C] = hard tp / fp / fn
 *   of argmax(logits) vs target over the valid pixels, summed over the batch (get_tp_fp_fn_tn with axes (0,2,3)).
 * backward: grad_logits fp32 [B, C, plane] = *ce_scale * dCE/dlogits + *dice_scale * d(dice term)/dlogits, exactly 0 at
 *   ignored pixels.  ce_scale, dice_scale: device scalars (NULL: 1), e.g. the local incoming gradient and its sum over
 *   ranks (the backward of AllGatherGrad, ddp_allgather.py:43-48).
 * finalize and backward take the batch Dice from batch_sums when given (batch_dice = 0 ignores them: per-sample Dice
 * stays local), else from the per-sample sums in work, with the same result bits. */
int64_t b2u_dice_ce_work_doubles(int32_t B, int32_t C, int64_t plane, int32_t has_ignore);
int b2u_dice_ce_stats(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                      int32_t ignore_label, double* work, double* batch_sums, int32_t* bad_label, int32_t B, int32_t C,
                      int64_t plane, b2u_stream_t stream);
int b2u_dice_ce_finalize(double* work, const double* batch_sums, float* out3, int64_t* tp_fp_fn, int32_t B, int32_t C,
                         int64_t plane, int32_t has_ignore, float weight_ce, float weight_dice, int32_t batch_dice,
                         int32_t do_bg, float smooth, b2u_stream_t stream);
int b2u_dice_ce_backward(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                         int32_t ignore_label, const double* work, const double* batch_sums, float* grad_logits,
                         int32_t B, int32_t C, int64_t plane, float weight_ce, float weight_dice, int32_t batch_dice,
                         int32_t do_bg, float smooth, const float* ce_scale, const float* dice_scale,
                         b2u_stream_t stream);

/* ---- Region-based Dice + BCE (compound_losses.py:59-99 `DC_and_BCE_loss` with MemoryEfficientSoftDiceLoss on
 * sigmoid(logits), do_bg, built at nnUNetTrainer.py:356-361; validation_step's region branch :973-994).
 * logits fp32 [B, R, plane], 1 <= R <= 32; target [B, R + has_ignore, plane] of target_kind (as above), used as real
 * values; with has_ignore the last channel is the ignore channel: a pixel is valid where (1 - t_ign) != 0.
 * work: b2u_dice_bce_work_doubles(B, R, plane) doubles.  The same three calls as the label maps, except that batch_sums
 * fp64 [R][3] is required: the batch Dice comes from it only.  finalize: out3[1] = BCE (mean over B*R*plane; with has_ignore sum(bce * valid) / max(#valid pixels, 1e-8)),
 * out3[2] = -mean_r (2I+smooth)/max(G+P+smooth, 1e-8);  tp_fp_fn (optional) float [3][R] = sum over the batch of
 * pred*y*w, pred*(1-y)*w, (1-pred)*y*w with pred = sigmoid(z) > 0.5 and w = 1 - t_ign (1 without an ignore channel).
 * backward: grad = *ce_scale * dBCE/dlogits + *dice_scale * d(dice term)/dlogits (both scalars required). */
int64_t b2u_dice_bce_work_doubles(int32_t B, int32_t R, int64_t plane);
int b2u_dice_bce_stats(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore, double* work,
                       double* batch_sums, int32_t B, int32_t R, int64_t plane, b2u_stream_t stream);
int b2u_dice_bce_finalize(double* work, const double* batch_sums, float* out3, float* tp_fp_fn, int32_t B, int32_t R,
                          int64_t plane, float weight_ce, float weight_dice, int32_t batch_dice, int32_t has_ignore,
                          float smooth, b2u_stream_t stream);
int b2u_dice_bce_backward(const float* logits, const void* target, int32_t target_kind, int32_t has_ignore,
                          const double* work, const double* batch_sums, float* grad_logits, int32_t B, int32_t R,
                          int64_t plane, float weight_ce, float weight_dice, int32_t batch_dice, float smooth,
                          const float* ce_scale, const float* dice_scale, b2u_stream_t stream);

/* Adapter tail (dinov3_adapter.py:467-482): out[b,y,x,:] = BN_eval( base[b,y,x,:] + bilinear(tap[b,:,:,:] -> HxW) ).
 * base: fp32 token stream slice or 16-bit image (base_fp32), tap fp32 [B, Ht*Wt, D] (token-major), align_corners=False. */
int b2u_tail_fuse(const void* base, int32_t base_fp32, int64_t base_batch_stride, const float* tap, void* out,
                  const float* scale, const float* shift, int32_t B, int32_t H, int32_t W, int32_t Ht, int32_t Wt,
                  int32_t D, int32_t dtype, b2u_stream_t stream);

/* InstanceNorm statistics: sums[b, c, 0..1] = (sum x, sum (x - mean)^2) over the rows of image b (accumulated as shifted
 * sums around the image's first pixel: no cancellation when |mean| >> std).  x 16-bit [B*rows, C] with row
 * stride ldx (dinounet_training.py:400-401; ConvDropoutNormReLU norm).  Deterministic two-level reduction (no float
 * atomics): `work` holds >= b2u_in_stats_work_floats(B, rows, C) floats whose first B words are ticket counters that
 * must be ZERO before the first call (the kernel leaves them zero); a workspace may be shared by consecutive calls. */
int64_t b2u_in_stats_work_floats(int32_t B, int32_t rows, int32_t C);
int b2u_in_stats(const void* x, int64_t ldx, float* sums, float* work, int32_t B, int32_t rows, int32_t C, int32_t dtype,
                 b2u_stream_t stream);

/* InstanceNorm apply + LeakyReLU(0.01): y = lrelu((x - mean) * rstd * gamma + beta), biased variance, eps. */
int b2u_in_apply(const void* x, int64_t ldx, void* y, int64_t ldy, const float* sums, const float* gamma,
                 const float* beta, int32_t B, int32_t rows, int32_t C, float eps, int32_t dtype, b2u_stream_t stream);

/* FiLM: z[r, j] = gb[r, j] * zz[r, zoff + j] + gb[r, R + j]  (dinounet_training.py:427-429). */
int b2u_film(const void* gb, const void* zz, int64_t ldzz, int32_t zoff, void* z, int32_t rows, int32_t R,
             int32_t dtype, b2u_stream_t stream);

/* Squeeze-excitation gate + shortcut (dinounet_training.py:222-225,437-439):
 *   pooled[b,c] = mean_rows t ; g = sigmoid(W2 relu(W1 pooled + b1) + b2) ; out = t * g + sc. */
int b2u_se_gate(const float* sums, const float* w1, const float* b1, const float* w2, const float* b2, float* gate,
                int32_t B, int32_t C, int32_t Cr, int32_t rows, b2u_stream_t stream);
int b2u_se_apply(const void* t, const void* sc, int64_t ldsc, const float* gate, void* out, int32_t B, int32_t rows,
                 int32_t C, int32_t dtype, b2u_stream_t stream);

/* Final InstanceNorm + LeakyReLU + 1x1 segmentation head + argmax (dinounet_training.py:597,619; nnUNetTrainer.py:977):
 *   x 16-bit [B*rows, C]; logits NCHW fp32 [B, ncls, rows]; labels uint8 [B, rows] (may be NULL). */
int b2u_seg_head(const void* x, const float* sums, const float* gamma, const float* beta, float eps, const float* w,
                 const float* b, float* logits, uint8_t* labels, int32_t B, int32_t rows, int32_t C, int32_t ncls,
                 int32_t dtype, b2u_stream_t stream);

/* cudaMemsetAsync(ptr, 0, bytes) on the stream (statistics accumulators must be zeroed every forward). */
int b2u_zero(void* ptr, int64_t bytes, b2u_stream_t stream);

/* Tuning / A-B switches (b2u_set_option).  key 1 (B2U_OPT_MSDA_IMPL): 0 = shared-memory value-slab gather (default),
 * 1 = first-generation warp-per-query kernel.  key 5: 1 = programmatic dependent launch across the plan (default off).
 * key 7: 1 = no L2 prefetch of the next tile's residual rows in short-K GEMMs (default on). */
enum { B2U_OPT_MSDA_IMPL = 1 };
/* ---------------------------------------------------------------------------------------------------------------
 * fp32 parity tier (csrc/fp32_tier.cu): the same forward in IEEE fp32 with plain SIMT kernels, selected by
 * `DinoUNet.precision = "fp32"`.  It is the path held to north_star's 1e-5 against the reference's fp32 (CPU) forward;
 * it is not the benchmarked path.  All tensors fp32, same layouts as above (tokens [rows, C], images NHWC).
 * Epilogue of b2u_f32_gemm (same meaning as b2u_epilogue): v = acc + bias[n]; v = act1(v); v = v*scale[n] + shift[n];
 * v = act2(v); v += residual[orow, ocol]; out[orow, ocol] = v.  conv != 0: A is an NHWC image, W is [N, 9*Cpad].
 * A-row remap (a_rows_in > 0): arow = (m / a_rows_in) * a_rows_out + a_row_off + m % a_rows_in. */
typedef struct b2u_f32_gemm_params {
  int64_t M;
  int32_t N, K;
  const float* A;
  int64_t lda;
  int32_t a_rows_in, a_rows_out, a_row_off;
  const float* W;
  int64_t ldw;
  int32_t conv, Hin, Win, C, Cpad;
  float* out;
  int64_t ldc;
  int32_t col_off;
  int32_t rows_in, rows_out, row_off;
  int32_t ps_cout, ps_h, ps_w;
  const float* bias;
  const float* scale;
  const float* shift;
  int32_t act1, act2;
  const float* residual;
  int64_t ldres;
  /* backward-pass addressing (csrc/train_bwd.cu callers): a_trans: A'(m, k) = A[k][m]; w_mode 1: W'(n, k) = W[k][n];
   * w_mode 2 (with conv != 0): 3x3 data gradient, W'(c, (tap', n)) = W[n][(8 - tap') * w_cpad + c];
   * w_mode 3 (with conv != 0, a_trans): 3x3 weight gradient, W is the layer's NHWC input, W'((tap, c), pixel) = its window;
   * ksplit > 1: the K range is split over gridDim.z and the raw products are atomically ADDED to out (zero it first);
   * accumulate: out += instead of out =. */
  int32_t a_trans, w_mode, w_cpad, ksplit, accumulate;
} b2u_f32_gemm_params;
int b2u_f32_gemm(const b2u_f32_gemm_params* p, b2u_stream_t stream);   /* F.linear / Conv2d 1x1, 3x3 / ConvTranspose2d k2 s2 */
/* Same parameter block, addressing modes and epilogue on the tensor cores (csrc/gemm_tf32.cu): operands rounded to TF32
 * (round-to-nearest, 10 mantissa bits = the fp16 autocast the reference trains under, nnUNetTrainer.py:899-929, with fp32's
 * exponent range), fp32 accumulation (wgmma kind tf32).  The fast tier of the TRAINING step's
 * matrix products (forward, data gradient, weight gradient of F.linear / Conv2d / ConvTranspose2d); not bit-comparable
 * with b2u_f32_gemm (about 1e-3 relative per product). */
int b2u_tf32_gemm(const b2u_f32_gemm_params* p, b2u_stream_t stream);
/* F.layer_norm; input row = (r / out_per_b) * in_per_b + in_off + r % out_per_b when in_per_b > 0 (ViT taps drop the prefix) */
int b2u_f32_layernorm(const float* in, float* out, const float* w, const float* b, int64_t rows, int32_t D, float eps,
                      int32_t in_per_b, int32_t out_per_b, int32_t in_off, b2u_stream_t stream);
int b2u_f32_patchify(const float* x_nchw, float* rows768, int32_t B, int32_t S, b2u_stream_t stream);   /* patch_embed.py:64-76 */
int b2u_f32_nchw_to_nhwc(const float* x, float* out, int32_t B, int32_t C, int64_t HW, b2u_stream_t stream);
int b2u_f32_seg_out(const float* lin, float* logits_nchw, uint8_t* labels, int32_t B, int64_t HW, int32_t ncls, b2u_stream_t stream);
int b2u_f32_maxpool3x3s2(const float* in, float* out, int32_t B, int32_t H, int32_t W, int32_t C, b2u_stream_t stream);
int b2u_f32_dwconv3x3(const float* in, float* out, const float* w9, const float* bias, int32_t B, int32_t H, int32_t W,
                      int32_t C, int32_t planes, int32_t act, b2u_stream_t stream);              /* dinov3_adapter.py:99-109 */
/* attention.py:66-118 on the fused qkv rows [B*N, 3D]: RoPE on tokens >= prefix, exact softmax, fp32 */
int b2u_f32_attention(const float* qkv, const float* rope_sin, const float* rope_cos, float* out, int32_t B, int32_t N,
                      int32_t heads, int32_t head_dim, int32_t prefix, float scale, b2u_stream_t stream);
int b2u_f32_msda(const float* value, const float* offaw, float* out, int32_t B, int32_t Hv, int32_t Wv, int32_t heads,
                 int32_t dh, b2u_stream_t stream);                                                 /* ms_deform_attn.py:158-216 */
/* InstanceNorm2d(affine) (+ LeakyReLU 0.01): work = 2*B*C doubles (scratch), stats = [B][C][2] floats (mean, rstd) out */
int b2u_f32_instnorm(const float* in, int64_t ld_in, float* out, int64_t ld_out, const float* w, const float* b, double* work,
                     float* stats, int32_t B, int64_t HW, int32_t C, float eps, int32_t lrelu, b2u_stream_t stream);
int b2u_f32_se(const float* t, const float* shortcut, int64_t ld_shortcut, float* pooled_work, const float* w1, const float* b1,
               const float* w2, const float* b2, float* out, int32_t B, int64_t HW, int32_t C, int32_t hidden, b2u_stream_t stream);
int b2u_f32_film(const float* gamma_beta, const float* zs_zp, float* z, int64_t px, int32_t R, b2u_stream_t stream);
int b2u_f32_tail(const float* c, int64_t c_rows_per_b, int64_t c_off, const float* tap, float* out, const float* bn_scale,
                 const float* bn_shift, int32_t B, int32_t r, int32_t h, int32_t D, b2u_stream_t stream);   /* dinov3_adapter.py:468-482 */

/* ---------------------------------------------------------------------------------------------------------------
 * Backward of the trainable part + optimizer (csrc/train_bwd.cu; SURVEY.md section 8f rank 2, BASELINE config 3).
 * fp32, same layouts as the fp32 tier.  Matrix-product gradients use b2u_f32_gemm (a_trans / w_mode / ksplit).  Every
 * parameter-gradient output is ACCUMULATED with atomics: zero it first.  Replaces ATen autograd kernels of
 * nnUNetTrainer.train_step (nnUNetTrainer.py:899-929); the one native backward op of the reference is b2u_msda_backward_f32. */
int b2u_f32_add(const float* a, const float* b, float* out, int64_t n, b2u_stream_t stream);
int b2u_f32_act(const float* x, float* y, int64_t n, int32_t act, b2u_stream_t stream);
int b2u_f32_act_bwd(const float* x_pre, const float* dy, float* dx, int64_t n, int32_t act, b2u_stream_t stream);
int b2u_f32_colsum(const float* in, int64_t ld, int64_t rows, int32_t C, float* out_accum, b2u_stream_t stream);
int b2u_f32_layernorm_bwd(const float* x, const float* w, const float* dy, float* dx, float* dw, float* db, int64_t rows,
                          int32_t D, float eps, b2u_stream_t stream);
int b2u_f32_instnorm_bwd(const float* x, int64_t ldx, const float* dy, int64_t lddy, const float* w, const float* b,
                         const float* stats, double* work, float* dx, int64_t lddx, float* dw, float* db, int32_t B, int64_t HW,
                         int32_t C, int32_t lrelu, b2u_stream_t stream);
/* eval-mode (Sync)BatchNorm + optional ReLU, forward and backward (the gradient oracle's semantics) */
int b2u_f32_bn_act(const float* x, float* y, const float* gamma, const float* beta, const float* running_mean,
                   const float* running_var, float eps, int64_t rows, int32_t C, int32_t act, b2u_stream_t stream);
int b2u_f32_bn_act_bwd(const float* x, const float* dy, const float* gamma, const float* beta, const float* running_mean,
                       const float* running_var, float eps, float* dx, float* dgamma, float* dbeta, int64_t rows, int32_t C,
                       int32_t act, b2u_stream_t stream);
int b2u_f32_dwconv_wgrad(const float* x, const float* dy, float* dw9, float* db, int32_t B, int32_t H, int32_t W, int32_t C,
                         int32_t planes, b2u_stream_t stream);
int b2u_f32_maxpool3x3s2_bwd(const float* x, const float* dy, float* dx_zeroed, int32_t B, int32_t H, int32_t W, int32_t C,
                             b2u_stream_t stream);
int b2u_f32_film_bwd(const float* gamma_beta, const float* zs_zp, const float* dz, float* dgb, float* dzz, int64_t px, int32_t R,
                     b2u_stream_t stream);
int b2u_f32_se_bwd(const float* t, const float* dy, const float* pooled, const float* w1, const float* b1, const float* w2,
                   const float* b2, float* work_3BC, float* dt, float* dw1, float* db1, float* dw2, float* db2, int32_t B,
                   int64_t HW, int32_t C, int32_t hidden, b2u_stream_t stream);
int b2u_f32_msda_prep(const float* offaw, float* loc, float* attw, int32_t B, int32_t Hv, int32_t Wv, int32_t heads, b2u_stream_t stream);
int b2u_f32_msda_prep_bwd(const float* attw, const float* dloc, const float* dattw, float* doffaw, int32_t B, int32_t Hv, int32_t Wv,
                          int32_t heads, b2u_stream_t stream);
int b2u_f32_unshuffle(const float* dy_image, int64_t ld, int32_t col_off, float* rows_4cout, int32_t B, int32_t h, int32_t w,
                      int32_t Cout, b2u_stream_t stream);
int b2u_f32_conv3x3_dgrad(const float* dy, const float* W, float* dx, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t Cpad,
                          int32_t N, int32_t stride, b2u_stream_t stream);
int b2u_f32_conv3x3_wgrad(const float* x, const float* dy, float* dW_accum, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t Cpad,
                          int32_t N, int32_t stride, b2u_stream_t stream);
int b2u_f32_sqsum(const float* g, int64_t n, double* out_accum, b2u_stream_t stream);
int b2u_f32_sgd_nesterov(float* p, const float* g, float* momentum_buf, int64_t n, float lr, float momentum, float weight_decay,
                         const double* grad_sqsum, float max_norm, int32_t first_step, b2u_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Train-mode semantics of the reference (csrc/train_mode.cu): batch-statistics (Sync)BatchNorm with the running-statistic
 * update, the extractors' DropPath residual and per-block RoPE tables with rescaled coordinates.  No atomics: every
 * reduction goes through fixed-order fp64 partials, so two identical launches give identical bits.
 *
 * BatchNorm training step on x [rows, C] (torch SyncBatchNorm in train mode):
 *   b2u_f32_bn_stats     sums[0:C] = sum x, sums[C:2C] = sum x^2, sums[2C] = rows (fp64; work: b2u_f32_bn_work_doubles).
 *                        Data-parallel callers all-reduce `sums` (all 2C+1 doubles) before the finalize.
 *   b2u_f32_bn_finalize  n = sums[2C]: batch mean and biased variance -> mean, var (fp32); running_mean/var <- (1-m)*r +
 *                        m*(mean | var*n/(n-1)); *num_batches_tracked += 1.  Normalise with b2u_f32_bn_act(mean, var).
 *   b2u_f32_bn_train_bwd_reduce  dy' = dy (ReLU-masked when act): red[0:C] = sum dy', red[C:2C] = sum dy' xhat,
 *                        red[2C] = rows; dgamma = sum dy' xhat, dbeta = sum dy' (written, local).  All-reduce `red` for sync.
 *   b2u_f32_bn_train_bwd_apply   dx = gamma*invstd*(dy' - red[c]/n - xhat*red[C+c]/n), n = red[2C]. */
int64_t b2u_f32_bn_work_doubles(int64_t rows, int32_t C);
int b2u_f32_bn_stats(const float* x, int64_t rows, int32_t C, double* work, double* sums, b2u_stream_t stream);
int b2u_f32_bn_finalize(const double* sums, int32_t C, float* mean, float* var, float* running_mean, float* running_var,
                        int64_t* num_batches_tracked, float momentum, b2u_stream_t stream);
int b2u_f32_bn_train_bwd_reduce(const float* x, const float* dy, const float* gamma, const float* beta, const float* mean,
                                const float* var, float eps, int64_t rows, int32_t C, int32_t act, double* work, double* red,
                                float* dgamma, float* dbeta, b2u_stream_t stream);
int b2u_f32_bn_train_bwd_apply(const float* x, const float* dy, const float* gamma, const float* beta, const float* mean,
                               const float* var, float eps, const double* red, float* dx, int64_t rows, int32_t C, int32_t act,
                               b2u_stream_t stream);
/* DropPath residual (dinov3_adapter.py:18-27): y = c + s[row / rows_per_sample] * f over [rows, D]; c == NULL gives
 * y = s * f (the backward of the branch). */
int b2u_f32_droppath_add(const float* c, const float* f, const float* s, float* y, int64_t rows, int32_t D,
                         int64_t rows_per_sample, b2u_stream_t stream);
/* Per-block RoPE tables (rope_position_encoding.py:57-106, 'separate' coordinates times scales[i]):
 * sin/cos [depth, h*w, head_dim] fp32 from periods [head_dim/4] and scales [depth] (device). */
int b2u_rope_tables(const float* periods, const float* scales, float* sin, float* cos, int32_t depth, int32_t h, int32_t w,
                    int32_t head_dim, b2u_stream_t stream);

int b2u_set_option(int32_t key, int32_t value);

const char* b2u_last_error(void);
int b2u_version(void);
/* Number of kernel launches issued through this library since load (bench.py's gpu_launches evidence). */
int64_t b2u_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DINOUNET_B200_H_ */
