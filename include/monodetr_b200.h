/*
 * monodetr_b200.h -- C ABI of libmonodetr_b200.so (H100 / sm_90a).
 *
 * Plain pointers and sizes only; every pointer is a DEVICE pointer unless its comment says HOST.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Every entry point is
 * asynchronous on `stream`, never synchronises, never creates streams, and returns 0 on success,
 * a positive cudaError_t value if the launch failed, or a negative MDB_E* code for bad arguments.
 * (The reference only printf()s launch errors -- ms_deform_im2col_cuda.cuh:948-952,1321-1325 -- the
 * host side of this library turns a non-zero return into a Python RuntimeError instead.)
 *
 * Reference interface each group replaces (paths relative to the reference checkout):
 *   mdb_msda_*          lib/models/monodetr/ops/src/vision.cpp:13-16  (pybind ms_deform_attn_forward/backward)
 *                       lib/models/monodetr/ops/src/ms_deform_attn.h:20-61 (dispatch)
 *                       lib/models/monodetr/ops/src/cuda/ms_deform_attn_cuda.cu:20-80, 83-153 (host launchers)
 *                       lib/models/monodetr/ops/src/cuda/ms_deform_im2col_cuda.cuh:237-299, 301-403 (kernels)
 */
#ifndef MONODETR_B200_H_
#define MONODETR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDB_EINVAL (-1)      /* bad size / null pointer / misaligned pointer */
#define MDB_EUNSUPPORTED (-2) /* shape outside what the kernels implement */
#define MDB_EWORKSPACE (-3)   /* scratch buffer missing / too small: see mdb_set_workspace */

/* Library/ABI version (bumped when a signature changes). */
int mdb_abi_version(void);
/* Human-readable name of the last error code returned on this thread ("ok" if 0). HOST string. */
const char* mdb_error_string(int code);

/* Reproducible mode (process-wide; default 0).  By default the MSDeformAttn value gradient (like the reference's kernel,
 * ms_deform_im2col_cuda.cuh:125-152), the split-K weight gradients, the norm-parameter gradients, the GroupNorm statistics, the
 * depth-map gradients of the heads and the depth tail's embedding gradient combine partial sums with float atomics, so results
 * differ in the last bits from run to run.  With 1, every floating-point output element has exactly one writer that adds its terms
 * in an order fixed by the problem shape (never by the SM count or the scheduling):
 *   - mdb_msda_backward_f32 / _f64 accumulate grad_value in (query, point, corner) order; mdb_msda_fused_backward_f32 returns
 *     MDB_EUNSUPPORTED (callers take mdb_msda_prep_* + mdb_msda_backward_*),
 *   - mdb_conv2d_wgrad_* run without split-K and mdb_colsum_f32 in one pass,
 *   - mdb_add_layernorm_backward_f32: dgamma / dbeta in a second launch (fixed row partition, combined in a thread-block cluster),
 *   - mdb_groupnorm_forward_f32 / _backward_f32: one CTA per (group, image) / per group writes the statistics and dgamma / dbeta,
 *   - mdb_head_depth_backward_f32 / mdb_depth_sample_backward_f32: the map gradient in gather form (a second launch for the former),
 *   - mdb_depth_tail_backward_f32: demb in a second launch, per (row, channel) over the pixels in pixel order,
 *   - mdb_sum_mean_squares_forward_f32 reduces in one CTA in tensor order.
 * Integer atomics (criterion counts, decode count) are exact and stay.  Guarantee: on the same GPU model with the same build, in
 * one process, two runs of a training iteration (forward with dropout, the device criterion, backward, mdb_adamw_step_f32) from
 * the same weights, optimizer state, inputs and dropout seed give identical bits, eagerly or as a replayed CUDA graph.  Not
 * covered: the reduction order of a multi-GPU all-reduce.  A test / debugging mode, several times slower (DESIGN.md section 5). */
int mdb_set_deterministic(int on);
int mdb_get_deterministic(void);

/* ---- Multi-scale deformable attention (MSDeformAttn core) -----------------------------------
 * value          (B, S, M, D)          contiguous
 * spatial_shapes (L, 2) int64 (H_l, W_l), device        [ms_deform_attn_cuda.cu:28-38 asserts the same]
 * level_start    (L,)   int64, device
 * sampling_loc   (B, Lq, M, L, P, 2)   (x, y) normalised to [0,1]
 * attn_weight    (B, Lq, M, L, P)
 * out            (B, Lq, M*D)          fully written by the call
 * Any B is accepted (the reference's im2col_step chunking, ms_deform_attn_cuda.cu:50-52, is not needed).
 */
int mdb_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                         const float* sampling_loc, const float* attn_weight,
                         int B, int S, int M, int D, int L, int Lq, int P,
                         float* out, void* stream);
int mdb_msda_forward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start,
                         const double* sampling_loc, const double* attn_weight,
                         int B, int S, int M, int D, int L, int Lq, int P,
                         double* out, void* stream);

/* Backward.  grad_value (B,S,M,D) is zero-filled by the call and then accumulated with atomics
 * (ms_deform_attn_cuda.cu:121-123 + cuh:125-152); grad_loc / grad_attn are fully written. */
int mdb_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                          const float* sampling_loc, const float* attn_weight, const float* grad_out,
                          int B, int S, int M, int D, int L, int Lq, int P,
                          float* grad_value, float* grad_loc, float* grad_attn, void* stream);
int mdb_msda_backward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start,
                          const double* sampling_loc, const double* attn_weight, const double* grad_out,
                          int B, int S, int M, int D, int L, int Lq, int P,
                          double* grad_value, double* grad_loc, double* grad_attn, void* stream);

/* Fused MSDeformAttn pre-processing (ops/modules/ms_deform_attn.py:145-155): sampling_locations and
 * softmax(attention logits) from the raw projections in one pass, and its backward.
 * off (B,Lq,M,L,P,2), logits (B,Lq,M,L*P), ref (B,Lq,L,ref_dim) contiguous, ref_dim in {2,6}; L*P <= 16.
 * backward: doff / dlogits from dloc / dattn (+ saved attn); the gradient wrt ref (only decoder layer 0 needs it)
 * is a plain reduction of dloc done by the caller. */
int mdb_msda_prep_forward_f32(const float* off, const float* logits, const float* ref, const int64_t* spatial_shapes,
                              int B, int Lq, int M, int L, int P, int ref_dim, float* loc, float* attn, void* stream);
int mdb_msda_prep_backward_f32(const float* dloc, const float* dattn, const float* attn, const float* ref,
                               const int64_t* spatial_shapes, int B, int Lq, int M, int L, int P, int ref_dim,
                               float* doff, float* dlogits, void* stream);

/* The module's forward with the pre-processing INSIDE the sampling kernels (constant reference points; D = 32, L = 4, P = 4,
 * otherwise MDB_EUNSUPPORTED): offsets (B,Lq,M,L,P,2) and logits (B,Lq,M,L*P) are the raw projections, ref (B,Lq,L,ref_dim).
 * backward: grad_value zero-filled then accumulated; grad_offsets / grad_logits fully written. */
int mdb_msda_fused_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* offsets,
                               const float* logits, const float* ref, int B, int S, int M, int D, int L, int Lq, int P, int ref_dim,
                               float* out, void* stream);
int mdb_msda_fused_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* offsets,
                                const float* logits, const float* ref, const float* grad_out, int B, int S, int M, int D, int L, int Lq,
                                int P, int ref_dim, float* grad_value, float* grad_offsets, float* grad_logits, void* stream);
/* mdb_msda_fused_backward_f32 for 6-d reference boxes that require a gradient (ref_dim == 6 only): also writes the box partials
 * ref_part (B,Lq,M,L,4) = [sum d loc_x, sum d loc_y, sum d loc_x off_x, sum d loc_y off_y] over each level's points, reduced in a
 * fixed order across the unit's lanes.  MDB_EUNSUPPORTED in reproducible mode, like mdb_msda_fused_backward_f32. */
int mdb_msda_fused_backward_ref_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                    const float* offsets, const float* logits, const float* ref, const float* grad_out, int B, int S,
                                    int M, int D, int L, int Lq, int P, int ref_dim, float* grad_value, float* grad_offsets,
                                    float* grad_logits, float* ref_part, void* stream);

/* ---- Tensor-core convolution / linear family (wgmma + TMA, fp32 storage, BF16x3 / TF32 math) ----
 * Replaces the cuDNN / cuBLAS calls behind nn.Conv2d / nn.Linear on the reference path
 * (backbone.py:100-102; monodetr.py:83-91; depth_predictor/depth_predictor.py:29-47;
 *  ops/modules/ms_deform_attn.py:138-161; depthaware_transformer.py:339-343,467-473).
 * Activations are NHWC fp32: x[B][H][W][Cin], y[B][Ho][Wo][Cout]; weights are "packed"
 * [kh*kw][Cout][Cin] (mdb_pack_conv_weight_f32).  A linear layer y[M,N] = x[M,K] w[N,K]^T is the call
 * with B=1, H=1, W=M, Cin=K, Cout=N, kh=kw=1, stride=1, pad=0 (w itself is already "packed").
 * Supported: kh=kw in {1,3}, stride in {1,2}, Cin%4==0, 16-byte aligned pointers; Cout%4==0 for dgrad / wgrad (the
 * forward writes any Cout, e.g. the 3-class / 81-bin head widths of monodetr.py:102-117); outputs below 2^31 elements.
 * The *_dilated entry points take a dilation d >= 1 after pad (torch.nn.Conv2d's dilation: taps d pixels apart, output
 * size (H + 2*pad - d*(kh-1) - 1)/stride + 1); d > 1 requires kh == kw == 3 and stride 1, and the weight gradient also
 * pad % d == 0 (the dilated C5 stage of torchvision's ResNets, backbone.py:100-106: pad == d); anything else returns
 * MDB_EUNSUPPORTED.  A dilated launch runs the same
 * tiles, k order and split-K decision as the undilated one of the same shape, so every statement below holds for it too
 * (the dilated weight gradient is the sum of d*d undilated ones over the dilation's pixel lattices, launched in turn);
 * with d == 1 they are the plain entry points.
 * Forward and dgrad store their output with TMA (staged in shared memory, residual or mask fetched by TMA) when the output
 * width is a multiple of 4 and y / dx, residual and relu_mask are 16-byte aligned, and from registers otherwise (e.g. the
 * odd head widths); both give the same bits.
 * Forward and dgrad are bit-reproducible run to run, and image b of a batch gets the same bits as the same image in any
 * other batch, in every precision mode.  wgrad accumulates its split-K partial sums with fp32 atomics.  A forward with
 * >= 256 k-blocks of 32 input channels (kh*kw*ceil(Cin/32); the 3x3 stride-2 2048->256 of monodetr.py:83-91), Cout > 64,
 * Cout % 4 == 0, no residual, no ReLU, a NULL or 16-byte aligned bias and precision mode 1 or 2 is split into
 * ceil(k-blocks/32) slices whatever the batch; the slices go through the scratch buffer the caller registers with
 * mdb_set_workspace (per device; the library itself never allocates or frees device memory) and are added in slice order.
 * The one exception to batch independence: when B*Ho*Wo*Cout*slices >= 2^31 that forward runs unsplit, so its bits match
 * a smaller batch's only while the product stays below 2^31 (below 3884 images for the 12x40 neck conv).
 * Below that bound mdb_conv2d_forward_workspace_bytes is B times a per-image size.
 */
/* Arithmetic of the tensor-core family (a process-wide numerical setting): 2 (default) = error-compensated BF16x3 (operands
 * split into bf16 hi + lo, A_hi*B_hi + A_lo*B_hi + A_hi*B_lo at twice the TF32 tensor rate, dropped terms ~2^-17 per product;
 * forward / dgrad take pre-split weights through mdb_pack_gemm_weights_bf16x3 and the *_bf16x3 entry points, wgrad splits both
 * activations on the fly; the _f32 forward / dgrad entry points run 3xTF32 in this mode); 1 = error-compensated 3xTF32
 * (A*B + A_lo*B + A*B_lo, ~fp32 accuracy); 0 = single-pass TF32 with round-to-nearest operands (cuDNN's allow_tf32 class). */
int mdb_set_precision(int mode);
int mdb_get_precision(void);
/* Split-K scratch of mdb_conv2d_forward_* for the CURRENT device (cudaGetDevice): the library never allocates device
 * memory.  Ask _workspace_bytes (0 = none needed; negative = MDB_E*), register a buffer at least that large that stays
 * valid while launches (or captured CUDA graphs) may use it; otherwise those shapes return MDB_EWORKSPACE. */
int mdb_set_workspace(void* buf, unsigned long long bytes);
long long mdb_conv2d_forward_workspace_bytes(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                             int flags, int has_residual, int split_weights);
/* Precision mode 2: weights split once per step into bf16 (hi, lo) pairs.  wf[tap][Cout][ceil(Cin/32)][hi 32 | lo 32] is the
 * forward operand, wd[tap][Cin][ceil(Cout/32)][hi 32 | lo 32] (the transposed weight) the dgrad operand; sizes in bf16
 * elements: taps*Cout*ceil(Cin/32)*64 and taps*Cin*ceil(Cout/32)*64.  n tensors per call, HOST arrays; scale (FrozenBN
 * fold, backbone.py:54-64) and wd may be NULL or hold NULL entries.  src_packed: 0 = OIHW sources (nn.Conv2d / nn.Linear
 * weights as stored), 1 = [tap][Cout][Cin] sources.  taps <= 9. */
int mdb_pack_gemm_weights_bf16x3(int n, const float* const* w, const float* const* scale, void* const* wf, void* const* wd,
                                 const int* O, const int* I, const int* taps, int src_packed, void* stream);
int mdb_conv2d_forward_bf16x3(const float* x, const void* w_split, const float* bias, const float* residual, float* y,
                              int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                              void* stream);
int mdb_conv2d_dgrad_bf16x3(const float* dy, const void* w_split_t, const float* residual, const float* relu_mask,
                            float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                            int flags, void* stream);
int mdb_conv2d_forward_f32(const float* x, const float* w_packed, const float* bias /*[Cout]|NULL*/,
                           const float* residual /*like y|NULL*/, float* y,
                           int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                           int flags /* bit0: ReLU, bit1: store y rounded-to-nearest TF32 */, void* stream);
/* dx = (conv_transpose(dy, w) + residual) * (relu_mask > 0); residual / relu_mask are shaped like dx or NULL. */
int mdb_conv2d_dgrad_f32(const float* dy, const float* w_packed, const float* residual, const float* relu_mask,
                         float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                         int flags /* bit1: store dx rounded-to-nearest TF32 */, void* stream);
/* dw_packed[tap][Cout][Cin] (+)= rowscale[co] * sum dy * x ; zero-filled first unless accumulate. */
int mdb_conv2d_wgrad_f32(const float* dy, const float* x, const float* rowscale /*[Cout]|NULL*/, float* dw_packed,
                         int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                         int accumulate, void* stream);
/* Same, plus db[Cout] (+)= sum over output pixels of dy: the bias gradient of nn.Conv2d / nn.Linear, produced by the
 * same launch (zero-filled first unless accumulate; db may sit directly behind dw_packed to share the memset). */
int mdb_conv2d_wgrad_bias_f32(const float* dy, const float* x, const float* rowscale /*[Cout]|NULL*/, float* dw_packed,
                              float* db /*[Cout]|NULL*/, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride,
                              int pad, int accumulate, void* stream);
/* Dilated twins of the forward / dgrad / wgrad / workspace calls above (see "Supported"): `dilation` follows `pad`. */
int mdb_conv2d_forward_dilated_bf16x3(const float* x, const void* w_split, const float* bias, const float* residual, float* y,
                                      int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                      int flags, void* stream);
int mdb_conv2d_forward_dilated_f32(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
                                   int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                   int flags, void* stream);
int mdb_conv2d_dgrad_dilated_bf16x3(const float* dy, const void* w_split_t, const float* residual, const float* relu_mask,
                                    float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                    int dilation, int flags, void* stream);
int mdb_conv2d_dgrad_dilated_f32(const float* dy, const float* w_packed, const float* residual, const float* relu_mask,
                                 float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                 int dilation, int flags, void* stream);
int mdb_conv2d_wgrad_bias_dilated_f32(const float* dy, const float* x, const float* rowscale /*[Cout]|NULL*/, float* dw_packed,
                                      float* db /*[Cout]|NULL*/, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride,
                                      int pad, int dilation, int accumulate, void* stream);
long long mdb_conv2d_forward_workspace_bytes_dilated(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                                     int dilation, int flags, int has_residual, int split_weights);
/* w_packed[t][o][i] = w_oihw[o][i][t] * (scale ? scale[o] : 1), rounded to nearest TF32 in precision mode 0
 * (FrozenBatchNorm fold, backbone.py:54-64) */
int mdb_pack_conv_weight_f32(const float* w_oihw, const float* scale, float* w_packed, int O, int I, int taps,
                             void* stream);
int mdb_unpack_conv_wgrad_f32(const float* dw_packed, float* dw_oihw, int O, int I, int taps, int accumulate,
                              void* stream);
/* Multi-tensor forms of the two calls above: n tensors per call (one launch per 64); the array arguments are HOST arrays
 * (scale may be NULL, or hold NULL entries). */
int mdb_pack_conv_weights_multi_f32(int n, const float* const* w_oihw, const float* const* scale, float* const* w_packed,
                                    const int* O, const int* I, const int* taps, void* stream);
int mdb_unpack_conv_wgrads_multi_f32(int n, const float* const* dw_packed, float* const* dw_oihw, const int* O, const int* I,
                                     const int* taps, void* stream);
/* out[n] (+)= sum_m x[m][n]  (bias gradients) */
int mdb_colsum_f32(const float* x, float* out, long long M, int N, int accumulate, void* stream);

/* ---- Fused multi-head attention core, head_dim 32 (attention.cu) -------------------------------------
 * Replaces the core of torch's F.multi_head_attention_forward as called at depthaware_transformer.py:456-459,
 * :496 and depth_predictor/transformer.py:59.  q[b][i][h][32] with token stride ldq floats (batch stride
 * Lq*ldq), k/v likewise (Lk*ldk, Lk*ldv), out[b][i][h*32] with token stride ldo.  key_padding_mask [B][Lk]
 * bytes (nonzero = ignore) or NULL.  lse [B][H][Lq] is written by forward and read by backward.
 * Dropout on the probabilities: drop_p in [0,1); *seed is read on the device (CUDA-graph safe); `site`
 * decorrelates call sites.  delta_ws: B*H*Lq floats of workspace.
 * A query row whose keys are all masked gets out = 0 and lse = -inf, and contributes nothing to the backward: its dq row
 * is 0 and it adds nothing to dk / dv (a batch whose keys are all masked gets dq = dk = dv = 0).  torch's
 * F.multi_head_attention_forward returns NaN for such a row instead.
 */
int mdb_attention_forward_f32(const float* q, const float* k, const float* v, const unsigned char* key_padding_mask,
                              float* out, float* lse, int B, int H, int Lq, int Lk, int head_dim,
                              int ldq, int ldk, int ldv, int ldo, float drop_p,
                              const unsigned long long* seed, unsigned long long site, void* stream);
int mdb_attention_backward_f32(const float* q, const float* k, const float* v, const unsigned char* key_padding_mask,
                               const float* out, const float* lse, const float* dout, float* delta_ws,
                               float* dq, float* dk, float* dv, int B, int H, int Lq, int Lk, int head_dim,
                               int ldq, int ldk, int ldv, int ldo, int lddq, int lddk, int lddv, float drop_p,
                               const unsigned long long* seed, unsigned long long site, void* stream);

/* ---- Normalisation (norm.cu) ---------------------------------------------------------------------------
 * y = LayerNorm(x + dropout(res)) * gamma + beta, rows of C floats (C in {128,256,512}); res may be NULL.
 * Replaces the `src = norm(src + dropout(src2))` pattern of depthaware_transformer.py:341-349,461-462,502-513
 * and depth_predictor/transformer.py:60-65.  mean / rstd: [M] saved for backward.
 * backward: dx = grad wrt x (and wrt res when drop_p == 0); dres (may be NULL iff drop_p == 0) = grad wrt res.
 */
int mdb_add_layernorm_forward_f32(const float* x, const float* res, const float* gamma, const float* beta, float* y,
                                  float* mean, float* rstd, long long M, int C, float eps, float drop_p,
                                  const unsigned long long* seed, unsigned long long site, void* stream);
int mdb_add_layernorm_backward_f32(const float* dy, const float* x, const float* res, const float* gamma,
                                   const float* mean, const float* rstd, float* dx, float* dres, float* dgamma,
                                   float* dbeta, long long M, int C, float drop_p, const unsigned long long* seed,
                                   unsigned long long site, int accumulate, void* stream);
/* GroupNorm(G, C) on NHWC x[B][HW][C] (+ optional fused ReLU) -- monodetr.py:83-91, depth_predictor.py:29-45.
 * stats_ws: B*G*2 doubles; mean / rstd: [B][G]. */
int mdb_groupnorm_forward_f32(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                              double* stats_ws, int B, int HW, int C, int G, float eps, int relu, void* stream);
int mdb_groupnorm_backward_f32(const float* dy, const float* x, const float* y, const float* gamma, const float* mean,
                               const float* rstd, float* dx, float* dgamma, float* dbeta, double* stats_ws,
                               int B, int HW, int C, int G, int relu, void* stream);

/* ---- Elementwise helpers and the frozen ResNet stem (elementwise.cu) ------------------------------------ */
int mdb_relu_backward_f32(const float* dy, const float* y, float* out, long long n, float scale, void* stream);
int mdb_dropout_f32(const float* x, float* out, long long n, float p, const unsigned long long* seed,
                    unsigned long long site, void* stream);
int mdb_round_tf32_f32(const float* x, float* out, long long n, void* stream);
/* backbone.py:100-102 conv1 + bn1 (FrozenBatchNorm2d, backbone.py:54-64) + relu; x NCHW [B][3][H][W] -> y NHWC [B][H/2][W/2][64] */
int mdb_stem_conv7x7_bn_relu_f32(const float* x, const float* w, const float* scale, const float* bias, float* y,
                                 int B, int H, int W, void* stream);
/* torchvision ResNet maxpool(3, 2, 1) on NHWC */
int mdb_maxpool3x3s2_nhwc_f32(const float* x, float* y, int B, int H, int W, int C, void* stream);

/* Depth-map lookup of the head (monodetr.py:248-253): grid_sample(bilinear, zeros, align_corners=True) of
 * depth (B,H,W) at xy (B,N,2) in [-1,1] -> out (B,N); backward wrt the map only (centres are detached). */
int mdb_depth_sample_forward_f32(const float* depth, const float* xy, float* out, int B, int H, int W, int N, void* stream);
int mdb_depth_sample_backward_f32(const float* dout, const float* xy, float* ddepth, int B, int H, int W, int N, void* stream);

/* ---- Fused elementwise chains around the heads and the depth predictor's tail (heads.cu) -----------------------------------
 * box refinement (depthaware_transformer.py:602-613): y[n][6] = sigmoid(tmp + inverse_sigmoid(ref)) on the first ref_dim (2 or 6)
 * components, inverse_sigmoid as utils/misc.py:473-477; backward: dtmp, and dref when non-NULL. */
int mdb_box_refine_forward_f32(const float* tmp, const float* ref, float* y, long long n, int ref_dim, void* stream);
int mdb_box_refine_backward_f32(const float* dy, const float* y, const float* ref, float* dtmp, float* dref /*or NULL*/, long long n,
                                int ref_dim, void* stream);
/* ---- Anchor-box queries (use_dab, dab.cu); every sum runs in a fixed order, no atomics ----------------------------------------
 * sine embedding (depthaware_transformer.py:29-65, 6-d case): box (n,6) -> out (n,768) = [y | x | l | r | t | b], each block 128
 * wide: sin of the even, cos of the odd features of (v * 2pi) / dim_t, dim_t[i] = 10000 ** (2 (i // 2) / 128).  backward: dbox (n,6). */
int mdb_dab_sine_embed_forward_f32(const float* box, float* out, long long n, void* stream);
int mdb_dab_sine_embed_backward_f32(const float* box, const float* dout, float* dbox, long long n, void* stream);
/* query position out (B,rows,C) = scale (B,rows,C) * raw, scale NULL = 1; raw (rows,C) shared by all images when `shared`, else
 * (B,rows,C).  backward: dscale (or NULL) = dqp * raw; draw (or NULL) = dqp * scale, summed over b = 0..B-1 in order when shared. */
int mdb_dab_query_pos_forward_f32(const float* scale, const float* raw, float* out, int B, long long rows, int C, int shared, void* stream);
int mdb_dab_query_pos_backward_f32(const float* dqp, const float* scale, const float* raw, float* dscale, float* draw, int B,
                                   long long rows, int C, int shared, void* stream);
/* gradient of 6-d reference boxes from the sampling locations of the two-step MSDA path: grad_loc / offsets (B,Lq,M,L,P,2) ->
 * dref (B,Lq,6), or (Lq,6) summed over the batch when `shared`.  loc = ref_xy + off / P * (l + r, t + b) / 2. */
int mdb_msda_ref_grad_f32(const float* grad_loc, const float* offsets, int B, int Lq, int M, int L, int P, int shared, float* dref,
                          void* stream);
/* the same from the box partials of mdb_msda_fused_backward_ref_f32: ref_part (B,Lq,M,L,4) -> dref (B,Lq,6), or (Lq,6) summed
 * over the batch when `shared`; 16-byte aligned. */
int mdb_msda_ref_partials_reduce_f32(const float* ref_part, int B, int Lq, int M, int L, int P, int shared, float* dref, void* stream);
/* anchors: r, r2 (n) = sigmoid(w) (one copy per consumer), r_batch (B,n) = r repeated over the batch.  backward: dw = (d_sine + d_msda + sum_b d_head[b]) *
 * r (1 - r); d_sine / d_msda (n) and d_head (B,n) may each be NULL. */
int mdb_dab_anchor_forward_f32(const float* w, float* r, float* r2, float* r_batch, int B, long long n, void* stream);
int mdb_dab_anchor_backward_f32(const float* r, const float* d_sine, const float* d_msda, const float* d_head, int B, long long n,
                                float* dw, void* stream);
/* ---- Learned position embedding (position_embedding: 'learned' / 'v3', pos_embed.cu); no atomics, nothing allocated ----------
 * col, row (50,128) tables.  For a map of H x W: i = x / W * 49 (fp32, each operation rounded), f = floor(i), c = min(f + 1, 49),
 * d = i - f; x_emb[x] = col[f] (1 - d) + col[c] d, y_emb[y] likewise from row over H.  out (H*W,256) channels-last:
 * out[y*W + x] = [x_emb[x] | y_emb[y]] (column embedding first), bit-identical to the separately rounded fp32 operations;
 * col, row and out 16-byte aligned.  backward: dpos (H*W,256) (summed over the batch) -> dcol, drow (50,128); every row is written
 * (zero where no coordinate reaches it), summed per row over the coordinates in ascending order, each the ascending sum over the
 * other axis times (1 - d) or d. */
int mdb_pos_learned_forward_f32(const float* col, const float* row, int H, int W, float* out, void* stream);
int mdb_pos_learned_backward_f32(const float* dpos, int H, int W, float* dcol, float* drow, void* stream);
/* depth of a query (monodetr.py:230-262): out[b][q] = ((1/(sigmoid(reg0)+1e-6) - 1) + size3d0 / clamp((c4+c5)*img_h, 1) * fu +
 * grid_sample(weighted_depth, (c01 - 0.5)*2, bilinear, zeros, align_corners=True)) / 3 , reg1.  coord (B,N,6), size3d (B,N,3),
 * depth_reg (B,N,2), wdepth (B,H,W), calibs (B,3,4), img_sizes (B,2) = [W, H].  backward: dwdepth is zero-filled by the call. */
int mdb_head_depth_forward_f32(const float* coord, const float* size3d, const float* depth_reg, const float* wdepth, const float* calibs,
                               const float* img_sizes, float* out, int B, int N, int H, int W, void* stream);
int mdb_head_depth_backward_f32(const float* dout, const float* coord, const float* size3d, const float* depth_reg, const float* calibs,
                                const float* img_sizes, float* dcoord, float* dsize3d, float* dreg, float* dwdepth, int B, int N, int H,
                                int W, void* stream);
/* depth predictor tail (depth_predictor.py:74-104): per pixel softmax over nb (<= 96) bin logits, weighted depth = sum p * bins,
 * ip = lerp of the embedding rows floor / floor+1 of clamp(depth, 0, dmax).  logits (npix, nb), emb (E, C), C % 4 == 0, C <= 256.
 * backward: d_wd_ext (npix) = gradient reaching weighted_depth from elsewhere, or NULL; demb is zero-filled by the call. */
int mdb_depth_tail_forward_f32(const float* logits, const float* bins, const float* emb, float* wdepth, float* ip, long long npix, int nb,
                               int E, int C, float dmax, void* stream);
int mdb_depth_tail_backward_f32(const float* logits, const float* bins, const float* emb, const float* d_ip, const float* d_wd_ext,
                                float* dlogits, float* demb, long long npix, int nb, int E, int C, float dmax, void* stream);
/* F.interpolate(mode="bilinear", align_corners=False) to a given size on NHWC maps: x (B,Hi,Wi,C) -> y (B,Ho,Wo,C), C % 4 == 0.
 * src = (in / out) * (dst + 0.5) - 0.5 clamped at 0, i1 = i0 + (i0 < in - 1) (torch's rule).  backward: dx (B,Hi,Wi,C) fully
 * written in gather form (no atomics, bit-reproducible). */
int mdb_upsample_bilinear_nhwc_forward_f32(const float* x, float* y, int B, int Hi, int Wi, int Ho, int Wo, int C, void* stream);
int mdb_upsample_bilinear_nhwc_backward_f32(const float* dy, float* dx, int B, int Hi, int Wi, int Ho, int Wo, int C, void* stream);
/* (a + b + c) / 3 and a * s; n % 4 == 0 */
int mdb_mean3_f32(const float* a, const float* b, const float* c, float* out, long long n, void* stream);
int mdb_scale_f32(const float* a, float* out, long long n, float s, void* stream);
/* loss = sum_k mean(x_k^2) over `count` (<= 32) tensors (the surrogate loss of bench.py's step) and its gradient
 * g_k = 2 x_k / n_k * dloss; x / g / n are HOST arrays, loss / dloss device scalars. */
int mdb_sum_mean_squares_forward_f32(int count, const float* const* x, const long long* n, float* loss, void* stream);
int mdb_sum_mean_squares_backward_f32(int count, const float* const* x, float* const* g, const long long* n, const float* dloss,
                                      void* stream);

/* ---- Fused AdamW over flat buffers (optim.cu) -- lib/helpers/optimizer_helper.py:69-129 (the reference's AdamW.step) ----
 * p, g, m, v: n floats each, 16-byte aligned; elements [0, n_decay) get `weight_decay`, the rest 0 (the reference's
 * 'bias' in name -> no decay rule, optimizer_helper.py:9-16, realised by the flat ordering).  step_size =
 * lr * sqrt(1 - beta2^t) / (1 - beta1^t) is computed by the caller: as a host float, or -- step_size_dev != NULL -- read from
 * device memory at run time (a captured CUDA graph then sees the new value every replay).  one_minus_beta* are passed
 * separately so that they are the fp32 roundings of the DOUBLE expressions 1 - beta*, as in the reference. */
int mdb_adamw_step_f32(float* p, const float* g, float* m, float* v, long long n, long long n_decay, float beta1,
                       float one_minus_beta1, float beta2, float one_minus_beta2, float eps, float weight_decay,
                       float step_size, const float* step_size_dev, void* stream);

/* Device-resident schedule of one optimizer: what a captured CUDA graph reads every replay instead of host floats.  The caller
 * owns the block (40 bytes, 8-byte aligned, device memory), initialises t (the number of steps taken so far, an integer value)
 * and the three hyper-parameters as the DOUBLES the host holds, and may overwrite lr between steps with an asynchronous copy
 * ordered on the training stream (a learning-rate schedule then reaches a graph that was captured earlier). */
typedef struct MdbAdamwHyper {
    double t;         /* steps taken; mdb_adamw_advance adds 1 */
    double lr;
    double beta1;
    double beta2;
    float step_size;  /* written by mdb_adamw_advance; pass its address as mdb_adamw_step_f32's step_size_dev */
    float reserved_;
} MdbAdamwHyper;
/* One single-thread launch: t += 1; step_size = (float)(lr * sqrt(1 - beta2^t) / (1 - beta1^t)), every operation in fp64 in
 * that order and one rounding to fp32 -- the value optimizer_helper.py:122-124 computes on the host. */
int mdb_adamw_advance(MdbAdamwHyper* hyper, void* stream);

/* ---- Inference post-process on the device (decode.cu) -- SURVEY.md 8 f3 ----
 * extract: lib/helpers/decode_helper.py:57-110 (extract_dets_from_outputs).  logits (B,Q,C), boxes (B,Q,6) cx cy l r t b,
 * dim3 (B,Q,3), depth (B,Q,2) [depth, log-variance], angle (B,Q,24).  dets (B,topk,37) = label, score, xs2d, ys2d, w, h, depth,
 * heading[24], size3d[3], xs3d, ys3d, sigma; rows ordered by descending score, ties by ascending (query, class).
 * Q*C <= 4096 (else MDB_EUNSUPPORTED), topk <= Q*C.
 * decode: lib/helpers/decode_helper.py:8-54 (decode_detections) with the camera arithmetic of
 * lib/datasets/kitti/kitti_utils.py:150-155,207-208,277-282.  img_size (B,2) [W,H], P2 (B,3,4), cls_mean_size (C,3).
 * out (B,topk,14) = cls, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score*sigma for the count[b] leading rows whose score
 * reaches `threshold` (the rest zero-filled); count (B) int32.  Both run on `stream` without synchronising. */
int mdb_extract_dets_f32(const float* logits, const float* boxes, const float* dim3, const float* depth, const float* angle, int B,
                         int Q, int C, int topk, float* dets, void* stream);
int mdb_decode_dets_f32(const float* dets, const float* img_size, const float* P2, const float* cls_mean_size, int B, int topk, int C,
                        float threshold, float* out, int* count, void* stream);

/* ---- Training criterion on the device (criterion.cu) -- SURVEY.md 8 f1 ----
 * lib/models/monodetr/matcher.py:36-104 (HungarianMatcher.forward), monodetr.py:297-532 (SetCriterion), depth_predictor/ddn_loss/
 * {ddn_loss.py:43-127, balancer.py:21-81, focalloss.py:52-125}, lib/helpers/trainer_helper.py:175-186 (prepare_targets).
 * Targets are the data loader's PADDED arrays (B, Gmax, ...) plus the validity mask (B, Gmax) -- no compaction on the host:
 *   labels int32, boxes2d (cx cy w h), boxes3d (cx cy l r t b), depth, size3d (3), heading_bin int32, heading_res.
 * Predictions are passed per decoder layer (layer 0 = the final outputs, then the aux outputs), L <= MDB_CRITERION_MAX_LAYERS:
 *   logits (B,Q,C), boxes (B,Q,6), dim3 (B,Q,3), depth (B,Q,2), angle (B,Q,24), all contiguous fp32.
 * Call order: prepare -> [all-reduce `total` across ranks] -> match -> depth_map -> losses; backward: depth_map (gradient mode) and
 * losses_backward.  Nothing synchronises with the host.  Q / group <= 64, Gmax <= 64, B <= 1024 (else MDB_EUNSUPPORTED). */
#define MDB_CRITERION_MAX_LAYERS 4
#define MDB_CRITERION_NUM_LOSSES 10
#define MDB_LOSS_CE 0           /* loss slots of one layer in `losses` / `grad_losses` (L, MDB_CRITERION_NUM_LOSSES) */
#define MDB_LOSS_CLASS_ERROR 1  /* (logging only, no gradient) */
#define MDB_LOSS_BBOX 2
#define MDB_LOSS_GIOU 3
#define MDB_LOSS_CARDINALITY 4  /* (logging only, no gradient) */
#define MDB_LOSS_DEPTH 5
#define MDB_LOSS_DIM 6
#define MDB_LOSS_ANGLE 7
#define MDB_LOSS_CENTER 8
#define MDB_LOSS_DEPTH_MAP 9    /* layer 0 only */
/* tlist (B,Gmax): indices of the valid targets of each image in their original order, -1 padded; count (B); total (1) = sum */
int mdb_criterion_prepare(const unsigned char* mask, int B, int Gmax, int* tlist, int* count, float* total, void* stream);
/* match (L,B,group,Gmax): query index in [0,Q) assigned to the j-th valid target of the image by the group's assignment problem
 * (cost = w_bbox*L1(box) + w_center*L1(centre) + w_class*focal cost + w_giou*(-GIoU)), -1 where none; tclass (L,B,Q): class of
 * the target a query is matched to, C for "no object". */
int mdb_criterion_match_f32(int L, const float* const* logits, const float* const* boxes, const int* labels, const float* boxes3d,
                            const int* tlist, const int* count, int B, int Q, int C, int group, int Gmax, float w_class, float w_center,
                            float w_bbox, float w_giou, int* match, int* tclass, void* stream);
/* Depth-map loss per pixel.  logits are addressed as logits[b*stride_b + pixel*stride_pix + c*stride_c], c in [0, num_bins]
 * (NHWC: stride_pix = num_bins+1, stride_c = 1; NCHW: stride_pix = 1, stride_c = H*W).  boxes2d are scaled by (scale_x, scale_y)
 * (the reference hard-codes 80, 24).  dlogits == NULL: writes pix_loss (B*H*W), already weighted fg/bg; otherwise writes
 * dlogits (same addressing) = grad_loss[0] * d(mean-balanced loss)/d logits. */
int mdb_criterion_depth_map_f32(const float* logits, long long stride_b, long long stride_pix, long long stride_c, const float* boxes2d,
                                const float* depth, const int* tlist, const int* count, int B, int H, int W, int num_bins, int Gmax,
                                float scale_x, float scale_y, float depth_min, float depth_max, float alpha, float fg_weight,
                                float bg_weight, float* pix_loss, const float* grad_loss, float* dlogits, void* stream);
/* losses (L, MDB_CRITERION_NUM_LOSSES), un-weighted, normalised by num_boxes = max(total * group / world_size, 1) as the reference.
 * pix_loss / npix: output of the depth-map kernel (NULL / 0: slot stays 0).  aux (L): per-layer scalar kept for backward (the
 * gradient-free compensation weight of the dimension loss, monodetr.py:414-416).  Deterministic (fixed-order reductions). */
int mdb_criterion_losses_f32(int L, const float* const* logits, const float* const* boxes, const float* const* dim3,
                             const float* const* depth, const float* const* angle, const int* labels, const float* boxes3d,
                             const float* tdepth, const float* size3d, const int* hbin, const float* hres, const int* tlist,
                             const int* count, const float* total, const int* match, const int* tclass, const float* pix_loss, int npix,
                             int B, int Q, int C, int group, int Gmax, float focal_alpha, float world_size, float* losses, float* aux,
                             void* stream);
/* d(sum_k grad_losses[l][k] * losses[l][k]) / d predictions; every d* buffer is fully written (zeros for unmatched queries). */
int mdb_criterion_losses_backward_f32(int L, const float* const* logits, const float* const* boxes, const float* const* dim3,
                                      const float* const* depth, const float* const* angle, const int* labels, const float* boxes3d,
                                      const float* tdepth, const float* size3d, const int* hbin, const float* hres, const int* tlist,
                                      const int* count, const float* total, const int* match, const int* tclass, int B, int Q, int C,
                                      int group, int Gmax, float focal_alpha, float world_size, const float* grad_losses,
                                      const float* aux, float* const* dlogits, float* const* dboxes, float* const* ddim3, float* const* ddepth,
                                      float* const* dangle, void* stream);

/* ---- Loss log of the training loop (trainlog.cu) -- lib/helpers/trainer_helper.py:145-152 without the 26 `.item()` calls ----
 * Appends one record to a device ring: record k = *counter % slots receives values[i] * weights[i] (one fp32 multiply each, the
 * bits of `(loss * weight).item()`) for i < n, then their sum in index order at position n; afterwards *counter += 1.  The slot
 * index comes from device memory, so a captured launch is the same every replay; the host, which counts its own pushes, knows
 * which record a step went to and copies it out when it wants to print.  ring: slots * (n + 1) floats; counter: one int64 the
 * caller zeroes; 1 <= n <= 255, slots >= 1. */
int mdb_trainlog_push_f32(const float* values, const float* weights, int n, float* ring, int slots, long long* counter, void* stream);

/* ---- Input pipeline on the device (preprocess.cu) -- SURVEY.md 8 f4 ----
 * lib/datasets/kitti/kitti_dataset.py:140-161: [flip] -> PIL Image.transform(AFFINE, BILINEAR) -> float32 / 255 -> (x - mean) / std -> CHW.
 * src: DEVICE array of B device pointers to 8-bit RGB images (3 bytes per pixel), src_wh (B,2) [W,H] int32 and src_pitch (B) bytes
 * per row (device); trans_inv (B,6) fp64 device = PIL's `data` (output pixel centre -> input coordinates, the reference's
 * trans_inv); flip (B) bytes or NULL: sample the left-right mirrored image.  mean3 / std3: HOST floats.
 * out (B,3,out_h,out_w) fp32.  The 8-bit interpolation result and the float conversion are bit-identical to PIL + numpy. */
int mdb_warp_affine_normalize_u8(const unsigned char* const* src, const int* src_wh, const long long* src_pitch, const double* trans_inv,
                                 const unsigned char* flip, int B, int out_w, int out_h, const float* mean3, const float* std3, float* out,
                                 void* stream);

/* Photometric distortion, the dataset's `aug_pd` step before the warp: kitti_dataset.py:136-138
 * `pd(np.array(img).astype(np.float32)).astype(np.uint8)` with lib/datasets/kitti/pd.py:376-397.  One record per image holds the
 * reference's random draws (drawn on the host; a step whose coin said no carries its neutral value, which gives the same bits as
 * skipping it).  Record layout, 24 bytes, 4-byte aligned: */
typedef struct mdb_photometric_params {
    float brightness;   /* RandomBrightness delta, added to every channel first (0 = off) */
    float contrast;     /* RandomContrast alpha, multiplies every channel (1 = off) */
    float saturation;   /* RandomSaturation factor on S (1 = off) */
    float hue;          /* RandomHue delta in degrees added to H, then > 360 -> -360, < 0 -> +360 (0 = off) */
    int contrast_last;  /* 0: contrast, HSV, saturation, hue, BGR (pd[:-1]); 1: HSV, saturation, hue, BGR, contrast (pd[1:]) */
    int perm;           /* RandomLightingNoise: out channel k = channel perms[perm][k] of pd.py:143-145, 0..5 (0 = identity = off) */
} mdb_photometric_params;
/* Per pixel in fp32, every scalar rounded to fp32 first: + brightness, then the colour steps in the record's order, then the
 * channel permutation.  The RGB image is read as BGR (channel 0 is "B"), as the reference does.  The two cv2.cvtColor conversions
 * are restated as cv2 4.13 computes them on float32 with AVX2 + FMA3: the hue of the last W % 8 pixels of each row comes from
 * cv2's scalar loop, the others from its 8-wide vector loop, and the two round differently.  Those bits follow the reference's CPU
 * dispatch; other cv2 builds or dispatch levels are not verified.  The final cast copies the REFERENCE'S QUIRK: numpy's float32 ->
 * uint8 cast on x86 truncates toward zero and keeps the low 8 bits (290.3 -> 34, -5.7 -> 251), and values outside [0, 256) are
 * common after a saturation or contrast factor above 1.
 * src / src_wh / src_pitch: as mdb_warp_affine_normalize_u8 (all DEVICE arrays); params (B) DEVICE records; dst: DEVICE array of B
 * device pointers to the 8-bit RGB outputs (W_b x H_b x 3, may not overlap the sources), dst_pitch (B) bytes per row (device).
 * One launch; the library allocates nothing.  MDB_EINVAL for a null array or B outside 1..65535.  The records and sizes are read
 * on the device, so the caller checks them: an image whose record has perm outside 0..5 or contrast_last outside 0..1, or whose
 * size is not positive, is left unwritten (monodetr_b200.preprocess raises ValueError before launching). */
int mdb_photometric_distort_u8(const unsigned char* const* src, const int* src_wh, const long long* src_pitch,
                               const mdb_photometric_params* params, unsigned char* const* dst, const long long* dst_pitch, int B,
                               void* stream);

/* ---- KITTI training targets on the device (labels.cu) ----
 * The label half of the dataset's __getitem__ (lib/datasets/kitti/kitti_dataset.py:173-330): every label line of a split is parsed
 * once on the host into a LABEL BANK kept on the device, in CSR form: obj_off (n_bank+1) int64 prefix sums of the per-image line
 * counts, objects (obj_off[n_bank], MDB_LABEL_RECORD_WIDTH) fp64 records, P2 (n_bank, 3, 4) fp32.  Every line is kept, in file
 * order (DontCare and unknown classes included): target slot i is line i, as in the reference.  Record columns: */
#define MDB_LABEL_RECORD_WIDTH 16
#define MDB_LABEL_CLS 0      /* class code: 0 Pedestrian, 1 Car, 2 Cyclist, -1 any other type */
#define MDB_LABEL_TRUNC 1    /* truncation, occlusion, alpha: fp64 as parsed */
#define MDB_LABEL_OCC 2
#define MDB_LABEL_ALPHA 3
#define MDB_LABEL_BOX2D 4    /* x1 y1 x2 y2: float32 values (the reference parses box2d as float32) */
#define MDB_LABEL_HWL 8      /* h w l: fp64 */
#define MDB_LABEL_POS 11     /* x y z: float32 values */
#define MDB_LABEL_RY 14      /* fp64; column 15 is unused */
#define MDB_LABEL_MAX_OBJS 1024
/* One record per image of the batch, 72 bytes, 8-byte aligned: the draws of kitti_dataset.py:130-154. */
typedef struct mdb_label_image {
    double trans[6];    /* 2x3 affine map source image -> network input (get_affine_transform(..., inv=1)[0]), row-major */
    double crop_scale;  /* 1 when no crop was drawn */
    int bank_index;     /* image in the bank, 0..n_bank-1 */
    int img_w, img_h;   /* source image size (the flip mirrors about img_w) */
    int flip;           /* 0 / 1 */
} mdb_label_image;
/* Dataset options (HOST struct, read at launch). */
#define MDB_DEPTH_NORMAL 0   /* depth = z * crop_scale */
#define MDB_DEPTH_INVERSE 1  /* depth = z / crop_scale */
#define MDB_DEPTH_NONE 2     /* depth = z */
typedef struct mdb_label_config {
    double mean_size[9];  /* (3 classes, h w l) subtracted from the size; zeros unless `meanshape` */
    int class_mask;       /* bit c set: class code c is in the writelist */
    int clip_2d;          /* clip negative l / r / t / b to [0, 1] instead of dropping the object */
    int depth_scale;      /* MDB_DEPTH_* */
    int res_w, res_h;     /* network input `resolution` (W, H) */
    int max_objs;         /* target slots per image, 1..MDB_LABEL_MAX_OBJS (the reference: 50) */
} mdb_label_config;
/* Padded targets of B images, one thread per (image, slot), every slot written (zeros where the reference leaves zeros), in the
 * reference's collated dtypes: calibs (B,S,3,4) f32, indices (B,S) int64 (zeros), labels (B,S) int8, boxes (B,S,4), boxes_3d
 * (B,S,6), depth (B,S,1), size_2d (B,S,2), size_3d (B,S,3), src_size_3d (B,S,3) f32, heading_bin (B,S,1) int64, heading_res (B,S,1)
 * f32, mask_2d (B,S) bytes 0 / 1; S = max_objs.  Filters and encoding follow the reference step by step: writelist; level
 * 'UnKnown' (from the float32 box); z < 2 or > 65; flip of box2d and ry; affine map of the box corners and of the projected 3-d
 * centre (which must land inside the resolution); l / r / t / b sign test or clip; depth scaling; ry2alpha + angle2class on the
 * flipped ORIGINAL box; size encoding; mask rule.  Each step runs at the precision numpy 2 gives it there (fp64 with explicit _rn
 * operations, or float32 _rn), rounded to float32 where the reference stores it; arctan2 is atan2 in fp64 rounded to float32
 * (numpy's float32 arctan2 is not correctly rounded, so heading_res can differ from the reference's by a few float32 ulp).
 * obj_off / objects / P2 / images and the outputs are DEVICE arrays; cfg is a HOST pointer.  One launch; the library allocates
 * nothing.  MDB_EINVAL for a null pointer, B outside 1..65535, n_bank < 1, max_objs outside 1..MDB_LABEL_MAX_OBJS, a non-positive
 * resolution or an unknown depth_scale.  The image records are read on the device: an image whose bank_index is outside
 * 0..n_bank-1 gets all-zero targets (monodetr_b200.labels raises ValueError before launching). */
int mdb_kitti_encode_targets(const long long* obj_off, const double* objects, const float* P2, int n_bank,
                             const mdb_label_image* images, int B, const mdb_label_config* cfg, float* calibs, long long* indices,
                             signed char* labels, float* boxes, float* boxes_3d, float* depth, float* size_2d, float* size_3d,
                             float* src_size_3d, long long* heading_bin, float* heading_res, unsigned char* mask_2d, void* stream);

/* ---- KITTI evaluation on the device (kitti_eval.cu) ----
 * lib/datasets/kitti/kitti_eval_python/eval.py:9-412,614-644 (get_thresholds, clean_data, image_box_overlap, d3_box_overlap,
 * compute_statistics_jit, fused_compute_statistics) and rotate_iou.py:17-330 (the rotated-box IoU).  The annotations of n_img images
 * are packed in CSR form: gt_off / dt_off (n_img+1) int32 prefix sums of the per-image box counts, ov_off (n_img+1) int64 prefix
 * sums of n_dt_b * n_gt_b (the per-image overlap blocks; n_ov = ov_off[n_img]).  max_gt / max_dt are the largest per-image counts
 * (HOST values; above MDB_KITTI_MAX_BOXES -> MDB_EUNSUPPORTED).
 *   gt_f (n_gt, MDB_KITTI_GT_COLS) fp64: bbox x0 y0 x1 y1, alpha, truncated, location x y z, dimensions l h w, rotation_y
 *   gt_i (n_gt, 3) int32: occluded, class code, DontCare flag (name == "DontCare", case-sensitive)
 *   dt_f (n_dt, MDB_KITTI_DT_COLS) fp64: bbox x0 y0 x1 y1, alpha, score, location x y z, dimensions l h w, rotation_y
 *   dt_cls (n_dt) int32: class code
 * A class code is the index of the lower-cased name in {car, pedestrian, cyclist, van, person_sitting, truck}, -1 for any other.
 * overlaps (3, n_ov) fp64: metric 0 = 2-d IoU (fp64), 1 = bird's-eye-view IoU of [x, z, l, w, ry] (fp32 polygon clipping,
 * widened), 2 = 3-d IoU (the fp32 BEV intersection times the fp64 height overlap, rounded to fp32); the block of image b starts at
 * ov_off[b], detection-major (n_dt_b, n_gt_b).  No FMA contraction anywhere: 2-d overlaps are bit-identical to the reference. */
#define MDB_KITTI_MAX_BOXES 1024       /* gt boxes, and detections, per image */
#define MDB_KITTI_MAX_CLASSES 6
#define MDB_KITTI_MAX_TOTAL_GT (1 << 22)
#define MDB_KITTI_NUM_THRESH 41        /* score thresholds (sample points) per configuration */
#define MDB_KITTI_GT_COLS 13
#define MDB_KITTI_DT_COLS 13
int mdb_kitti_overlaps(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int max_gt, int max_dt,
                       long long n_ov, const double* gt_f, const double* dt_f, double* overlaps, void* stream);
/* Bytes of scratch mdb_kitti_eval needs (negative = MDB_E*): about n_cfg * 8 * next_pow2(n_gt) for the score sort, plus
 * n_cfg * 41 * n_img * 8 when compute_aos, plus per-box flags; n_cfg = 18 * n_cls. */
long long mdb_kitti_eval_workspace_bytes(int n_img, int n_gt, int n_dt, int n_cls, int compute_aos);
/* Every configuration cfg = ((metric * n_cls + m) * 3 + difficulty) * 2 + k of the classes `classes` (n_cls int32, codes as above)
 * in one call: clean_data, the TP scores (compute_fp=False), the score thresholds, then tp / fp / fn / AOS similarity at each
 * threshold (compute_fp=True).  min_overlaps (2, 3, n_cls) fp64 = the reference's min_overlaps[:, :, current_classes].
 * result (n_cfg, 1 + 4 * MDB_KITTI_NUM_THRESH) fp64: [number of thresholds T, then (tp, fp, fn, similarity) per threshold]; rows
 * t >= T are zero.  T > MDB_KITTI_NUM_THRESH is reported as is (the reference fails on such input).  similarity is summed per
 * image in gt order and over images in image order, only for metric 0 with compute_aos.  n_img >= 1.  Five kernel launches, no float atomics:
 * the result is the same in both reproducible modes.  workspace: at least mdb_kitti_eval_workspace_bytes (else MDB_EWORKSPACE). */
int mdb_kitti_eval(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int n_gt, int n_dt, int max_gt,
                   int max_dt, long long n_ov, const double* gt_f, const int* gt_i, const double* dt_f, const int* dt_cls,
                   const double* overlaps, const int* classes, const double* min_overlaps, int n_cls, int compute_aos,
                   void* workspace, long long workspace_bytes, double* result, void* stream);
/* The distance-binned evaluation (eval.py:85-159 clean_data_by_distance, DISTANCE_COVER = False, as do_eval(..., DIForDIS=False)
 * runs it): mdb_kitti_eval with the third configuration index a distance bin instead of a difficulty, cfg = ((metric * n_cls + m)
 * * 3 + bin) * 2 + k.  Bin 0 keeps the gt with ||location|| <= 30 m, bin 1 those in (30, 50] m, bin 2 those in (50, 70] m
 * (fp64 x*x + y*y + z*z in that order, correctly rounded square root); the others are ignored.  Every bin applies the hard level's
 * occlusion / truncation / height limits to gt and its height limit (25) to detections.  Same arguments, workspace and launches. */
int mdb_kitti_eval_distance(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int n_gt, int n_dt,
                            int max_gt, int max_dt, long long n_ov, const double* gt_f, const int* gt_i, const double* dt_f,
                            const int* dt_cls, const double* overlaps, const int* classes, const double* min_overlaps, int n_cls,
                            int compute_aos, void* workspace, long long workspace_bytes, double* result, void* stream);

/* Detections of a validation pass kept on the device instead of result files (tester_helper.py:112-132 writes them,
 * kitti_common.py:294-347 reads them back).  mdb_kitti_collect_dets_f32 takes mdb_decode_dets_f32's rows (B, topk, 14) and
 * count (B) and writes the count[b] leading rows of image b to position slot[b] of the split:
 *   table_f (n_img, topk, MDB_KITTI_DT_COLS) fp64 in dt_f's column order, each value rint((double)x * 100) / 100 -- exactly
 *           float('{:.2f}'.format(x)) of the float32 x, sign of zero included;
 *   table_cls (n_img, topk) int32: cls_code[int(row class)] (the tester's class name as an eval class code), -1 outside 0..n_code-1;
 *   slot_info (3, n_img) int32: [0] the count, [1] += 1 per write of the slot (the caller zeroes it per pass and rejects values
 *           other than 1), [2] 1 when the slot has detections and the first one's printed alpha is not -10 (eval.py:745-751).
 * slot (B) and cls_code (n_code) are HOST arrays, passed to the kernel by value; a slot outside 0..n_img-1 -> MDB_EINVAL before
 * any launch.  topk <= MDB_KITTI_MAX_BOXES, n_code <= MDB_KITTI_COLLECT_MAX_CLASSES (else MDB_EUNSUPPORTED).  One launch per
 * MDB_KITTI_COLLECT_MAX_BATCH images; no synchronisation, no allocation. */
#define MDB_KITTI_COLLECT_MAX_BATCH 512
#define MDB_KITTI_COLLECT_MAX_CLASSES 8
int mdb_kitti_collect_dets_f32(const float* rows, const int* count, const int* slot, int B, int topk, int n_img,
                               const int* cls_code, int n_code, double* table_f, int* table_cls, int* slot_info, void* stream);
/* The padded table -> CSR dt_f (n_dt, 13) / dt_cls (n_dt) of mdb_kitti_eval; dt_off (n_img + 1) device int32 prefix sums of the
 * per-slot counts (slot_info[0]).  One launch. */
int mdb_kitti_compact_dets(const int* dt_off, const double* table_f, const int* table_cls, int n_img, int topk, double* dt_f,
                           int* dt_cls, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MONODETR_B200_H_ */
