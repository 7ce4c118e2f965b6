/* tfimm_b200 -- C ABI of the H100 (sm_90a) kernel library behind the tfimm forward path.
 *
 * The reference (martinsbruveris/tensorflow-image-models) has no FFI of its own: its device
 * boundary is inside TensorFlow.  This header is the boundary a maintainer would bind instead
 * (ctypes stub in INTEGRATION.md; the in-tree binding is
 * tensorflow-image-models_b200/tfimm/backend/lib.py).  Every entry point names the reference
 * call site(s) it replaces.
 *
 * Conventions
 *   - plain C, no torch / C++ types; every pointer is a DEVICE pointer owned by the caller
 *   - activations are channels-last: (rows, C) / (B, H, W, C); Dense/conv weights are passed
 *     pre-transposed as W[N][K] (K contiguous), i.e. the TF kernel (in,out) / (kh,kw,in,out)
 *     flattened over its leading axes and transposed once at load time
 *   - dtype codes: TFIMM_F32 / TFIMM_BF16 / TFIMM_U8; bias / gamma / beta / BN vectors are fp32
 *   - every launch takes the cudaStream_t to enqueue on (as void*); calls are asynchronous
 *   - return value: 0 = OK, otherwise a TFIMM_ERR_* code; tfimm_b200_last_error() returns a
 *     thread-local human-readable message.  Nothing here allocates device memory.
 *   - there is NO CPU fallback: without an H100 these calls fail with a CUDA error.
 */
#ifndef TFIMM_B200_H_
#define TFIMM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFIMM_F32 0
#define TFIMM_BF16 1
#define TFIMM_U8 2

#define TFIMM_ACT_NONE 0
#define TFIMM_ACT_GELU 1    /* exact erf form == Keras "gelu" (tfimm/layers/factory.py:8-9) */
#define TFIMM_ACT_SWISH 2   /* x * sigmoid(x) */
#define TFIMM_ACT_RELU 3
#define TFIMM_ACT_RELU6 4   /* tf.keras.layers.ReLU(max_value=6) (tfimm/layers/factory.py:10-11) */
#define TFIMM_ACT_TANH 5
#define TFIMM_ACT_SIGMOID 6

#define TFIMM_OK 0
#define TFIMM_ERR_INVALID_ARGUMENT 1
#define TFIMM_ERR_CUDA 2
#define TFIMM_ERR_UNSUPPORTED 3

/* Library identification / diagnostics. */
const char* tfimm_b200_version(void);
const char* tfimm_b200_last_error(void);
/* Number of SMs of the current device (0 if no device); used by the host to size workspaces. */
int tfimm_b200_sm_count(void);

/* Dense / 1x1 conv with fused epilogue:  C = residual + gamma * act(A @ W^T + bias), or with
 * act_after_residual != 0:  C = act(residual + gamma * (A @ W^T + bias))  (ResNet blocks, resnet.py:186-188).
 * A:[M,K] bf16 (ld = lda), W:[N,K] bf16 (ld = ldw), C/residual:[M,N] of out_dtype (bf16|f32);
 * residual may alias C (in-place residual stream).  wgmma tensor cores, TMA, fp32 accumulate.
 * Replaces tf.keras.layers.Dense at tfimm/architectures/vit.py:142-146, swin.py:124-128,343-345,
 * tfimm/layers/transformers.py:192-205, the classifier heads (vit.py:364-368, swin.py:457-461,
 * convnext.py:356-360, efficientnet.py:259-263) and 1x1 Conv2D (efficientnet_blocks.py:412-434,
 * resnet.py:220-248); gamma/residual fuse ConvNeXtBlock's layer-scale + shortcut (convnext.py:226-227).
 * force_block_n: 0 = auto; 64/128/256 = that tile width (testing / A-B measurements); 2 = the widest tile,
 * the same as 256; 1 = the persistent kernel (128 x 256 tiles, one CTA per SM; bf16 output with N % 8 != 0 runs the
 * 256-wide tile instead). */
int tfimm_b200_gemm_bf16(const void* A, int lda, const void* W, int ldw, const float* bias,
                         const float* gamma, const void* residual, int ldr, void* C, int ldc, int M, int N,
                         int K, int act, int act_after_residual, int out_dtype, int force_block_n, void* stream);

/* Dense / 1x1 conv whose INPUT rows carry a squeeze-excite gate:  C = residual + act((A * gate[row / rows_per_image]) @ W^T
 * + bias), bf16 in / out.  gate: fp32 [n_images][K] (the sigmoid of tfimm_b200_se_gate).  The gate is applied to the A
 * tile in shared memory between the TMA load and the tensor-core product, with the rounding of the separate pass
 * (bf16(x * g), tfimm_b200_scale_channels) -- which, as its own kernel, read and wrote the whole expanded activation
 * (3.4 ms of a 24 ms EfficientNet-B4 step at batch 256).  Replaces `x * gate` of SEModule.call
 * (tfimm/layers/attention.py, used at efficientnet_blocks.py:241-248, 438-453) + the projection Conv2D that follows. */
int tfimm_b200_gemm_bf16_gated(const void* A, int lda, const float* gate, int rows_per_image, int n_images,
                               const void* W, int ldw, const float* bias, const void* residual, int ldr, void* C,
                               int ldc, int M, int N, int K, int act, void* stream);

/* Fused MLP block of the narrow stages:  out = residual + gamma * (act(A @ W1^T + b1) @ W2^T + b2).
 * A:[M,C] bf16 (the normalised activations), W1:[hidden,C] bf16, W2:[C,hidden] bf16, b1:[hidden], b2:[C], gamma:[C] or
 * NULL (ConvNeXt layer scale), residual / out:[M,C] fp32 (residual may alias out, or be NULL).  C in {96, 128, 192, 256},
 * hidden a multiple of 128: other shapes return TFIMM_ERR_UNSUPPORTED and the caller runs two tfimm_b200_gemm_bf16.
 * One CTA per 128 rows walks the hidden dimension in chunks of 64: fc1 chunk (wgmma) -> bias + activation -> bf16
 * register fragments -> A operand of the fc2 chunk product (wgmma with A from registers); the [M,hidden]
 * activations never reach HBM (the hidden tensor is 61 % of the bytes the two-GEMM form moves at C = 128).  The
 * rounding points are those of the two-GEMM form (bf16 hidden, fp32 accumulation in ascending k).
 * Replaces MLP.call (tfimm/layers/transformers.py:208-214) + layer scale + shortcut in ConvNeXtBlock.call
 * (tfimm/architectures/convnext.py:219-228) and the MLP half of SwinTransformerBlock.call (swin.py:315-318). */
int tfimm_b200_mlp_bf16(const void* A, int lda, const void* W1, int ldw1, const float* b1, const void* W2, int ldw2,
                        const float* b2, const float* gamma, const void* residual, int ldr, void* out, int ldc, int M,
                        int C, int hidden, int act, void* stream);

/* Dense k x k convolution (+ folded-BN bias, activation, optional residual, act(x + shortcut)) as an IMPLICIT GEMM
 * on the wgmma tensor cores: tf.keras.layers.ZeroPadding2D(pad) + Conv2D(k, strides) (+ BatchNormalization, act)
 * at tfimm/architectures/resnet.py:129-150 (BasicBlock 3x3), 230-238 (Bottleneck conv2), 486-512 (deep stems).
 * x: NHWC bf16 [B][H][W][C], C % 64 == 0; W: bf16 [N][k*k*C] in (ky, kx, c) order (the TF kernel (kh,kw,cin,cout)
 * flattened and transposed), leading dimension ldw; out / residual: NHWC [B][Ho][Wo][N], bf16 or fp32.
 * No im2col matrix is materialised: each A tile (128 output pixels x 64 channels of one tap) is one 4-D TMA box
 * of the input whose out-of-bounds elements are the zero padding; stride 2 is the box's traversal stride. */
int tfimm_b200_conv_bf16(const void* x, const void* W, int ldw, const float* bias, const void* residual, void* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act,
                         int act_after_residual, int out_dtype, void* stream);

/* Same contract in fp32 on CUDA cores (precision="fp32" parity mode). */
int tfimm_b200_gemm_f32(const float* A, int lda, const float* W, int ldw, const float* bias,
                        const float* gamma, const float* residual, int ldr, float* C, int ldc, int M, int N,
                        int K, int act, int act_after_residual, void* stream);

/* precision="tf32": fp32 storage, TF32 tensor-core products (TensorFlow's default for fp32 matmuls and convolutions
 * on Ampere and newer GPUs).  Same contract as tfimm_b200_gemm_bf16 with A, W, C, residual all fp32; the kernel rounds
 * every A element to TF32 (round to nearest, ties away from zero: cvt.rna.tf32.f32) in shared memory before the
 * product and accumulates in fp32; bias, activation, gamma and residual are applied in fp32.
 * PRECONDITION: W must already be TF32-representable (the low 13 bits of every element zero), i.e. rounded the same way
 * once, when the weights are prepared; the kernel does not round W.  K % 4 == 0; A, W, C, residual 16-byte aligned with
 * row strides of a multiple of 16 bytes.  force_block_n: 0 = auto; 64 / 128 = that tile width; 2 = the widest (128). */
int tfimm_b200_gemm_tf32(const float* A, int lda, const float* W, int ldw, const float* bias, const float* gamma,
                         const float* residual, int ldr, float* C, int ldc, int M, int N, int K, int act,
                         int act_after_residual, int force_block_n, void* stream);

/* Implicit k x k convolution of tfimm_b200_conv_bf16 in fp32 with TF32 products: x NHWC fp32 with C % 32 == 0,
 * W fp32 [N][k*k*C] (TF32-representable, as for tfimm_b200_gemm_tf32), out / residual NHWC fp32. */
int tfimm_b200_conv_tf32(const float* x, const float* W, int ldw, const float* bias, const float* residual, float* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act,
                         int act_after_residual, void* stream);

/* ViT self-attention of tfimm_b200_attention_bf16 on fp32 qkv / out with TF32 products: q, k, v rounded to TF32
 * (cvt.rna) as they are loaded, fp32 online softmax, P rounded to TF32 before P V, fp32 accumulation.  K / V stream
 * through shared memory in 64-key blocks, so N is not limited.  dh == 64 (other head dims: TFIMM_ERR_UNSUPPORTED). */
int tfimm_b200_attention_tf32(const float* qkv, float* out, int B, int N, int H, int dh, float scale, void* stream);

/* LayerNorm over the last axis, fp32 statistics (tfimm/layers/factory.py:37-45).
 * in_stride/out_stride in elements (lets the caller normalise only token 0 of each image:
 * tfimm/architectures/vit.py:452,462). */
int tfimm_b200_layernorm(const void* x, int in_dtype, long in_stride, const float* gamma, const float* beta,
                         void* out, int out_dtype, long out_stride, long rows, int C, float eps, void* stream);

/* LayerNorm per pixel of an NHWC map, written directly in the im2col layout of the following
 * 2x2 / stride-2 conv: out[(b, y/2, x/2), ((y%2)*2 + x%2)*C + c].
 * ConvNeXt downsample, tfimm/architectures/convnext.py:257-266,286-295. */
int tfimm_b200_layernorm_patch2x2(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                                  int out_dtype, int B, int H, int W, int C, float eps, void* stream);

/* Swin PatchMerging gather (neighbour order (0,0),(1,0),(0,1),(1,1)) + LayerNorm over 4C;
 * tfimm/architectures/swin.py:348-362.  out: (B*H/2*W/2, 4C). */
int tfimm_b200_patch_merge_ln(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                              int out_dtype, int B, int H, int W, int C, float eps, void* stream);

/* Fused softmax(scale * q k^T) v over the packed qkv projection (B*N, 3*H*dh), column order
 * [q|k|v] each head-major; out (B*N, H*dh).  tfimm/architectures/vit.py:149-165. bf16, dh == 64. */
int tfimm_b200_attention_bf16(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* stream);

/* Attention for the first nq query tokens only (class / distillation tokens) against all N keys: the attention core
 * of the LAST ViT block, whose other query rows cannot reach the logits (ViT.forward_features keeps token 0, or
 * tokens 0..1 for distilled models: tfimm/architectures/vit.py:452-464).  qkv: bf16 [B*N][3*H*64] (same packing as
 * tfimm_b200_attention_bf16); out: bf16 [B*nq][H*64]. */
int tfimm_b200_attention_cls_bf16(const void* qkv, void* out, int B, int N, int H, int head_dim, int nq, float scale,
                                  void* stream);

/* fp32 attention with optional additive bias[H,N,N] and mask[nmask,N,N] (window b uses mask b % nmask)
 * and optional probability output probs[B,H,N,N] (features["attn"], vit.py:163).
 * row_map (optional, int32[nw_img*N]): window b reads/writes image (b / nw_img), token
 * row_map[(b % nw_img)*N + j] -- the tf.roll + window_partition / window_reverse + tf.roll permutation of
 * SwinTransformerBlock.call (swin.py:299-313) folded into addressing.
 * Covers vit.py:149-165 and swin.py:172-194 in precision="fp32". */
int tfimm_b200_attention_f32(const float* qkv, float* out, const float* bias, const float* mask, int nmask,
                             long B, int N, int H, int dh, float scale, float* probs, const int* row_map,
                             int nw_img, void* stream);

/* Swin (shifted-)window attention, bf16, head_dim 32, N = window_size^2 <= 144 tokens per window (mma.sync; instantiated for
 * 64 and 144 padded rows -- the latter serves the 12 x 12 windows of the *_window12_384 models):
 * softmax(scale q k^T + bias[h] + mask) v per (window, head) with the cyclic shift and window
 * partition/reverse folded into row addressing (row_map as above).  labels (optional, int32[nw_img*N]):
 * region ids of the shifted-window mask; tokens with different ids get -100 added, exactly the
 * attn_mask of swin.py:249-273.  qkv:(B*L, 3*H*dh) in token order, out:(B*L, H*dh), L = nw_img*N.
 * Replaces swin.py:159-198 + 299-313. */
int tfimm_b200_window_attention_bf16(const void* qkv, void* out, const float* bias, const int* row_map,
                                     const int* labels, int B, int nw_img, int N, int H, int dh, float scale,
                                     void* stream);

/* Same operator with the bias and mask in the layout the model precomputes for 7 x 7 windows (head_dim 32, N <= 52
 * tokens per window; the mma.sync kernel above, one warp per (window, head)).
 * bias_pad: fp32 [H][64][64] (the gathered relative-position bias, rows / columns >= N unused);
 * maskbits: uint64 [nw_img][64], bit j of entry (w, i) set when tokens i and j of window w are in different shift
 * regions (the -100 entries of swin.py:249-273), or NULL for unshifted blocks. */
int tfimm_b200_window_attention_tc_bf16(const void* qkv, void* out, const float* bias_pad, const int* row_map,
                                        const void* maskbits, int B, int nw_img, int N, int H, int dh, float scale,
                                        void* stream);

/* Non-overlapping p x p patch gather (im2col of Conv2D(k=p, s=p, VALID)); out (B*H/p*W/p, Kpad),
 * column order (ky, kx, c), zero-padded to Kpad.  Optional fused create_preprocessing:
 * v = (x*scale - mean[c]) * inv_std[c] (tfimm/models/factory.py:153-169).
 * tfimm/layers/transformers.py:128-139, convnext.py:319-326. */
int tfimm_b200_patchify(const void* img, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C,
                        int p, int Kpad, float scale, const float* mean, const float* inv_std, void* stream);

/* x[b] = concat(cls, [dist], patches[b]) + pos_embed;  tfimm/architectures/vit.py:427-434. */
int tfimm_b200_assemble_tokens(const void* patches, int patch_dtype, const float* cls, const float* dist,
                               const float* pos, void* out, int out_dtype, int B, int P, int ntok, int D,
                               void* stream);

/* ZeroPadding2D(k/2) -> DepthwiseConv2D(k x k, stride 1, bias) -> LayerNorm over C (k == 7):
 * first half of ConvNeXtBlock.call, tfimm/architectures/convnext.py:189-198,219-223.
 * x:(B,H,W,C) f32|bf16, wgt: fp32 [k*k][C] (= TF depthwise_kernel (k,k,C,1) flattened), out:(B*H*W, C). */
int tfimm_b200_dwconv_ln(const void* x, int in_dtype, const float* wgt, const float* bias, const float* gamma,
                         const float* beta, void* out, int out_dtype, int B, int H, int W, int C, int ks,
                         float eps, void* stream);

/* DepthwiseConv2D(k in {3,5,7}, stride in {1,2}) with explicit top/left zero padding (covers TF "same"
 * and PadDepthwiseConv2D "symmetric", tfimm/layers/conv.py:91-148) + per-channel bias (folded BatchNorm)
 * + activation; optional fused squeeze: pool_sum[b][c] += sum over the output pixels (fp32 atomics; the
 * caller zeroes it and divides by Ho*Wo).  tfimm/architectures/efficientnet_blocks.py:312-323,393-404,241-242. */
int tfimm_b200_dwconv_bias_act(const void* x, int dtype, const float* wgt, const float* bias, void* out,
                               float* pool_sum, int B, int H, int W, int C, int ks, int stride, int pad_t,
                               int pad_l, int Ho, int Wo, int act, void* stream);

/* Mean over the spatial axis: (B, HW, C) -> (B, C) fp32.  GlobalAveragePooling (convnext.py:433,
 * efficientnet.py:256, swin.py:456, layers/classifier.py:34). */
int tfimm_b200_global_avg_pool(const void* x, int dtype, float* out, int B, int HW, int C, void* stream);

/* im2col for dense k x k convolutions (stems, fused-MBConv / ResNet 3x3, 7x7) that then run as tensor-core
 * GEMMs: out[(b,oy,ox), (ky,kx,c)] = x[b, oy*s+ky-pad_t, ox*s+kx-pad_l, c], zero outside / beyond k*k*C.
 * Replaces the gather half of tf.keras.layers.Conv2D at efficientnet.py:216-222,
 * efficientnet_blocks.py:482-497 (conv_exp), resnet.py:130-137,230-238,506-512.
 * groups > 1 (wide ResNeXt groups, resnet.py:230-238 with cardinality 32 and >= 48 channels per group):
 * out[g][(b,oy,ox)][(ky,kx,c)] with c < C/groups, i.e. one [M][Kpad] matrix per group, each followed by its own GEMM. */
int tfimm_b200_im2col(const void* x, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C, int groups,
                      int ks, int stride, int pad_t, int pad_l, int Ho, int Wo, int Kpad, void* stream);

/* Same gather from RAW uint8 pixels (the stems of the convolutional families) with the reference's preprocessing fused in:
 * every in-bounds value is (v * scale - mean[c]) * inv_std[c] (create_preprocessing, tfimm/models/factory.py:153-169),
 * the zero padding stays zero.  mean / inv_std: fp32 [C] on the device.  The host then uploads 1 byte per value
 * instead of 4 (EfficientNet-B4 at 380 px, batch 256: 111 MB instead of 443 MB per step). */
int tfimm_b200_im2col_u8(const void* x, void* out, int out_dtype, int B, int H, int W, int C, int ks, int stride,
                         int pad_t, int pad_l, int Ho, int Wo, int Kpad, float scale, const float* mean,
                         const float* inv_std, void* stream);

/* GroupNormalization over NHWC (tfimm/layers/norm.py:22-101, norm_layer "group_norm" = 32 groups, eps 1e-5;
 * used by resnet50_gn in place of every BatchNormalization): moments over (H, W, C/groups) per image and group,
 * biased variance, per-channel gamma/beta, then optional "+ residual" and activation (resnet.py:284-290).
 * stats: workspace of B * groups * 2 floats. */
int tfimm_b200_group_norm(const void* x, int dtype, const float* gamma, const float* beta, const void* residual,
                          void* out, float* stats, int B, int HW, int C, int groups, float eps, int act, void* stream);

/* BlurPool2D (tfimm/layers/blurpool.py:54-62; resnetblur50: resnet.py:127-140, 218-241, 532-536): REFLECT pad 1,
 * depthwise [1 2 1] x [1 2 1] / 16, stride s, VALID.  Ho = (H - 1) / s + 1. */
int tfimm_b200_blur_pool(const void* x, int dtype, void* out, int B, int H, int W, int C, int stride, int Ho, int Wo,
                         void* stream);

/* SqueezeExcite gate from pooled sums: gate[b] = gate_act(W_e act(W_r mean[b] + b_r) + b_e), fp32.
 * efficientnet_blocks.py:241-247 (mean -> conv_reduce -> act1 -> conv_expand -> gate), layers/attention.py:67-75.
 * w_reduce:[rd][C] (the TF kernel (1,1,C,rd) transposed), w_expand:[rd][C] (the TF kernel (1,1,rd,C) as is: the
 * expand loop then reads it coalesced across channels). */
int tfimm_b200_se_gate(const float* pooled_sum, float inv_hw, const float* w_reduce, const float* b_reduce,
                       const float* w_expand, const float* b_expand, float* gate, int B, int C, int rd, int act,
                       int gate_act, void* stream);

/* x[b, p, c] *= gate[b, c] in place (the "x * x_se" of efficientnet_blocks.py:247). */
int tfimm_b200_scale_channels(void* x, int dtype, const float* gate, int B, int HW, int C, void* stream);

/* Window pooling on NHWC: mode 0 = max (ResNet stem MaxPool2D after ZeroPadding2D, resnet.py:536-539;
 * mode 2 = max where out-of-bounds cells are explicit zeros, i.e. ZeroPadding2D + VALID MaxPool2D),
 * mode 1 = average over in-bounds cells (AveragePooling2D padding="same", resnet.py:299-301). */
int tfimm_b200_pool2d(const void* x, int dtype, void* out, int B, int H, int W, int C, int ks, int stride,
                      int pad_t, int pad_l, int Ho, int Wo, int mode, void* stream);

/* Grouped k x k convolution + folded-BN bias + activation (ResNeXt bottleneck conv2, resnet.py:230-238).
 * cg = channels per group (in == out, one of 4/8/16/32); wgt: fp32 [k*k][cg][C] == TF kernel (kh,kw,cg,C). */
int tfimm_b200_grouped_conv(const void* x, int dtype, const float* wgt, const float* bias, void* out, int B,
                            int H, int W, int C, int cg, int ks, int stride, int pad, int Ho, int Wo, int act,
                            void* stream);

/* EcaModule gate: sigmoid(Conv1D_k(mean) over the channel axis, zero padded); layers/attention.py:120-130. */
int tfimm_b200_eca_gate(const float* mean, const float* w, float* gate, int B, int C, int ks, void* stream);

/* x = act(x * gate[b] + shortcut) in place: tail of SE / ECA residual blocks (resnet.py:182-188, 284-291). */
int tfimm_b200_scale_add_act(void* x, int dtype, const float* gate, const void* shortcut, int B, int HW, int C,
                             int act, void* stream);

/* Segment Anything image-encoder attention with decomposed relative-position terms, for global and windowed blocks:
 * RelPosAttention.call + add_decomposed_rel_pos + window_partition / window_unpartition
 * (tfimm/architectures/segment_anything/image_encoder.py:231-263, 121-168, 11-73).  Per image and head,
 *     out_i = softmax_j(scale q_i . k_j + q_i . R_h[qy - ky + S_h - 1] + q_i . R_w[qx - kx + S_w - 1]) v_j
 * with the UNSCALED q in the relative-position terms.  qkv: [B * gh * gw][3 * H * dh] of the real tokens (row-major over
 * the gh x gw grid), column order [q | k | v] each head-major; out: [B * gh * gw][H * dh].
 * window == 0: one sequence of S_h x S_w = gh x gw tokens.  window > 0: S x S windows of the grid zero-padded to a
 * multiple of S; a padding position is a key with k = b_k and v = b_v taken from pad_bias ([3 * H * dh], the qkv bias;
 * NULL: zero keys), as in the reference, where the padded rows of norm1's output are projected by the qkv Dense.
 * Padding positions produce no output row.  rel_h: fp32 [2 S_h - 1][dh], rel_w: fp32 [2 S_w - 1][dh] (already resized
 * to the sequence extent, get_rel_pos image_encoder.py:76-118).  S_h, S_w <= 127.  No N x N tensor is materialised.
 * bf16: qkv / out / pad_bias bf16, dh 64 or 80, S_h + S_w <= 153 (dh 64) / <= 137 (dh 80) -- shared memory; other
 * shapes: TFIMM_ERR_UNSUPPORTED --, 64-key blocks streamed through shared memory, mma.sync products, fp32 online
 * softmax, P rounded to bf16 per block. */
int tfimm_b200_relpos_attention_bf16(const void* qkv, void* out, const void* pad_bias, const float* rel_h,
                                     const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                     void* stream);

/* Same contract in fp32 on CUDA cores (precision="fp32"), any head_dim; S_h * S_w up to ~13k tokens. */
int tfimm_b200_relpos_attention_f32(const float* qkv, float* out, const float* pad_bias, const float* rel_h,
                                    const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                    void* stream);

/* ---- MLP-Mixer family (MLP-Mixer, gMixer, ResMLP, gMLP) ----
 * Token mixing: a Dense layer applied along the token axis of a transposed activation -- `transpose -> Dense ->
 * transpose` of MixerBlock.call's mlp_tokens (tfimm/architectures/mlp_mixer.py:115-121), ResBlock.linear_tokens
 * (mlp_mixer.py:175-181) and SpatialGatingUnit.proj (tfimm/layers/transformers.py:376-383) -- without the transposes:
 *     out[b][m][c] = epi(sum_n Wt[m][n] X[b][n][c]),   b < imgs, m < M (rows of Wt), n < K (tokens in), c < N
 * Wt: bf16 [M][K], K-major, row stride ldw (a multiple of 8: the Dense kernel transposed and padded at plan time).
 * X: bf16, row stride ldx and image stride img_x (multiples of 8 elements), read where it is stored (MN-major wgmma
 * operand; a strided view such as gMLP's normalised v half works).  Epilogue, in this order:
 *   + bias[m] (per output ROW)  -> act, or with glu: rows come in groups of 16 (8 value rows, then their 8 gate rows)
 *   and stored row 8 (m / 16) + m % 8 is value * act(gate)  -> * gamma[c]  -> * mul[b][row][c] (gMLP's u half;
 *   row stride ld_mul, image stride img_mul)  -> + residual[b][row][c] (may alias out)  -> store at
 *   out + b * img_c + row * ldc + c.  Rows >= m_out are not stored.  out / residual / mul: out_dtype (bf16 / fp32).
 * force_block_n: 0 = auto; 64 / 128 / 256 = that tile width. */
int tfimm_b200_token_gemm_bf16(const void* Wt, int ldw, const void* X, long ldx, long img_x, const float* bias,
                               const float* gamma, const void* residual, long ldr, long img_r, const void* mul,
                               long ld_mul, long img_mul, void* out, long ldc, long img_c, int imgs, int M, int N, int K,
                               int m_out, int act, int glu, int out_dtype, int force_block_n, void* stream);

/* Same contract in fp32 on CUDA cores (precision="fp32"); ldw >= K, no alignment requirements. */
int tfimm_b200_token_gemm_f32(const float* Wt, int ldw, const float* X, long ldx, long img_x, const float* bias,
                              const float* gamma, const float* residual, long ldr, long img_r, const float* mul,
                              long ld_mul, long img_mul, float* out, long ldc, long img_c, int imgs, int M, int N, int K,
                              int m_out, int act, int glu, void* stream);

/* Channel GLU: GluMLP's fc1 + split + x * act(gates) (tfimm/layers/transformers.py:345-348, gMixer's mlp_channels) in
 * one GEMM.  W: bf16 [N][K] whose rows 2j / 2j + 1 are value / gate feature j (interleaved at plan time), bias [N]
 * likewise; out: bf16 [M][N / 2], row stride ldc = (value + bias) * act(gate + bias).  The full-width hidden tensor
 * is never written. */
int tfimm_b200_gemm_glu_bf16(const void* A, int lda, const void* W, int ldw, const float* bias, void* C, int ldc, int M,
                             int N, int K, int act, int force_block_n, void* stream);

/* fp32 form of the channel GLU on CUDA cores: W rows in the token GEMM's pairing (per 16 rows: 8 value features, then
 * their 8 gates; N % 16 == 0), out: fp32 [M][n_out]. */
int tfimm_b200_gemm_glu_f32(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc,
                            int M, int N, int n_out, int K, int act, void* stream);

/* ResMLP's Affine norm (tfimm/layers/norm.py:32-34): out[r][c] = alpha[c] * x[r][c] + beta[c]; fp32 x (row stride
 * ldx), out bf16 / fp32 (row stride ldo). */
int tfimm_b200_affine(const float* x, long ldx, const float* alpha, const float* beta, void* out, int out_dtype,
                      long ldo, long rows, int C, void* stream);

/* Elementwise dtype conversion. */
int tfimm_b200_cast(const void* in, int in_dtype, void* out, int out_dtype, long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_H_ */
