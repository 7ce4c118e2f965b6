/* tfimm_b200 -- C ABI of the PVT v2 family's kernels (csrc/pvt_v2.cu), in libtfimm_b200.so beside the core entry points
 * of tfimm_b200.h, with the same conventions: device pointers owned by the caller, a status return (0 = OK, else a
 * TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.  The in-tree ctypes table is in
 * tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in pvt_v2_ops.py. */
#ifndef TFIMM_B200_PVT_V2_H_
#define TFIMM_B200_PVT_V2_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The ConvFFN of a PVT v2 block, fused, on the fp32 residual stream (out may be residual):
 *   out = residual + act(dwconv3x3(bf16(h w1^T + b1)) + bdw) w2^T + b2
 * h: bf16 (B * gh * gw, C), the tokens of each image in row-major grid order; w1: bf16 (hidden, C); b1: fp32 (hidden);
 * wdw: fp32 (9, hidden), the depthwise taps in (ky, kx) order; bdw: fp32 (hidden); w2: bf16 (C, hidden); b2: fp32
 * (C); residual, out: fp32 (B * gh * gw, C).  The convolution is stride 1 with one cell of zero padding: cells off the
 * map contribute 0.  The hidden activations are rounded to bf16 after b1 and after the activation, as the unfused
 * chain (GEMM, dwconv_bias_act, GEMM) stores them.  act: a TFIMM_ACT_* code.
 * Returns TFIMM_ERR_UNSUPPORTED unless C is 32, 64 or 128 and hidden % 64 == 0.  h, w1 and w2 16-byte aligned; the
 * fp32 pointers 8-byte aligned; B <= 65535. */
int tfimm_b200_pvt_v2_conv_mlp_bf16(const void* h, const void* w1, const float* b1, const float* wdw, const float* bdw,
                                    const void* w2, const float* b2, const float* residual, float* out, int B, int gh,
                                    int gw, int C, int hidden, int act, void* stream);

/* Spatial-reduction attention at head dim 32, as tfimm_b200_pvt_sr_attention_{bf16,f32} (tfimm_b200_pvt.h) do it at
 * head dim 64: q (B * N, H * 32), kv (B * N', 2 * H * 32) read as (B, N', 2, H, 32), out (B * N, H * 32).  dh must be
 * 32; q, kv and out 16-byte aligned; for bf16, B, H <= 65535. */
int tfimm_b200_pvt_v2_sr_attention_bf16(const void* q, const void* kv, void* out, int B, int N, int Nk, int H, int dh,
                                        float scale, void* stream);
int tfimm_b200_pvt_v2_sr_attention_f32(const float* q, const float* kv, float* out, int B, int N, int Nk, int H,
                                       int dh, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_PVT_V2_H_ */
