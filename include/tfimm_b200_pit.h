/* tfimm_b200 -- C ABI of the PiT family's kernels (csrc/pit.cu), in libtfimm_b200.so beside the core entry points of
 * tfimm_b200.h, with the same conventions: device pointers owned by the caller, a status return (0 = OK, else a
 * TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.  The in-tree ctypes table is in
 * tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in pit_ops.py.
 *
 * The residual stream of image b is rows b * T .. b * T + T - 1 of an fp32 (B * T, C) matrix: nb_tokens special tokens
 * (class, then distillation) followed by the H x W grid in row-major order (tfimm/architectures/pit.py:345-349). */
#ifndef TFIMM_B200_PIT_H_
#define TFIMM_B200_PIT_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* out = softmax(scale q k^T) v per image and head, from the packed bf16 qkv (B * T, 3 * H * dh) the qkv GEMM writes
 * ([q | k | v], each head-major) into bf16 out (B * T, H * dh).  Any T >= 1; dh 32, 48 or 64.  qkv and out 16-byte
 * aligned. */
int tfimm_b200_pit_attention_bf16(const void* qkv, void* out, int B, int T, int H, int dh, float scale, void* stream);

/* The spatial half of ConvHeadPooling (tfimm/architectures/pit.py:172-188): ZeroPadding2D(1) and the 3 x 3 / 2
 * Conv2D with groups = C and 2C filters, plus bias, in fp32.  Reads grid rows nb_tokens .. of every image of x
 * (B * (nb_tokens + H * W), C); writes grid rows nb_tokens .. of out (B * (nb_tokens + Ho * Wo), 2C), Ho = (H - 1) / 2 + 1,
 * Wo = (W - 1) / 2 + 1; output channel o reads input channel o / 2.  w: fp32 (9, 2C), the (3, 3, 1, 2C) kernel's taps
 * in (ky, kx) order; bias: fp32 (2C).  tokens_bf16, when not null, receives the token rows of x rounded to bf16,
 * (B * nb_tokens, C): the bf16 operand of the token Dense.  C % 4 == 0; x, w, bias, out 16-byte aligned, tokens_bf16
 * 8-byte aligned. */
int tfimm_b200_pit_pool(const float* x, const float* w, const float* bias, float* out, void* tokens_bf16, int B,
                        int nb_tokens, int H, int W, int C, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_PIT_H_ */
