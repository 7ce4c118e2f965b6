/* tfimm_b200 -- C ABI of the CaiT family's kernels (csrc/cait.cu), in libtfimm_b200.so beside the core entry points of
 * tfimm_b200.h, with the same conventions: device pointers owned by the caller, a status return (0 = OK, else a
 * TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.  The in-tree ctypes table is in
 * tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in cait_ops.py.
 *
 * Talking-heads attention (tfimm/architectures/cait.py:207-258), per image and query:
 *     L_g  = sum_h wl[h, g] (q_h . k_h) + bl[g]                 (log2 units: the caller folds dh^-0.5 log2 e into wl
 *                                                                and log2 e, not dh^-0.5, into bl)
 *     P_g  = 2^(L_g - max) / sum over keys of 2^(L_g - max)
 *     P'_f = sum_g P_g ww[g, f] + bw[f]
 *     O_f  = sum over keys of P'_f v_f
 * qkv is the (B * N, 3 * H * dh) output of the qkv Dense ([q | k | v], each head-major); out is (B * N, H * dh).
 * wl, ww: fp32 (H, H) row-major (h, g); bl, bw: fp32 (H). */
#ifndef TFIMM_B200_CAIT_H_
#define TFIMM_B200_CAIT_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bf16 qkv and out, dh 48 and H in {4, 6, 8, 16}, any N >= 1; on mma.sync, P' rounded to bf16 once as the P V operand.
 * qkv and out 16-byte aligned. */
int tfimm_b200_cait_talking_heads_bf16(const void* qkv, void* out, const float* wl, const float* bl, const float* ww,
                                       const float* bw, int B, int N, int H, int dh, void* stream);

/* fp32 qkv and out, H <= 16, dh % 4 == 0 and dh <= 64, any N >= 1; fp32 on the CUDA cores.  qkv 16-byte aligned. */
int tfimm_b200_cait_talking_heads_f32(const float* qkv, float* out, const float* wl, const float* bl, const float* ww,
                                      const float* bw, int B, int N, int H, int dh, void* stream);

/* Class attention (tfimm/architectures/cait.py:97-146): one query per image and head.  q (B, H * dh), kv
 * (B * T, 2 * H * dh) = [k | v] of all T rows of each image, out (B, H * dh) = softmax(scale q k^T) v; dtype
 * TFIMM_F32 or TFIMM_BF16 for all three, dh 32, 48 or 64, any T >= 1. */
int tfimm_b200_cait_class_attention(const void* q, const void* kv, void* out, int dtype, int B, int T, int H, int dh,
                                    float scale, void* stream);

/* x (B * N, D) fp32 += pos (N, D) fp32 for every image, in place: the position embedding of the patch tokens.  D % 4
 * == 0, x and pos 16-byte aligned. */
int tfimm_b200_cait_add_pos(float* x, const float* pos, int B, int N, int D, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_CAIT_H_ */
