/* tfimm_b200 -- C ABI of the ConvMixer family's kernel (csrc/convmixer.cu), in libtfimm_b200.so beside the core entry
 * points of tfimm_b200.h, with the same conventions: device pointers owned by the caller, channels-last tensors, a
 * status return (0 = OK, else a TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.
 * The in-tree ctypes table is in tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in
 * convmixer_ops.py. */
#ifndef TFIMM_B200_CONVMIXER_H_
#define TFIMM_B200_CONVMIXER_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The token mixer of a ConvMixer block (tfimm/architectures/convmixer.py:63-68) with the previous BatchNorm folded in.
 * a: fp32 (B, H, W, C), the previous 1 x 1 convolution's (or the stem's) activation output, before its BatchNorm.
 *   x = s_in[c] a + t_in[c]                       at in-image positions; 0 in the "same" padding (by position)
 *   y = x + s1[c] act(depthwise_k(x) + bias[c]) + t1[c]
 * taps: fp32 [k * k][C] (the reference's depthwise_kernel (k, k, C, 1)); s_in, t_in, bias, s1, t1: fp32 [C].
 * y: (B, H, W, C) of y_dtype (TFIMM_BF16: the next GEMM's operand; TFIMM_F32 for the fp32 and tf32 precisions); y must
 * not alias a.  act: a TFIMM_ACT_* code.  k in {7, 9} and C % 32 == 0, else TFIMM_ERR_UNSUPPORTED.  Each output is a
 * fixed-order fp32 sum (no atomics): the result is bitwise reproducible. */
int tfimm_b200_convmixer_dwconv(const float* a, const float* s_in, const float* t_in, const float* taps,
                                const float* bias, const float* s1, const float* t1, void* y, int y_dtype, int B, int H,
                                int W, int C, int k, int act, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_CONVMIXER_H_ */
