/* tfimm_b200 -- C ABI of the PoolFormer family's kernels (csrc/poolformer.cu), in libtfimm_b200.so beside the core
 * entry points of tfimm_b200.h, with the same conventions: device pointers owned by the caller, channels-last fp32
 * residual stream, a status return (0 = OK, else a TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.
 * The in-tree ctypes table is in tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in
 * poolformer_ops.py.
 *
 * GroupNorm with one group (tfimm/layers/norm.py:22-101, norm_layer "group_norm_1grp", eps 1e-5, biased variance)
 * normalises over a whole image.  Its statistics are kept as PARTIALS: image b's H * W * C values, flattened, are split
 * into `splits` = ceil(H * W * C / 4096) chunks of 4096, and partials[b][s] = (count, mean, M2) of chunk s, M2 the sum
 * of squares about the chunk's own mean.  Every kernel that needs an image's mean and variance merges its `splits`
 * partials itself (Chan's formula, in a fixed order), so the results do not depend on launch timing.
 * partials: fp32 [B][splits][3]. */
#ifndef TFIMM_B200_POOLFORMER_H_
#define TFIMM_B200_POOLFORMER_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Partials of x (B, H, W, C) fp32, C % 4 == 0: the statistics half of PoolFormerBlock's norm1 / norm2
 * (tfimm/architectures/poolformer.py:190, 197) and of the head norm (poolformer.py:320) for a tensor no PoolFormer
 * kernel wrote (the stem, a downsample, an MLP output). */
int tfimm_b200_gn1_partials(const float* x, float* partials, int B, int H, int W, int C, int splits, void* stream);

/* PoolFormer's token mixer, x + ls1 * (AvgPool3x3_same(GN(x)) - GN(x)) (tfimm/architectures/poolformer.py:189-194),
 * computed as out = x + ls1[c] gamma[c] rstd_b * mean over the in-bounds 3 x 3 neighbours j of (x_j - x), with rstd_b
 * from x's partials: beta and the mean cancel.  out must not alias x; out_partials (the next norm's statistics) are
 * written from the values the kernel stores. */
int tfimm_b200_poolformer_mixer(const float* x, const float* partials, const float* gamma, const float* ls1, float* out,
                                float* out_partials, int B, int H, int W, int C, int splits, float eps, void* stream);

/* GN(x) = (x - mean_b) rstd_b gamma[c] + beta[c] from x's partials (poolformer.py:197, 320), out (B * H * W, C) of
 * out_dtype (bf16: the fc1 operand; f32: features_all and the fp32 / tf32 fc1 operand). */
int tfimm_b200_gn1_apply(const float* x, const float* partials, const float* gamma, const float* beta, void* out,
                         int out_dtype, int B, int H, int W, int C, int splits, float eps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_POOLFORMER_H_ */
