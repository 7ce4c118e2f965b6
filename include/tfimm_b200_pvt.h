/* tfimm_b200 -- C ABI of the PVT family's kernels (csrc/pvt.cu), in libtfimm_b200.so beside the core entry points of
 * tfimm_b200.h, with the same conventions: device pointers owned by the caller, a status return (0 = OK, else a
 * TFIMM_ERR_* code with tfimm_b200_last_error()), the stream last.  The in-tree ctypes table is in
 * tensorflow-image-models_b200/tfimm/backend/lib.py, the launchers in pvt_ops.py.
 *
 * Spatial-reduction attention (the reference's SpatialReductionAttention): the queries come from all N tokens of an
 * image, the keys and values from N' tokens (the stage grid reduced by a stride-sr convolution, or the tokens
 * themselves when sr = 1).  q: (B * N, H * dh), the q Dense's output; kv: (B * N', 2 * H * dh), the kv Dense's output
 * read as (B, N', 2, H, dh): k of head h at columns h * dh .., v at H * dh + h * dh ..; out: (B * N, H * dh). */
#ifndef TFIMM_B200_PVT_H_
#define TFIMM_B200_PVT_H_

#include "tfimm_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* out = softmax(scale q k^T) v per image and head in bf16 on the tensor cores: 64-key blocks of an online softmax, P
 * rounded to bf16 per block, the output divided by the row sum with correct rounding.  Any N >= 1 and Nk >= 1; dh 64;
 * B, H <= 65535; q, kv and out 16-byte aligned. */
int tfimm_b200_pvt_sr_attention_bf16(const void* q, const void* kv, void* out, int B, int N, int Nk, int H, int dh,
                                     float scale, void* stream);

/* The same in fp32 on the CUDA cores (fp32 online softmax with expf).  dh 64; q, kv and out 16-byte aligned. */
int tfimm_b200_pvt_sr_attention_f32(const float* q, const float* kv, float* out, int B, int N, int Nk, int H, int dh,
                                    float scale, void* stream);

/* The end of a stage's patch embedding, into the fp32 residual stream out (B * (ntok + P), C):
 *   out[b, ntok + p] = LayerNorm_eps(tok[b, p]) * gamma + beta + pos[ntok + p]   (tok: fp32 (B * P, C))
 *   out[b, 0]        = cls + pos[0]                                              (only when ntok = 1)
 * pos: fp32 (ntok + P, C); cls: fp32 (C), ignored when ntok = 0.  ntok 0 or 1; C % 4 == 0, C <= 1024; every pointer
 * 16-byte aligned. */
int tfimm_b200_pvt_embed_norm(const float* tok, const float* gamma, const float* beta, const float* pos,
                              const float* cls, float* out, int B, int P, int ntok, int C, float eps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFIMM_B200_PVT_H_ */
