// extern "C" surface of libtfimm_b200.so (declared in include/tfimm_b200.h) plus the
// error-reporting plumbing shared by every translation unit.
#include "../../include/tfimm_b200.h"

#include <stdarg.h>

#include "common.cuh"

namespace tfimm {

namespace {
thread_local char g_last_error[1024] = "";
}

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_last_error("CUDA error in %s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return kCudaError;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  if (dev >= 0 && dev < 64 && cached[dev] > 0) return cached[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  if (dev >= 0 && dev < 64) cached[dev] = n;
  return n;
}

// implemented in the other translation units
int gemm_bf16_dispatch(const void*, int, const void*, int, const float*, const float*, const void*, int, void*,
                       int, int, int, int, int, int, int, int, cudaStream_t);
int attention_cls_bf16(const void*, void*, int, int, int, int, int, float, cudaStream_t);
int conv_bf16_dispatch(const void*, const void*, int, const float*, const void*, void*, int, int, int, int, int, int,
                       int, int, int, int, int, cudaStream_t);
int gemm_f32(const float*, int, const float*, int, const float*, const float*, const float*, int, float*, int,
             int, int, int, int, int, cudaStream_t);
int gemm_tf32_dispatch(const float*, int, const float*, int, const float*, const float*, const float*, int, float*, int,
                       int, int, int, int, int, int, cudaStream_t);
int conv_tf32_dispatch(const float*, const float*, int, const float*, const float*, float*, int, int, int, int, int, int,
                       int, int, int, int, cudaStream_t);
int attention_tf32(const float*, float*, int, int, int, int, float, cudaStream_t);
int layernorm_rows(const void*, int, long, const float*, const float*, void*, int, long, long, int, float,
                   cudaStream_t);
int layernorm_patch2x2(const void*, int, const float*, const float*, void*, int, int, int, int, int, float,
                       cudaStream_t);
int patch_merge_ln(const void*, int, const float*, const float*, void*, int, int, int, int, int, float,
                   cudaStream_t);
int attention_bf16(const void*, void*, int, int, int, int, float, cudaStream_t);
int attention_f32(const float*, float*, const float*, const float*, int, long, int, int, int, float, float*,
                  const int*, int, cudaStream_t);
int window_attention_bf16(const void*, void*, const float*, const int*, const int*, int, int, int, int, int,
                          float, cudaStream_t);
int window_attention_tc_bf16(const void*, void*, const float*, const int*, const unsigned long long*, int, int, int, int,
                             int, float, cudaStream_t);
int gemm_bf16_gated_dispatch(const void*, int, const float*, int, int, const void*, int, const float*, const void*, int,
                             void*, int, int, int, int, int, cudaStream_t);
int mlp_fused_bf16(const void*, int, const void*, int, const float*, const void*, int, const float*, const float*,
                   const void*, int, void*, int, int, int, int, int, cudaStream_t);
int patchify(const void*, int, void*, int, int, int, int, int, int, int, float, const float*, const float*,
             cudaStream_t);
int assemble_tokens(const void*, int, const float*, const float*, const float*, void*, int, int, int, int, int,
                    cudaStream_t);
int cast_tensor(const void*, int, void*, int, long, cudaStream_t);
int dwconv_ln(const void*, int, const float*, const float*, const float*, const float*, void*, int, int, int,
              int, int, int, float, cudaStream_t);
int dwconv_bias_act(const void*, int, const float*, const float*, void*, float*, int, int, int, int, int, int,
                    int, int, int, int, int, cudaStream_t);
int global_avg_pool(const void*, int, float*, int, int, int, cudaStream_t);
int im2col(const void*, int, void*, int, int, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t, float,
           const float*, const float*);
int group_norm(const void*, int, const float*, const float*, const void*, void*, float*, int, int, int, int, float, int,
               cudaStream_t);
int blur_pool(const void*, int, void*, int, int, int, int, int, int, int, cudaStream_t);
int se_gate(const float*, float, const float*, const float*, const float*, const float*, float*, int, int, int,
            int, int, cudaStream_t);
int scale_channels(void*, int, const float*, int, int, int, cudaStream_t);
int pool2d(const void*, int, void*, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int grouped_conv(const void*, int, const float*, const float*, void*, int, int, int, int, int, int, int, int, int,
                 int, int, cudaStream_t);
int eca_gate(const float*, const float*, float*, int, int, int, cudaStream_t);
int scale_add_act(void*, int, const float*, const void*, int, int, int, int, cudaStream_t);
int relpos_attention_bf16(const void*, void*, const void*, const float*, const float*, int, int, int, int, int, int,
                          float, cudaStream_t);
int relpos_attention_f32(const float*, float*, const float*, const float*, const float*, int, int, int, int, int, int,
                         float, cudaStream_t);

int token_gemm_bf16_dispatch(const void*, int, const void*, long, long, const float*, const float*, const void*, long,
                             long, const void*, long, long, void*, long, long, int, int, int, int, int, int, int, int,
                             int, cudaStream_t);
int token_gemm_f32(const float*, int, const float*, long, long, const float*, const float*, const float*, long, long,
                   const float*, long, long, float*, long, long, int, int, int, int, int, int, int, cudaStream_t);
int gemm_glu_bf16_dispatch(const void*, int, const void*, int, const float*, void*, int, int, int, int, int, int,
                           cudaStream_t);
int gemm_glu_f32(const float*, int, const float*, int, const float*, float*, int, int, int, int, int, int, cudaStream_t);
int affine(const float*, long, const float*, const float*, void*, int, long, long, int, cudaStream_t);

}  // namespace tfimm

using tfimm::set_last_error;
static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

const char* tfimm_b200_version(void) { return "tfimm_b200 0.1.0 (sm_90a)"; }
const char* tfimm_b200_last_error(void) { return tfimm::g_last_error; }
int tfimm_b200_sm_count(void) { return tfimm::sm_count(); }

int tfimm_b200_gemm_bf16(const void* A, int lda, const void* W, int ldw, const float* bias, const float* gamma,
                         const void* residual, int ldr, void* C, int ldc, int M, int N, int K, int act,
                         int act_after_residual, int out_dtype, int force_block_n, void* stream) {
  return tfimm::gemm_bf16_dispatch(A, lda, W, ldw, bias, gamma, residual, ldr, C, ldc, M, N, K, act,
                                   act_after_residual, out_dtype, force_block_n, S(stream));
}

int tfimm_b200_conv_bf16(const void* x, const void* W, int ldw, const float* bias, const void* residual, void* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act,
                         int act_after_residual, int out_dtype, void* stream) {
  return tfimm::conv_bf16_dispatch(x, W, ldw, bias, residual, out, B, H, Wd, C, N, ks, stride, pad, act,
                                   act_after_residual, out_dtype, S(stream));
}

int tfimm_b200_attention_cls_bf16(const void* qkv, void* out, int B, int N, int H, int head_dim, int nq, float scale,
                                  void* stream) {
  return tfimm::attention_cls_bf16(qkv, out, B, N, H, head_dim, nq, scale, S(stream));
}

int tfimm_b200_gemm_f32(const float* A, int lda, const float* W, int ldw, const float* bias, const float* gamma,
                        const float* residual, int ldr, float* C, int ldc, int M, int N, int K, int act,
                        int act_after_residual, void* stream) {
  return tfimm::gemm_f32(A, lda, W, ldw, bias, gamma, residual, ldr, C, ldc, M, N, K, act, act_after_residual,
                         S(stream));
}

int tfimm_b200_gemm_tf32(const float* A, int lda, const float* W, int ldw, const float* bias, const float* gamma,
                         const float* residual, int ldr, float* C, int ldc, int M, int N, int K, int act,
                         int act_after_residual, int force_block_n, void* stream) {
  return tfimm::gemm_tf32_dispatch(A, lda, W, ldw, bias, gamma, residual, ldr, C, ldc, M, N, K, act, act_after_residual,
                                   force_block_n, S(stream));
}

int tfimm_b200_conv_tf32(const float* x, const float* W, int ldw, const float* bias, const float* residual, float* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act,
                         int act_after_residual, void* stream) {
  return tfimm::conv_tf32_dispatch(x, W, ldw, bias, residual, out, B, H, Wd, C, N, ks, stride, pad, act,
                                   act_after_residual, S(stream));
}

int tfimm_b200_attention_tf32(const float* qkv, float* out, int B, int N, int H, int dh, float scale, void* stream) {
  return tfimm::attention_tf32(qkv, out, B, N, H, dh, scale, S(stream));
}

int tfimm_b200_layernorm(const void* x, int in_dtype, long in_stride, const float* gamma, const float* beta,
                         void* out, int out_dtype, long out_stride, long rows, int C, float eps, void* stream) {
  return tfimm::layernorm_rows(x, in_dtype, in_stride, gamma, beta, out, out_dtype, out_stride, rows, C, eps,
                               S(stream));
}

int tfimm_b200_layernorm_patch2x2(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                                  int out_dtype, int B, int H, int W, int C, float eps, void* stream) {
  return tfimm::layernorm_patch2x2(x, in_dtype, gamma, beta, out, out_dtype, B, H, W, C, eps, S(stream));
}

int tfimm_b200_patch_merge_ln(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                              int out_dtype, int B, int H, int W, int C, float eps, void* stream) {
  return tfimm::patch_merge_ln(x, in_dtype, gamma, beta, out, out_dtype, B, H, W, C, eps, S(stream));
}

int tfimm_b200_attention_bf16(const void* qkv, void* out, int B, int N, int H, int dh, float scale,
                              void* stream) {
  return tfimm::attention_bf16(qkv, out, B, N, H, dh, scale, S(stream));
}

int tfimm_b200_attention_f32(const float* qkv, float* out, const float* bias, const float* mask, int nmask,
                             long B, int N, int H, int dh, float scale, float* probs, const int* row_map,
                             int nw_img, void* stream) {
  return tfimm::attention_f32(qkv, out, bias, mask, nmask, B, N, H, dh, scale, probs, row_map, nw_img, S(stream));
}

int tfimm_b200_window_attention_bf16(const void* qkv, void* out, const float* bias, const int* row_map,
                                     const int* labels, int B, int nw_img, int N, int H, int dh, float scale,
                                     void* stream) {
  return tfimm::window_attention_bf16(qkv, out, bias, row_map, labels, B, nw_img, N, H, dh, scale, S(stream));
}

int tfimm_b200_window_attention_tc_bf16(const void* qkv, void* out, const float* bias_pad, const int* row_map,
                                        const void* maskbits, int B, int nw_img, int N, int H, int dh, float scale,
                                        void* stream) {
  return tfimm::window_attention_tc_bf16(qkv, out, bias_pad, row_map,
                                         reinterpret_cast<const unsigned long long*>(maskbits), B, nw_img, N, H, dh,
                                         scale, S(stream));
}

int tfimm_b200_gemm_bf16_gated(const void* A, int lda, const float* gate, int rows_per_image, int n_images,
                               const void* W, int ldw, const float* bias, const void* residual, int ldr, void* C,
                               int ldc, int M, int N, int K, int act, void* stream) {
  return tfimm::gemm_bf16_gated_dispatch(A, lda, gate, rows_per_image, n_images, W, ldw, bias, residual, ldr, C, ldc, M,
                                         N, K, act, S(stream));
}

int tfimm_b200_mlp_bf16(const void* A, int lda, const void* W1, int ldw1, const float* b1, const void* W2, int ldw2,
                        const float* b2, const float* gamma, const void* residual, int ldr, void* out, int ldc, int M,
                        int C, int hidden, int act, void* stream) {
  return tfimm::mlp_fused_bf16(A, lda, W1, ldw1, b1, W2, ldw2, b2, gamma, residual, ldr, out, ldc, M, C, hidden, act,
                               S(stream));
}

int tfimm_b200_patchify(const void* img, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C,
                        int p, int Kpad, float scale, const float* mean, const float* inv_std, void* stream) {
  return tfimm::patchify(img, in_dtype, out, out_dtype, B, H, W, C, p, Kpad, scale, mean, inv_std, S(stream));
}

int tfimm_b200_assemble_tokens(const void* patches, int patch_dtype, const float* cls, const float* dist,
                               const float* pos, void* out, int out_dtype, int B, int P, int ntok, int D,
                               void* stream) {
  return tfimm::assemble_tokens(patches, patch_dtype, cls, dist, pos, out, out_dtype, B, P, ntok, D, S(stream));
}

int tfimm_b200_cast(const void* in, int in_dtype, void* out, int out_dtype, long n, void* stream) {
  return tfimm::cast_tensor(in, in_dtype, out, out_dtype, n, S(stream));
}

int tfimm_b200_dwconv_ln(const void* x, int in_dtype, const float* wgt, const float* bias, const float* gamma,
                         const float* beta, void* out, int out_dtype, int B, int H, int W, int C, int ks,
                         float eps, void* stream) {
  return tfimm::dwconv_ln(x, in_dtype, wgt, bias, gamma, beta, out, out_dtype, B, H, W, C, ks, eps, S(stream));
}

int tfimm_b200_dwconv_bias_act(const void* x, int dtype, const float* wgt, const float* bias, void* out,
                               float* pool_sum, int B, int H, int W, int C, int ks, int stride, int pad_t,
                               int pad_l, int Ho, int Wo, int act, void* stream) {
  return tfimm::dwconv_bias_act(x, dtype, wgt, bias, out, pool_sum, B, H, W, C, ks, stride, pad_t, pad_l, Ho, Wo,
                                act, S(stream));
}

int tfimm_b200_global_avg_pool(const void* x, int dtype, float* out, int B, int HW, int C, void* stream) {
  return tfimm::global_avg_pool(x, dtype, out, B, HW, C, S(stream));
}

int tfimm_b200_im2col(const void* x, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C, int groups,
                      int ks, int stride, int pad_t, int pad_l, int Ho, int Wo, int Kpad, void* stream) {
  return tfimm::im2col(x, in_dtype, out, out_dtype, B, H, W, C, groups, ks, stride, pad_t, pad_l, Ho, Wo, Kpad,
                       S(stream), 1.0f, nullptr, nullptr);
}

int tfimm_b200_im2col_u8(const void* x, void* out, int out_dtype, int B, int H, int W, int C, int ks, int stride,
                         int pad_t, int pad_l, int Ho, int Wo, int Kpad, float scale, const float* mean,
                         const float* inv_std, void* stream) {
  return tfimm::im2col(x, tfimm::kU8, out, out_dtype, B, H, W, C, 1, ks, stride, pad_t, pad_l, Ho, Wo, Kpad, S(stream),
                       scale, mean, inv_std);
}

int tfimm_b200_group_norm(const void* x, int dtype, const float* gamma, const float* beta, const void* residual,
                          void* out, float* stats, int B, int HW, int C, int groups, float eps, int act,
                          void* stream) {
  return tfimm::group_norm(x, dtype, gamma, beta, residual, out, stats, B, HW, C, groups, eps, act, S(stream));
}

int tfimm_b200_blur_pool(const void* x, int dtype, void* out, int B, int H, int W, int C, int stride, int Ho, int Wo,
                         void* stream) {
  return tfimm::blur_pool(x, dtype, out, B, H, W, C, stride, Ho, Wo, S(stream));
}

int tfimm_b200_se_gate(const float* pooled_sum, float inv_hw, const float* w_reduce, const float* b_reduce,
                       const float* w_expand, const float* b_expand, float* gate, int B, int C, int rd, int act,
                       int gate_act, void* stream) {
  return tfimm::se_gate(pooled_sum, inv_hw, w_reduce, b_reduce, w_expand, b_expand, gate, B, C, rd, act, gate_act,
                        S(stream));
}

int tfimm_b200_scale_channels(void* x, int dtype, const float* gate, int B, int HW, int C, void* stream) {
  return tfimm::scale_channels(x, dtype, gate, B, HW, C, S(stream));
}

int tfimm_b200_pool2d(const void* x, int dtype, void* out, int B, int H, int W, int C, int ks, int stride,
                      int pad_t, int pad_l, int Ho, int Wo, int mode, void* stream) {
  return tfimm::pool2d(x, dtype, out, B, H, W, C, ks, stride, pad_t, pad_l, Ho, Wo, mode, S(stream));
}

int tfimm_b200_grouped_conv(const void* x, int dtype, const float* wgt, const float* bias, void* out, int B,
                            int H, int W, int C, int cg, int ks, int stride, int pad, int Ho, int Wo, int act,
                            void* stream) {
  return tfimm::grouped_conv(x, dtype, wgt, bias, out, B, H, W, C, cg, ks, stride, pad, Ho, Wo, act, S(stream));
}

int tfimm_b200_eca_gate(const float* mean, const float* w, float* gate, int B, int C, int ks, void* stream) {
  return tfimm::eca_gate(mean, w, gate, B, C, ks, S(stream));
}

int tfimm_b200_scale_add_act(void* x, int dtype, const float* gate, const void* shortcut, int B, int HW, int C,
                             int act, void* stream) {
  return tfimm::scale_add_act(x, dtype, gate, shortcut, B, HW, C, act, S(stream));
}

int tfimm_b200_relpos_attention_bf16(const void* qkv, void* out, const void* pad_bias, const float* rel_h,
                                     const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                     void* stream) {
  return tfimm::relpos_attention_bf16(qkv, out, pad_bias, rel_h, rel_w, B, gh, gw, H, dh, window, scale, S(stream));
}

int tfimm_b200_relpos_attention_f32(const float* qkv, float* out, const float* pad_bias, const float* rel_h,
                                    const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                    void* stream) {
  return tfimm::relpos_attention_f32(qkv, out, pad_bias, rel_h, rel_w, B, gh, gw, H, dh, window, scale, S(stream));
}

}  // extern "C"

int tfimm_b200_token_gemm_bf16(const void* Wt, int ldw, const void* X, long ldx, long img_x, const float* bias,
                               const float* gamma, const void* residual, long ldr, long img_r, const void* mul,
                               long ld_mul, long img_mul, void* out, long ldc, long img_c, int imgs, int M, int N, int K,
                               int m_out, int act, int glu, int out_dtype, int force_block_n, void* stream) {
  return tfimm::token_gemm_bf16_dispatch(Wt, ldw, X, ldx, img_x, bias, gamma, residual, ldr, img_r, mul, ld_mul, img_mul,
                                         out, ldc, img_c, imgs, M, N, K, m_out, act, glu, out_dtype, force_block_n,
                                         S(stream));
}

int tfimm_b200_token_gemm_f32(const float* Wt, int ldw, const float* X, long ldx, long img_x, const float* bias,
                              const float* gamma, const float* residual, long ldr, long img_r, const float* mul,
                              long ld_mul, long img_mul, float* out, long ldc, long img_c, int imgs, int M, int N, int K,
                              int m_out, int act, int glu, void* stream) {
  return tfimm::token_gemm_f32(Wt, ldw, X, ldx, img_x, bias, gamma, residual, ldr, img_r, mul, ld_mul, img_mul, out, ldc,
                               img_c, imgs, M, N, K, m_out, act, glu, S(stream));
}

int tfimm_b200_gemm_glu_bf16(const void* A, int lda, const void* W, int ldw, const float* bias, void* C, int ldc, int M,
                             int N, int K, int act, int force_block_n, void* stream) {
  return tfimm::gemm_glu_bf16_dispatch(A, lda, W, ldw, bias, C, ldc, M, N, K, act, force_block_n, S(stream));
}

int tfimm_b200_gemm_glu_f32(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc,
                            int M, int N, int n_out, int K, int act, void* stream) {
  return tfimm::gemm_glu_f32(A, lda, W, ldw, bias, C, ldc, M, N, n_out, K, act, S(stream));
}

int tfimm_b200_affine(const float* x, long ldx, const float* alpha, const float* beta, void* out, int out_dtype,
                      long ldo, long rows, int C, void* stream) {
  return tfimm::affine(x, ldx, alpha, beta, out, out_dtype, ldo, rows, C, S(stream));
}
