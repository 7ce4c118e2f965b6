// CUDA-core kernels of the MLP-Mixer family (tfimm/architectures/mlp_mixer.py); the bf16 contractions run on the wgmma
// GEMM (gemm_sm90.cu: token mixing, channel GLU).
//
//   token_gemm_f32_kernel  precision="fp32" form of the token-mixing GEMM, same contract as the wgmma instance:
//                              out[b][m][c] = epi(sum_k Wt[m][k] X[b][k][c])
//                          with X addressed through (token, channel) strides and the output through (row, column)
//                          strides, so the same kernel also runs the channel GLU (m = feature, c = token row).
//                          64 x 64 tiles, 4 x 4 micro-tiles, k-blocks of 16.  A thread's four rows are r, r + 8, r + 16,
//                          r + 24, so with glu it holds both rows of its value / gate pairs (8 value rows, then their 8
//                          gate rows, per 16).
//   affine_kernel          ResMLP's Affine norm, alpha[c] x + beta[c]: fp32 in, bf16 / fp32 out, HBM-bound.
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int TM = 64, TN = 64, TK = 16;

struct TokenF32Params {
  const float* wt; int ldw;
  const float* x; long x_img, x_k, x_c;
  const float* bias; const float* gamma;
  const float* res; long r_img, ldr;
  const float* mul; long u_img, ld_mul;
  float* out; long o_img, o_m, o_c;
  int M, N, K, m_out, act, glu;
};

__global__ void __launch_bounds__(256) token_gemm_f32_kernel(const TokenF32Params p) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Xs[TK][TN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const float* X = p.x + (long)b * p.x_img;
  const int r0 = 32 * (ty >> 3) + (ty & 7);   // rows r0 + 8 i
  float acc[4][4] = {};
  const int la = tid >> 2, lka = (tid & 3) * 4;   // Wt: row la, k lka..lka+3
  const int lkx = tid >> 4, lcx = (tid & 15) * 4;  // X: k lkx, channels lcx..lcx+3
  for (int k0 = 0; k0 < p.K; k0 += TK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + lka + j, m = m0 + la;
      As[lka + j][la] = (m < p.M && k < p.K) ? p.wt[(long)m * p.ldw + k] : 0.f;
      const int kx = k0 + lkx, c = n0 + lcx + j;
      Xs[lkx][lcx + j] = (kx < p.K && c < p.N) ? X[(long)kx * p.x_k + (long)c * p.x_c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float av[4], xv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][r0 + 8 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) xv[j] = Xs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], xv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + r0 + 8 * i;
    if (p.glu && (i & 1)) continue;   // gate rows are consumed with their value rows
    const int row = p.glu ? (m >> 4) * 8 + (m & 7) : m;
    if (m >= p.M || row >= p.m_out) continue;
    const float bm = p.bias != nullptr ? p.bias[m] : 0.f;
    const float bg = p.glu && p.bias != nullptr ? p.bias[m + 8] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = n0 + tx * 4 + j;
      if (c >= p.N) continue;
      float v = acc[i][j] + bm;
      v = p.glu ? v * apply_act<true>(acc[i + 1][j] + bg, p.act) : apply_act<true>(v, p.act);
      if (p.gamma != nullptr) v *= p.gamma[c];
      if (p.mul != nullptr) v *= p.mul[(long)b * p.u_img + (long)row * p.ld_mul + c];
      if (p.res != nullptr) v += p.res[(long)b * p.r_img + (long)row * p.ldr + c];
      p.out[(long)b * p.o_img + (long)row * p.o_m + (long)c * p.o_c] = v;
    }
  }
}

template <typename OutT>
__global__ void affine_kernel(const float* __restrict__ x, long ldx, const float* __restrict__ alpha,
                              const float* __restrict__ beta, OutT* __restrict__ out, long ldo, long rows, int C) {
  const long n = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    const float v = fmaf(__ldg(alpha + c), x[r * ldx + c], __ldg(beta + c));
    if constexpr (sizeof(OutT) == 2) out[r * ldo + c] = __float2bfloat16_rn(v);
    else out[r * ldo + c] = v;
  }
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

// Token mixing in fp32 (precision="fp32"): the contract of tfimm_b200_token_gemm_bf16 with fp32 operands and output.
int tfimm_b200_token_gemm_f32(const float* Wt, int ldw, const float* X, long ldx, long img_x, const float* bias,
                              const float* gamma, const float* residual, long ldr, long img_r, const float* mul,
                              long ld_mul, long img_mul, float* out, long ldc, long img_c, int imgs, int M, int N,
                              int K, int m_out, int act, int glu, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(imgs > 0 && M > 0 && N > 0 && K > 0 && m_out > 0 && ldw >= K,
                  "token_gemm_f32: bad shape (imgs %d M %d N %d K %d)", imgs, M, N, K);
  TFIMM_CHECK_ARG(glu ? (M % 16 == 0 && m_out <= M / 2) : m_out <= M, "token_gemm_f32: m_out %d does not fit M %d",
                  m_out, M);
  TokenF32Params p{Wt, ldw, X, img_x, ldx, 1, bias, gamma, residual, img_r, ldr, mul, img_mul, ld_mul,
                   out, img_c, ldc, 1, M, N, K, m_out, act, glu};
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM, imgs);
  token_gemm_f32_kernel<<<grid, 256, 0, stream>>>(p);
  TFIMM_LAUNCH_OK("token_gemm_f32_kernel");
  return kOk;
}

// Channel GLU in fp32: out[M][n_out] = (A W_value^T + b) * act(A W_gate^T + b) with W's rows in the SIMT kernel's
// pairing (per 16 rows: 8 value features, then their 8 gates), run as a token GEMM whose "tokens" are A's columns.
int tfimm_b200_gemm_glu_f32(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc,
                            int M, int N, int n_out, int K, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0 && N % 16 == 0 && ldw >= K && n_out > 0 && n_out <= N / 2,
                  "gemm_glu_f32: need N %% 16 == 0 and n_out <= N / 2 (got N %d, n_out %d)", N, n_out);
  TokenF32Params p{W, ldw, A, 0, 1, lda, bias, nullptr, nullptr, 0, 0, nullptr, 0, 0,
                   C, 0, 1, ldc, N, M, K, n_out, act, 1};
  dim3 grid((M + TN - 1) / TN, (N + TM - 1) / TM, 1);
  token_gemm_f32_kernel<<<grid, 256, 0, stream>>>(p);
  TFIMM_LAUNCH_OK("token_gemm_f32_kernel (channel glu)");
  return kOk;
}

int tfimm_b200_affine(const float* x, long ldx, const float* alpha, const float* beta, void* out, int out_dtype,
                      long ldo, long rows, int C, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(rows > 0 && C > 0 && ldx >= C && ldo >= C, "affine: bad shape");
  TFIMM_CHECK_ARG(out_dtype == kBF16 || out_dtype == kF32, "affine: out_dtype must be bf16 or f32");
  const long n = rows * C;
  const int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  if (out_dtype == kBF16)
    affine_kernel<<<blocks, 256, 0, stream>>>(x, ldx, alpha, beta, reinterpret_cast<__nv_bfloat16*>(out), ldo, rows, C);
  else
    affine_kernel<<<blocks, 256, 0, stream>>>(x, ldx, alpha, beta, reinterpret_cast<float*>(out), ldo, rows, C);
  TFIMM_LAUNCH_OK("affine_kernel");
  return kOk;
}

}  // extern "C"
