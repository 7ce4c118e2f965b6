// fp32 SIMT GEMM with the same fused epilogue as the tensor-core kernel:
//     C = residual + gamma * act(A @ W^T + bias)       A:[M,K]  W:[N,K]  (fp32, K contiguous)
// Used only by precision="fp32" (the 1e-5 structural-parity mode of the engine);
// the performance path is gemm_sm90.cu.  64x64 tiles, 4x4 micro-tiles, BK = 16.
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int TM = 64, TN = 64, TK = 16;

__global__ void __launch_bounds__(256)
gemm_f32_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W, int ldw,
                const float* __restrict__ bias, const float* __restrict__ gamma,
                const float* __restrict__ residual, int ldr, float* __restrict__ C, int ldc, int M, int N,
                int K, int act, int act_post) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Ws[TK][TN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  float acc[4][4] = {};
  // loader mapping: 256 threads x 4 floats = 64 rows x 16 k
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  for (int k0 = 0; k0 < K; k0 += TK) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), w = a;
    if (m0 + lr < M && k0 + lk < K) a = *reinterpret_cast<const float4*>(A + (long)(m0 + lr) * lda + k0 + lk);
    if (n0 + lr < N && k0 + lk < K) w = *reinterpret_cast<const float4*>(W + (long)(n0 + lr) * ldw + k0 + lk);
    As[lk + 0][lr] = a.x; As[lk + 1][lr] = a.y; As[lk + 2][lr] = a.z; As[lk + 3][lr] = a.w;
    Ws[lk + 0][lr] = w.x; Ws[lk + 1][lr] = w.y; Ws[lk + 2][lr] = w.z; Ws[lk + 3][lr] = w.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float av[4], wv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) wv[j] = Ws[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (bias != nullptr) v += bias[n];
      if (!act_post) v = apply_act<true>(v, act);
      if (gamma != nullptr) v *= gamma[n];
      if (residual != nullptr) v += residual[(long)m * ldr + n];
      if (act_post) v = apply_act<true>(v, act);
      C[(long)m * ldc + n] = v;
    }
  }
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_gemm_f32(const float* A, int lda, const float* W, int ldw, const float* bias, const float* gamma,
                        const float* residual, int ldr, float* C, int ldc, int M, int N, int K, int act, int act_post,
                        void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm_f32: M, N, K must be positive");
  TFIMM_CHECK_ARG(K % 4 == 0 && lda % 4 == 0 && ldw % 4 == 0, "gemm_f32: K, lda, ldw must be multiples of 4");
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15u) == 0 && (reinterpret_cast<uintptr_t>(W) & 15u) == 0,
                  "gemm_f32: A and W must be 16-byte aligned");
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM);
  gemm_f32_kernel<<<grid, 256, 0, stream>>>(A, lda, W, ldw, bias, gamma, residual, ldr, C, ldc, M, N, K, act, act_post);
  TFIMM_LAUNCH_OK("gemm_f32_kernel");
  return kOk;
}

}  // extern "C"
