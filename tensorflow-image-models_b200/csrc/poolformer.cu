// CUDA-core kernels of the PoolFormer family (tfimm/architectures/poolformer.py): the one-group GroupNorm and the
// pooling token mixer.  The 1 x 1-conv MLPs, the stem and the downsamples run on the GEMM paths.
//
// One CTA of 256 threads owns one chunk of 4096 consecutive values of one image (the flattened (h, w, c) order of the
// NHWC tensor), 16 per thread as four float4, so a chunk never splits a float4 across pixels (C % 4 == 0).  The grid
// is (splits, B) for all three kernels, and a chunk's statistics are partials[b][s] = (count, mean, M2):
//   - the chunk mean first, then M2 = sum (v - mean)^2 over the values still in registers.  A one-pass sum and sum of
//     squares would lose every digit of the variance when |mean| >> std; the centred form loses only ~ (mean error)^2.
//   - a consumer merges its image's partials at its start (image_stats): lane l of warp 0 folds s = l, l + 32, ... in
//     order with Chan's formula, then a fixed shfl_down tree folds the lanes.  No atomics anywhere, so every output is
//     bitwise reproducible from run to run.
//
//   gn1_partials_kernel     the partials of a tensor no PoolFormer kernel wrote: one read of the tensor.
//   poolformer_mixer_kernel the token mixer.  Inside one image GN(x) = a_c x + b_c with a_c = rstd gamma_c, and the
//                           "same" 3 x 3 average excludes padded cells, so its weights over the real pixels sum to 1:
//                               pool(GN(x))_i - GN(x)_i = a_c (pool(x)_i - x_i) = a_c mean_{j in N(i)} (x_j - x_i)
//                           (N(i): the in-bounds neighbours, i included).  Beta and the mean cancel, and GN(0) = b_c never
//                           enters: padded cells are skipped in both the sum and the count.  Summing the centred
//                           differences keeps the rounding error proportional to the local variation, not to |x|.
//                           out_i = x_i + ls1_c gamma_c rstd (sum_j (x_j - x_i)) / |N(i)|.  Neighbours are read with
//                           __ldg: the rows above and below belong to the neighbouring chunks, which the CTAs beside this
//                           one are reading at the same time, so they come from L1 / L2 and HBM sees about one read and
//                           one write of the tensor.  The stored values are still in registers, so the kernel also writes
//                           out's partials (norm2's statistics).  out must not alias x: the halo is other CTAs' input.
//   gn1_apply_kernel        y = (x - mean) rstd gamma_c + beta_c, bf16 (the fc1 operand) or fp32 (features_all).
#include "common.cuh"
#include "tfimm_b200_poolformer.h"

namespace tfimm {
namespace {

constexpr int kThreads = 256;
constexpr int kVec = 4;                          // float4 per thread
constexpr int kChunk = kThreads * kVec * 4;      // values per CTA; the host computes splits = ceil(H W C / kChunk)

// Sum over the CTA in a fixed order: a shfl_down tree per warp, then every thread adds the 8 warp totals in order, so
// all threads hold the same value.  `red` may be reused by the next call.
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) t += red[w];
  return t;
}

// Chan's formula: (n, mean, m2) <- (n, mean, m2) merged with (nb, mb, qb).
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float mb, float qb) {
  if (nb == 0.f) return;
  const float nn = n + nb;
  const float d = mb - mean;
  const float f = nb / nn;
  mean = fmaf(d, f, mean);
  m2 = m2 + qb + d * d * n * f;
  n = nn;
}

// (mean, rstd) of one image from its partials; every thread of the CTA gets them.
__device__ __forceinline__ float2 image_stats(const float* __restrict__ part, int splits, float eps, float2* sh) {
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int s = lane; s < splits; s += 32)
      chan_merge(n, mean, m2, __ldg(part + 3 * s), __ldg(part + 3 * s + 1), __ldg(part + 3 * s + 2));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float nb = __shfl_down_sync(0xffffffffu, n, o);
      const float mb = __shfl_down_sync(0xffffffffu, mean, o);
      const float qb = __shfl_down_sync(0xffffffffu, m2, o);
      if (lane + o < 32) chan_merge(n, mean, m2, nb, mb, qb);
    }
    if (lane == 0) *sh = make_float2(mean, rsqrtf(m2 / n + eps));
  }
  __syncthreads();
  return *sh;
}

// Partials of the chunk held in v (ok: the float4 lies inside the image; n: the chunk's value count).
__device__ __forceinline__ void chunk_partials(const float4 (&v)[kVec], const bool (&ok)[kVec], int n, float* red,
                                               float* __restrict__ dst) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i)
    if (ok[i]) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = block_sum(s, red) / (float)n;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    if (!ok[i]) continue;
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += fmaf(a, a, b * b) + fmaf(c, c, d * d);
  }
  const float m2 = block_sum(q, red);
  if (threadIdx.x == 0) {
    dst[0] = (float)n;
    dst[1] = mean;
    dst[2] = m2;
  }
}

__device__ __forceinline__ long elem_of(int s, int i) { return (long)s * kChunk + ((long)i * kThreads + threadIdx.x) * 4; }

__device__ __forceinline__ int chunk_count(int s, long N) {
  const long rest = N - (long)s * kChunk;
  return (int)(rest < kChunk ? rest : kChunk);
}

__global__ void __launch_bounds__(kThreads) gn1_partials_kernel(const float* __restrict__ x, float* __restrict__ part,
                                                                long N, int splits) {
  __shared__ float red[kThreads / 32];
  const int s = blockIdx.x, b = blockIdx.y;
  const float* xb = x + (long)b * N;
  float4 v[kVec];
  bool ok[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const long e = elem_of(s, i);
    ok[i] = e < N;
    v[i] = ok[i] ? __ldg(reinterpret_cast<const float4*>(xb + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  chunk_partials(v, ok, chunk_count(s, N), red, part + ((long)b * splits + s) * 3);
}

__global__ void __launch_bounds__(kThreads) poolformer_mixer_kernel(
    const float* __restrict__ x, const float* __restrict__ part, const float* __restrict__ gamma,
    const float* __restrict__ ls1, float* __restrict__ out, float* __restrict__ out_part, int H, int W, int C,
    int splits, float eps) {
  __shared__ float red[kThreads / 32];
  __shared__ float2 st;
  const int s = blockIdx.x, b = blockIdx.y;
  const long N = (long)H * W * C;
  const float* xb = x + (long)b * N;
  float* ob = out + (long)b * N;
  const float rstd = image_stats(part + (long)b * splits * 3, splits, eps, &st).y;
  const long row = (long)W * C;
  float4 v[kVec];
  bool ok[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const long e = elem_of(s, i);
    ok[i] = e < N;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!ok[i]) continue;
    const long p = e / C;
    const int c = (int)(e - p * C);
    const int h = (int)(p / W), w = (int)(p - (long)h * W);
    const float4 xi = __ldg(reinterpret_cast<const float4*>(xb + e));
    const int h0 = h > 0 ? -1 : 0, h1 = h < H - 1 ? 1 : 0;
    const int w0 = w > 0 ? -1 : 0, w1 = w < W - 1 ? 1 : 0;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        if (dy < h0 || dy > h1 || dx < w0 || dx > w1) continue;
        const float4 xj = __ldg(reinterpret_cast<const float4*>(xb + e + dy * row + (long)dx * C));
        acc.x += xj.x - xi.x;
        acc.y += xj.y - xi.y;
        acc.z += xj.z - xi.z;
        acc.w += xj.w - xi.w;
      }
    }
    const float inv = 1.f / (float)((h1 - h0 + 1) * (w1 - w0 + 1));
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 l = __ldg(reinterpret_cast<const float4*>(ls1 + c));
    v[i].x = fmaf(l.x * g.x * rstd, acc.x * inv, xi.x);
    v[i].y = fmaf(l.y * g.y * rstd, acc.y * inv, xi.y);
    v[i].z = fmaf(l.z * g.z * rstd, acc.z * inv, xi.z);
    v[i].w = fmaf(l.w * g.w * rstd, acc.w * inv, xi.w);
    *reinterpret_cast<float4*>(ob + e) = v[i];
  }
  chunk_partials(v, ok, chunk_count(s, N), red, out_part + ((long)b * splits + s) * 3);
}

template <typename OutT>
__global__ void __launch_bounds__(kThreads) gn1_apply_kernel(const float* __restrict__ x, const float* __restrict__ part,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, OutT* __restrict__ out,
                                                             long N, int C, int splits, float eps) {
  __shared__ float2 st;
  const int s = blockIdx.x, b = blockIdx.y;
  const float2 ms = image_stats(part + (long)b * splits * 3, splits, eps, &st);
  const float* xb = x + (long)b * N;
  OutT* ob = out + (long)b * N;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const long e = elem_of(s, i);
    if (e >= N) continue;
    const int c = (int)(e % C);
    const float4 xv = __ldg(reinterpret_cast<const float4*>(xb + e));
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
    const float y0 = fmaf(xv.x - ms.x, ms.y * g.x, be.x), y1 = fmaf(xv.y - ms.x, ms.y * g.y, be.y);
    const float y2 = fmaf(xv.z - ms.x, ms.y * g.z, be.z), y3 = fmaf(xv.w - ms.x, ms.y * g.w, be.w);
    if constexpr (sizeof(OutT) == 2) {
      *reinterpret_cast<uint2*>(ob + e) = make_uint2(pack_bf16x2(y0, y1), pack_bf16x2(y2, y3));
    } else {
      *reinterpret_cast<float4*>(ob + e) = make_float4(y0, y1, y2, y3);
    }
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

long expected_splits(int H, int W, int C) { return ((long)H * W * C + kChunk - 1) / kChunk; }

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_gn1_partials(const float* x, float* partials, int B, int H, int W, int C, int splits, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0,
                  "gn1_partials: need B, H, W > 0 and C %% 4 == 0 (B=%d H=%d W=%d C=%d)", B, H, W, C);
  TFIMM_CHECK_ARG(splits == expected_splits(H, W, C) && splits <= 65535,
                  "gn1_partials: splits %d, the chunking of H*W*C=%ld gives %ld", splits, (long)H * W * C,
                  expected_splits(H, W, C));
  TFIMM_CHECK_ARG(B <= 65535 && x != nullptr && partials != nullptr && aligned16(x),
                  "gn1_partials: need B <= 65535 and a 16-byte aligned x");
  gn1_partials_kernel<<<dim3(splits, B), kThreads, 0, stream>>>(x, partials, (long)H * W * C, splits);
  TFIMM_LAUNCH_OK("gn1_partials_kernel");
  return kOk;
}

int tfimm_b200_poolformer_mixer(const float* x, const float* partials, const float* gamma, const float* ls1, float* out,
                                float* out_partials, int B, int H, int W, int C, int splits, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0,
                  "poolformer_mixer: need B, H, W > 0 and C %% 4 == 0 (B=%d H=%d W=%d C=%d)", B, H, W, C);
  TFIMM_CHECK_ARG(splits == expected_splits(H, W, C) && splits <= 65535,
                  "poolformer_mixer: splits %d, the chunking of H*W*C=%ld gives %ld", splits, (long)H * W * C,
                  expected_splits(H, W, C));
  TFIMM_CHECK_ARG(B <= 65535 && x != nullptr && partials != nullptr && gamma != nullptr && ls1 != nullptr &&
                      out_partials != nullptr && aligned16(x) && aligned16(out) && aligned16(gamma) && aligned16(ls1),
                  "poolformer_mixer: need B <= 65535 and 16-byte aligned x, out, gamma, ls1");
  TFIMM_CHECK_ARG(out != x && out_partials != partials,
                  "poolformer_mixer: out and out_partials must not alias x and partials");
  poolformer_mixer_kernel<<<dim3(splits, B), kThreads, 0, stream>>>(x, partials, gamma, ls1, out, out_partials, H, W,
                                                                    C, splits, eps);
  TFIMM_LAUNCH_OK("poolformer_mixer_kernel");
  return kOk;
}

int tfimm_b200_gn1_apply(const float* x, const float* partials, const float* gamma, const float* beta, void* out,
                         int out_dtype, int B, int H, int W, int C, int splits, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0,
                  "gn1_apply: need B, H, W > 0 and C %% 4 == 0 (B=%d H=%d W=%d C=%d)", B, H, W, C);
  TFIMM_CHECK_ARG(splits == expected_splits(H, W, C) && splits <= 65535,
                  "gn1_apply: splits %d, the chunking of H*W*C=%ld gives %ld", splits, (long)H * W * C,
                  expected_splits(H, W, C));
  TFIMM_CHECK_ARG(out_dtype == kBF16 || out_dtype == kF32, "gn1_apply: out_dtype must be bf16 or f32");
  TFIMM_CHECK_ARG(B <= 65535 && x != nullptr && partials != nullptr && gamma != nullptr && beta != nullptr &&
                      aligned16(x) && aligned16(gamma) && aligned16(beta) &&
                      (reinterpret_cast<uintptr_t>(out) & (out_dtype == kBF16 ? 7 : 15)) == 0,
                  "gn1_apply: need B <= 65535, 16-byte aligned x, gamma, beta and an aligned out (8 bytes bf16, 16 f32)");
  const long N = (long)H * W * C;
  if (out_dtype == kBF16)
    gn1_apply_kernel<<<dim3(splits, B), kThreads, 0, stream>>>(x, partials, gamma, beta,
                                                               reinterpret_cast<__nv_bfloat16*>(out), N, C, splits, eps);
  else
    gn1_apply_kernel<<<dim3(splits, B), kThreads, 0, stream>>>(x, partials, gamma, beta, reinterpret_cast<float*>(out),
                                                               N, C, splits, eps);
  TFIMM_LAUNCH_OK("gn1_apply_kernel");
  return kOk;
}

}  // extern "C"
