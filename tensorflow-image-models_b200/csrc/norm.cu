// Row-wise LayerNorm kernels (HBM-bound; one warp per row, 128-bit loads,
// warp-shuffle reductions, statistics in fp32).
//
// Replaces tf.keras.layers.LayerNormalization as configured by
// tfimm/layers/factory.py:37-45 ("layer_norm" eps 1e-5, "layer_norm_eps_1e-6"):
//   y = (x - mean) * rsqrt(var + eps) * gamma + beta, biased variance over the last axis.
//
// Variants:
//   layernorm_rows        plain rows -> rows (optional input row stride, e.g. only the
//                         cls token of every image: tfimm/architectures/vit.py:452,462)
//   layernorm_patch2x2    LN per pixel, output written straight into the im2col layout
//                         of the following 2x2/stride-2 conv (ConvNeXt downsample,
//                         tfimm/architectures/convnext.py:257-266, 286-295)
//   patch_merge_ln        Swin PatchMerging gather (order (0,0),(1,0),(0,1),(1,1)) +
//                         LN over 4C (tfimm/architectures/swin.py:348-362)
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kWarpsPerBlock = 8;

// Each lane owns chunks of 8 channels: chunk index = lane + 32 * i, i < MAXI.
template <typename InT, typename OutT, int MAXI, typename RowMap>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
layernorm_kernel(const float* __restrict__ gamma, const float* __restrict__ beta, long rows, int C,
                 float eps, RowMap map) {
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = C >> 3;
  float v[MAXI][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int ch = lane + 32 * i;
    if (ch < nchunks) {
      ld8(map.template src<InT>(row, ch * 8), v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[i][j];
    }
  }
  const float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int ch = lane + 32 * i;
    if (ch < nchunks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int ch = lane + 32 * i;
    if (ch < nchunks) {
      float g[8], b[8], o[8];
      ld8(gamma + ch * 8, g);
      ld8(beta + ch * 8, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      st8(map.template dst<OutT>(row, ch * 8), o);
    }
  }
}

// Plain fp32 rows (the residual stream of ViT / Swin / ConvNeXt): 16-byte accesses with lane = chunk of FOUR channels,
// so every load instruction covers 512 contiguous bytes of the row (the generic kernel's 8-channel chunks make each
// fp32 load touch only half of every sector, and leave half the warp idle at C = 128), and ROWS rows per warp in flight
// for the narrow rows of the early Swin / ConvNeXt stages.
template <typename OutT, int MAXI, int ROWS>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
layernorm_f32_rows_kernel(const float* __restrict__ x, long in_stride, const float* __restrict__ gamma,
                          const float* __restrict__ beta, OutT* __restrict__ out, long out_stride, long rows, int C,
                          float eps) {
  const int lane = threadIdx.x & 31;
  const long row0 = ((long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5)) * ROWS;
  if (row0 >= rows) return;
  const int nchunks = C >> 2;
  const float inv_c = 1.0f / (float)C;
  float4 v[ROWS][MAXI];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const bool row_ok = row0 + r < rows;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      const int ch = lane + 32 * i;
      v[r][i] = (row_ok && ch < nchunks) ? *reinterpret_cast<const float4*>(x + (row0 + r) * in_stride + ch * 4)
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float mean[ROWS], rstd[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) s += (v[r][i].x + v[r][i].y) + (v[r][i].z + v[r][i].w);
    mean[r] = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXI; ++i) {
      if (lane + 32 * i < nchunks) {
        const float a = v[r][i].x - mean[r], b = v[r][i].y - mean[r], c = v[r][i].z - mean[r], d = v[r][i].w - mean[r];
        q += (a * a + b * b) + (c * c + d * d);
      }
    }
    rstd[r] = rsqrtf(warp_sum(q) * inv_c + eps);
  }
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int ch = lane + 32 * i;
    if (ch < nchunks) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + ch * 4));
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta + ch * 4));
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        if (row0 + r < rows) {
          const float y0 = (v[r][i].x - mean[r]) * rstd[r] * g.x + b.x, y1 = (v[r][i].y - mean[r]) * rstd[r] * g.y + b.y;
          const float y2 = (v[r][i].z - mean[r]) * rstd[r] * g.z + b.z, y3 = (v[r][i].w - mean[r]) * rstd[r] * g.w + b.w;
          OutT* dst = out + (row0 + r) * out_stride + ch * 4;
          if constexpr (sizeof(OutT) == 2) {
            *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(y0, y1), pack_bf16x2(y2, y3));
          } else {
            *reinterpret_cast<float4*>(dst) = make_float4(y0, y1, y2, y3);
          }
        }
      }
    }
  }
}

template <typename OutT>
int launch_ln_f32_rows(const float* x, long in_stride, const float* gamma, const float* beta, OutT* out,
                       long out_stride, long rows, int C, float eps, cudaStream_t stream) {
  const int maxi = (C / 4 + 31) / 32;
  const int threads = kWarpsPerBlock * 32;
#define TFIMM_LNR(I, R)                                                                                            \
  do {                                                                                                             \
    const long warps = (rows + R - 1) / R;                                                                         \
    layernorm_f32_rows_kernel<OutT, I, R><<<(unsigned)((warps + kWarpsPerBlock - 1) / kWarpsPerBlock), threads, 0, \
                                            stream>>>(x, in_stride, gamma, beta, out, out_stride, rows, C, eps);   \
  } while (0)
  if (maxi <= 1) TFIMM_LNR(1, 4);
  else if (maxi <= 2) TFIMM_LNR(2, 2);
  else if (maxi <= 4) TFIMM_LNR(4, 1);
  else if (maxi <= 6) TFIMM_LNR(6, 1);
  else if (maxi <= 8) TFIMM_LNR(8, 1);
  else if (maxi <= 16) TFIMM_LNR(16, 1);
  else if (maxi <= 32) TFIMM_LNR(32, 1);
  else {
    set_last_error("layernorm: C=%d too large (max 4096)", C);
    return kUnsupported;
  }
#undef TFIMM_LNR
  TFIMM_LAUNCH_OK("layernorm_f32_rows_kernel");
  return kOk;
}

struct PlainRows {
  const void* in;
  void* out;
  long in_stride, out_stride;  // elements
  template <typename T>
  __device__ const T* src(long row, int c) const {
    return reinterpret_cast<const T*>(in) + row * in_stride + c;
  }
  template <typename T>
  __device__ T* dst(long row, int c) const {
    return reinterpret_cast<T*>(out) + row * out_stride + c;
  }
};

// rows index pixels (b, y, x) of an NHWC map; destination row = (b, y/2, x/2),
// destination column = ((y%2)*2 + (x%2))*C + c  == im2col of a 2x2 stride-2 conv
// with kernel flattened as (kh, kw, cin).
struct Patch2x2Rows {
  const void* in;
  void* out;
  int H, W, C;
  template <typename T>
  __device__ const T* src(long row, int c) const {
    return reinterpret_cast<const T*>(in) + row * C + c;
  }
  template <typename T>
  __device__ T* dst(long row, int c) const {
    const int x = (int)(row % W);
    const long t = row / W;
    const int y = (int)(t % H);
    const long b = t / H;
    const long orow = (b * (H / 2) + (y >> 1)) * (W / 2) + (x >> 1);
    const int ocol = (((y & 1) << 1) + (x & 1)) * C + c;
    return reinterpret_cast<T*>(out) + orow * (4L * C) + ocol;
  }
};

// rows index merged tokens (b, y2, x2); channel c4 in [0, 4C) comes from source pixel
// (2*y2 + dy, 2*x2 + dx) with (dy, dx) = (0,0),(1,0),(0,1),(1,1) for c4 / C = 0,1,2,3.
struct PatchMergeRows {
  const void* in;
  void* out;
  int H, W, C;  // source map dims
  template <typename T>
  __device__ const T* src(long row, int c4) const {
    const int W2 = W / 2, H2 = H / 2;
    const int x2 = (int)(row % W2);
    const long t = row / W2;
    const int y2 = (int)(t % H2);
    const long b = t / H2;
    const int g = c4 / C, c = c4 % C;
    const int dy = g & 1, dx = g >> 1;
    return reinterpret_cast<const T*>(in) + ((b * H + (2 * y2 + dy)) * W + (2 * x2 + dx)) * (long)C + c;
  }
  template <typename T>
  __device__ T* dst(long row, int c4) const {
    return reinterpret_cast<T*>(out) + row * (4L * C) + c4;
  }
};

template <typename InT, typename OutT, typename RowMap>
int launch_ln(const float* gamma, const float* beta, long rows, int C, float eps, RowMap map,
              cudaStream_t stream) {
  const int maxi = (C / 8 + 31) / 32;
  const unsigned grid = (unsigned)((rows + kWarpsPerBlock - 1) / kWarpsPerBlock);
  const int threads = kWarpsPerBlock * 32;
#define TFIMM_LN_CASE(I)                                                                         \
  layernorm_kernel<InT, OutT, I, RowMap><<<grid, threads, 0, stream>>>(gamma, beta, rows, C, eps, map)
  if (maxi <= 1) TFIMM_LN_CASE(1);
  else if (maxi <= 2) TFIMM_LN_CASE(2);
  else if (maxi <= 4) TFIMM_LN_CASE(4);
  else if (maxi <= 8) TFIMM_LN_CASE(8);
  else if (maxi <= 16) TFIMM_LN_CASE(16);
  else {
    set_last_error("layernorm: C=%d too large (max 4096)", C);
    return kUnsupported;
  }
#undef TFIMM_LN_CASE
  TFIMM_LAUNCH_OK("layernorm_kernel");
  return kOk;
}

template <typename RowMap>
int dispatch_ln(int in_dtype, int out_dtype, const float* gamma, const float* beta, long rows, int C,
                float eps, RowMap map, cudaStream_t stream) {
  if (in_dtype == kF32 && out_dtype == kBF16)
    return launch_ln<float, __nv_bfloat16>(gamma, beta, rows, C, eps, map, stream);
  if (in_dtype == kBF16 && out_dtype == kBF16)
    return launch_ln<__nv_bfloat16, __nv_bfloat16>(gamma, beta, rows, C, eps, map, stream);
  if (in_dtype == kF32 && out_dtype == kF32)
    return launch_ln<float, float>(gamma, beta, rows, C, eps, map, stream);
  if (in_dtype == kBF16 && out_dtype == kF32)
    return launch_ln<__nv_bfloat16, float>(gamma, beta, rows, C, eps, map, stream);
  set_last_error("layernorm: unsupported dtype combination in=%d out=%d", in_dtype, out_dtype);
  return kInvalidArgument;
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_layernorm(const void* x, int in_dtype, long in_stride, const float* gamma, const float* beta, void* out,
                         int out_dtype, long out_stride, long rows, int C, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0, "layernorm: need rows>0 and C%%8==0 (rows=%ld C=%d)", rows, C);
  TFIMM_CHECK_ARG(in_stride % 8 == 0 && out_stride % 8 == 0, "layernorm: strides must be multiples of 8 elements");
  if (in_dtype == kF32 && C % 4 == 0 && in_stride % 4 == 0 && out_stride % 4 == 0 &&
      (reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
      (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15u) == 0) {
    if (out_dtype == kBF16)
      return launch_ln_f32_rows(reinterpret_cast<const float*>(x), in_stride, gamma, beta,
                                reinterpret_cast<__nv_bfloat16*>(out), out_stride, rows, C, eps, stream);
    if (out_dtype == kF32)
      return launch_ln_f32_rows(reinterpret_cast<const float*>(x), in_stride, gamma, beta, reinterpret_cast<float*>(out),
                                out_stride, rows, C, eps, stream);
  }
  PlainRows map{x, out, in_stride, out_stride};
  return dispatch_ln(in_dtype, out_dtype, gamma, beta, rows, C, eps, map, stream);
}

int tfimm_b200_layernorm_patch2x2(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                                  int out_dtype, int B, int H, int W, int C, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0,
                  "layernorm_patch2x2: need even H, W and C%%8==0 (H=%d W=%d C=%d)", H, W, C);
  Patch2x2Rows map{x, out, H, W, C};
  return dispatch_ln(in_dtype, out_dtype, gamma, beta, (long)B * H * W, C, eps, map, stream);
}

int tfimm_b200_patch_merge_ln(const void* x, int in_dtype, const float* gamma, const float* beta, void* out,
                              int out_dtype, int B, int H, int W, int C, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0,
                  "patch_merge_ln: need even H, W and C%%8==0 (H=%d W=%d C=%d)", H, W, C);
  PatchMergeRows map{x, out, H, W, C};
  return dispatch_ln(in_dtype, out_dtype, gamma, beta, (long)B * (H / 2) * (W / 2), 4 * C, eps, map, stream);
}

}  // extern "C"
