// Data-layout kernels on the edges of the dense contractions (all HBM-bound,
// 128-bit accesses where the geometry allows).
//
//   patchify         NHWC image -> im2col rows of a non-overlapping p x p / stride p conv
//                    (PatchEmbeddings, tfimm/layers/transformers.py:128-139,142-173; ConvNeXt
//                    stem, tfimm/architectures/convnext.py:319-326), optionally fused with
//                    create_preprocessing's (x/255 - mean)/std (tfimm/models/factory.py:153-169).
//   assemble_tokens  prepend cls (and dist) token, add position embedding
//                    (tfimm/architectures/vit.py:427-434).
//   cast             dtype conversion helper.
#include "common.cuh"

namespace tfimm {
namespace {

// out[m, k]: m = (b, gy, gx), k = (ky, kx, c)  (k order == TF conv kernel (kh, kw, cin, :) flattened)
template <typename InT, typename OutT, bool kVec>
__global__ void patchify_kernel(const InT* __restrict__ in, OutT* __restrict__ out, int B, int H, int W,
                                int C, int p, int Kpad, float scale, const float* __restrict__ mean,
                                const float* __restrict__ inv_std) {
  const int gh = H / p, gw = W / p;
  const int K = p * p * C;
  const int chunks = Kpad >> 3;
  const long total = (long)B * gh * gw * chunks;
  const int run = p * C;  // contiguous input elements per (patch, ky)
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % chunks);
    const long m = idx / chunks;
    const int gx = (int)(m % gw);
    const long t = m / gw;
    const int gy = (int)(t % gh);
    const long b = t / gh;
    const int k0 = ch * 8;
    float v[8];
    if (kVec) {
      // run % 8 == 0: the 8 outputs are contiguous in the input
      if (k0 < K) {
        const int ky = k0 / run, r = k0 % run;
        const InT* src = in + ((b * H + (long)gy * p + ky) * W + (long)gx * p) * C + r;
        if constexpr (sizeof(InT) == 1) {
          const uint2 u = *reinterpret_cast<const uint2*>(src);
          v[0] = (float)(u.x & 0xff); v[1] = (float)((u.x >> 8) & 0xff);
          v[2] = (float)((u.x >> 16) & 0xff); v[3] = (float)(u.x >> 24);
          v[4] = (float)(u.y & 0xff); v[5] = (float)((u.y >> 8) & 0xff);
          v[6] = (float)((u.y >> 16) & 0xff); v[7] = (float)(u.y >> 24);
        } else {
          ld8(src, v);
        }
        if (mean != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = (r + j) % C;
            v[j] = (v[j] * scale - mean[c]) * inv_std[c];
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = k0 + j;
        if (k < K) {
          const int ky = k / run, r = k % run;
          const int kx = r / C, c = r % C;
          float x = ld_as_float(in + ((b * H + (long)gy * p + ky) * W + (long)gx * p + kx) * C + c);
          if (mean != nullptr) x = (x * scale - mean[c]) * inv_std[c];
          v[j] = x;
        } else {
          v[j] = 0.f;
        }
      }
    }
    st8(out + m * Kpad + k0, v);
  }
}

template <typename PatchT, typename OutT>
__global__ void assemble_tokens_kernel(const PatchT* __restrict__ patches, const float* __restrict__ cls,
                                       const float* __restrict__ dist, const float* __restrict__ pos,
                                       OutT* __restrict__ out, int B, int P, int ntok, int D) {
  const int T = P + ntok;
  const int chunks = D >> 3;
  const long total = (long)B * T * chunks;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % chunks);
    const long row = idx / chunks;
    const int tk = (int)(row % T);
    const long b = row / T;
    float v[8], pe[8];
    if (tk < ntok) {
      ld8((tk == 0 ? cls : dist) + ch * 8, v);
    } else {
      ld8(patches + (b * P + (tk - ntok)) * (long)D + ch * 8, v);
    }
    ld8(pos + (long)tk * D + ch * 8, pe);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += pe[j];
    st8(out + row * (long)D + ch * 8, v);
  }
}

template <typename InT, typename OutT>
__global__ void cast_kernel(const InT* __restrict__ in, OutT* __restrict__ out, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    st_from_float(out + i, ld_as_float(in + i));
}

inline unsigned grid_for(long total, int threads) {
  long blocks = (total + threads - 1) / threads;
  const long cap = (long)sm_count() * 16;
  return (unsigned)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_patchify(const void* img, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C, int p,
                        int Kpad, float scale, const float* mean, const float* inv_std, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && p > 0 && H % p == 0 && W % p == 0, "patchify: H, W must be multiples of the patch size (H=%d W=%d p=%d)", H, W, p);
  TFIMM_CHECK_ARG(Kpad % 8 == 0 && Kpad >= p * p * C, "patchify: Kpad must be a multiple of 8 and >= p*p*C");
  TFIMM_CHECK_ARG((mean == nullptr) == (inv_std == nullptr), "patchify: mean and inv_std must be given together");
  const long total = (long)B * (H / p) * (W / p) * (Kpad / 8);
  const int threads = 256;
  const unsigned grid = grid_for(total, threads);
  // 8-element groups are contiguous and aligned in the input iff both the per-(patch,ky) run and the
  // image row pitch are multiples of 8 elements.
  const bool vec = ((p * C) % 8 == 0) && (((long)W * C) % 8 == 0) &&
                   ((reinterpret_cast<uintptr_t>(img) & 15u) == 0);
#define TFIMM_PATCHIFY(IN, OUT)                                                                       \
  do {                                                                                                \
    if (vec)                                                                                          \
      patchify_kernel<IN, OUT, true><<<grid, threads, 0, stream>>>(                                   \
          reinterpret_cast<const IN*>(img), reinterpret_cast<OUT*>(out), B, H, W, C, p, Kpad, scale, mean, inv_std); \
    else                                                                                              \
      patchify_kernel<IN, OUT, false><<<grid, threads, 0, stream>>>(                                  \
          reinterpret_cast<const IN*>(img), reinterpret_cast<OUT*>(out), B, H, W, C, p, Kpad, scale, mean, inv_std); \
  } while (0)
  if (in_dtype == kF32 && out_dtype == kBF16) TFIMM_PATCHIFY(float, __nv_bfloat16);
  else if (in_dtype == kF32 && out_dtype == kF32) TFIMM_PATCHIFY(float, float);
  else if (in_dtype == kBF16 && out_dtype == kBF16) TFIMM_PATCHIFY(__nv_bfloat16, __nv_bfloat16);
  else if (in_dtype == kBF16 && out_dtype == kF32) TFIMM_PATCHIFY(__nv_bfloat16, float);
  else if (in_dtype == kU8 && out_dtype == kBF16) TFIMM_PATCHIFY(uint8_t, __nv_bfloat16);
  else if (in_dtype == kU8 && out_dtype == kF32) TFIMM_PATCHIFY(uint8_t, float);
  else {
    set_last_error("patchify: unsupported dtype combination in=%d out=%d", in_dtype, out_dtype);
    return kInvalidArgument;
  }
#undef TFIMM_PATCHIFY
  TFIMM_LAUNCH_OK("patchify_kernel");
  return kOk;
}

int tfimm_b200_assemble_tokens(const void* patches, int patch_dtype, const float* cls, const float* dist,
                               const float* pos, void* out, int out_dtype, int B, int P, int ntok, int D, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && P > 0 && D % 8 == 0 && (ntok == 1 || ntok == 2), "assemble_tokens: bad shape");
  TFIMM_CHECK_ARG(ntok == 1 || dist != nullptr, "assemble_tokens: dist token missing");
  const long total = (long)B * (P + ntok) * (D / 8);
  const int threads = 256;
  const unsigned grid = grid_for(total, threads);
#define TFIMM_ASM(PT, OT)                                                                 \
  assemble_tokens_kernel<PT, OT><<<grid, threads, 0, stream>>>(                           \
      reinterpret_cast<const PT*>(patches), cls, dist, pos, reinterpret_cast<OT*>(out), B, P, ntok, D)
  if (patch_dtype == kBF16 && out_dtype == kF32) TFIMM_ASM(__nv_bfloat16, float);
  else if (patch_dtype == kBF16 && out_dtype == kBF16) TFIMM_ASM(__nv_bfloat16, __nv_bfloat16);
  else if (patch_dtype == kF32 && out_dtype == kF32) TFIMM_ASM(float, float);
  else if (patch_dtype == kF32 && out_dtype == kBF16) TFIMM_ASM(float, __nv_bfloat16);
  else {
    set_last_error("assemble_tokens: unsupported dtype combination");
    return kInvalidArgument;
  }
#undef TFIMM_ASM
  TFIMM_LAUNCH_OK("assemble_tokens_kernel");
  return kOk;
}

int tfimm_b200_cast(const void* in, int in_dtype, void* out, int out_dtype, long n, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(n > 0, "cast: n must be positive");
  const int threads = 256;
  const unsigned grid = grid_for(n, threads);
  if (in_dtype == kF32 && out_dtype == kBF16)
    cast_kernel<<<grid, threads, 0, stream>>>(reinterpret_cast<const float*>(in), reinterpret_cast<__nv_bfloat16*>(out), n);
  else if (in_dtype == kBF16 && out_dtype == kF32)
    cast_kernel<<<grid, threads, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(in), reinterpret_cast<float*>(out), n);
  else if (in_dtype == kU8 && out_dtype == kF32)
    cast_kernel<<<grid, threads, 0, stream>>>(reinterpret_cast<const uint8_t*>(in), reinterpret_cast<float*>(out), n);
  else if (in_dtype == kU8 && out_dtype == kBF16)
    cast_kernel<<<grid, threads, 0, stream>>>(reinterpret_cast<const uint8_t*>(in), reinterpret_cast<__nv_bfloat16*>(out), n);
  else {
    set_last_error("cast: unsupported dtype combination in=%d out=%d", in_dtype, out_dtype);
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("cast_kernel");
  return kOk;
}

}  // extern "C"
