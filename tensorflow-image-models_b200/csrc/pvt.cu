// Kernels of the PVT family (tfimm/architectures/pvt.py): spatial-reduction attention, whose keys and values come from
// a second, shorter sequence than the queries, in bf16 on the tensor cores and in fp32 on the CUDA cores; and the end of
// each stage's patch embedding (LayerNorm, position table, class row).  The blocks' LayerNorms and GEMMs, the patch and
// spatial-reduction convolutions (im2col + GEMM) run on the existing paths.
//
// pvt_sr_attention_bf16_kernel<64> / pvt_sr_attention_f32_kernel<64>  spatial-reduction attention at head dim 64, on
//   the tensor cores and on the CUDA cores (pvt_sr_attention.cuh, shared with the head-dim-32 instances of pvt_v2.cu).
// pvt_embed_norm_kernel  out[b, ntok + p] = LayerNorm_eps(tok[b, p]) gamma + beta + pos[ntok + p] and, when ntok = 1,
//   out[b, 0] = cls + pos[0]: the fp32 residual stream of a stage.  The LayerNorm is layernorm_f32_rows_kernel's
//   (norm.cu, one row per warp) with the position row added after it.
#include "common.cuh"
#include "pvt_sr_attention.cuh"
#include "tfimm_b200_pvt.h"

namespace tfimm {
namespace {

constexpr int kDH = 64;
using Sra = PvtSra<kDH>;

constexpr int kNormWarps = 8;

// Lane = chunk of four channels (chunk lane + 32 i, i < MAXI), one row per warp.
template <int MAXI>
__global__ void __launch_bounds__(kNormWarps * 32)
pvt_embed_norm_kernel(const float* __restrict__ tok, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ pos, const float* __restrict__ cls, float* __restrict__ out, long rows,
                      int T, int ntok, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * kNormWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = C >> 2;
  const long b = row / T;
  const int i = (int)(row - b * T);
  float4* dst = reinterpret_cast<float4*>(out + row * C);
  const float4* pr = reinterpret_cast<const float4*>(pos + (long)i * C);
  if (i < ntok) {   // the class row
    for (int ch = lane; ch < nchunks; ch += 32) {
      const float4 c = __ldg(reinterpret_cast<const float4*>(cls) + ch), p = __ldg(pr + ch);
      dst[ch] = make_float4(c.x + p.x, c.y + p.y, c.z + p.z, c.w + p.w);
    }
    return;
  }
  const float* x = tok + (b * (T - ntok) + (i - ntok)) * C;
  const float inv_c = 1.0f / (float)C;
  float4 v[MAXI];
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    const int ch = lane + 32 * k;
    v[k] = ch < nchunks ? *reinterpret_cast<const float4*>(x + ch * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXI; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
  const float mean = warp_sum(s) * inv_c;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    if (lane + 32 * k < nchunks) {
      const float a = v[k].x - mean, bb = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
      sq += (a * a + bb * bb) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) * inv_c + eps);
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    const int ch = lane + 32 * k;
    if (ch < nchunks) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + ch);
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta) + ch);
      const float4 p = __ldg(pr + ch);
      const float y0 = (v[k].x - mean) * rstd * g.x + be.x, y1 = (v[k].y - mean) * rstd * g.y + be.y;
      const float y2 = (v[k].z - mean) * rstd * g.z + be.z, y3 = (v[k].w - mean) * rstd * g.w + be.w;
      dst[ch] = make_float4(y0 + p.x, y1 + p.y, y2 + p.z, y3 + p.w);
    }
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_pvt_sr_attention_bf16(const void* q, const void* kv, void* out, int B, int N, int Nk, int H, int dh,
                                     float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_sr_attention_bf16: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_sr_attention_bf16: head_dim must be 64 (got %d)", dh);
  TFIMM_CHECK_ARG(B <= 65535 && H <= 65535, "pvt_sr_attention_bf16: need B, H <= 65535 (B=%d H=%d)", B, H);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_sr_attention_bf16: q, kv and out must be 16-byte aligned");
  auto kernel = pvt_sr_attention_bf16_kernel<kDH>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Sra::kSmem, attr_devs));
  const int ntiles = (N + Sra::kRows - 1) / Sra::kRows;
  const int tiles = pvt_tiles_per_cta<kDH>(ntiles, (Nk + Sra::kKeys - 1) / Sra::kKeys, B, H);
  const dim3 grid((ntiles + tiles - 1) / tiles, H, B);
  kernel<<<grid, Sra::kWarps * 32, Sra::kSmem, stream>>>(reinterpret_cast<const __nv_bfloat16*>(q),
                                               reinterpret_cast<const __nv_bfloat16*>(kv),
                                               reinterpret_cast<__nv_bfloat16*>(out), N, Nk, H, tiles,
                                               scale * kLog2e);
  TFIMM_LAUNCH_OK("pvt_sr_attention_bf16_kernel");
  return kOk;
}

int tfimm_b200_pvt_sr_attention_f32(const float* q, const float* kv, float* out, int B, int N, int Nk, int H, int dh,
                                    float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_sr_attention_f32: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_sr_attention_f32: head_dim must be 64 (got %d)", dh);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_sr_attention_f32: q, kv and out must be 16-byte aligned");
  const long rows = (long)B * H * N;
  const long blocks = (rows + kF32Warps - 1) / kF32Warps;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pvt_sr_attention_f32: problem too large (%ld blocks)", blocks);
  pvt_sr_attention_f32_kernel<kDH><<<(unsigned)blocks, kF32Warps * 32, 0, stream>>>(q, kv, out, rows, N, Nk, H, scale);
  TFIMM_LAUNCH_OK("pvt_sr_attention_f32_kernel");
  return kOk;
}

int tfimm_b200_pvt_embed_norm(const float* tok, const float* gamma, const float* beta, const float* pos,
                              const float* cls, float* out, int B, int P, int ntok, int C, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && P > 0 && (ntok == 0 || ntok == 1) && C > 0 && C % 4 == 0 && C <= 1024,
                  "pvt_embed_norm: need B, P > 0, ntok 0 or 1, C %% 4 == 0 and C <= 1024 (B=%d P=%d ntok=%d C=%d)", B,
                  P, ntok, C);
  TFIMM_CHECK_ARG(tok != nullptr && gamma != nullptr && beta != nullptr && pos != nullptr && out != nullptr &&
                      aligned(tok, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(pos, 16) &&
                      aligned(out, 16),
                  "pvt_embed_norm: tok, gamma, beta, pos and out must be 16-byte aligned");
  TFIMM_CHECK_ARG(ntok == 0 || (cls != nullptr && aligned(cls, 16)),
                  "pvt_embed_norm: ntok = 1 needs a 16-byte aligned cls");
  const int T = P + ntok;
  const long rows = (long)B * T;
  const long blocks = (rows + kNormWarps - 1) / kNormWarps;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pvt_embed_norm: problem too large (%ld blocks)", blocks);
  const int maxi = (C / 4 + 31) / 32;
#define TFIMM_PEN(I)                                                                                                 \
  pvt_embed_norm_kernel<I><<<(unsigned)blocks, kNormWarps * 32, 0, stream>>>(tok, gamma, beta, pos, cls, out, rows, \
                                                                             T, ntok, C, eps)
  if (maxi <= 1) TFIMM_PEN(1);
  else if (maxi <= 2) TFIMM_PEN(2);
  else if (maxi <= 4) TFIMM_PEN(4);
  else TFIMM_PEN(8);
#undef TFIMM_PEN
  TFIMM_LAUNCH_OK("pvt_embed_norm_kernel");
  return kOk;
}

}  // extern "C"
