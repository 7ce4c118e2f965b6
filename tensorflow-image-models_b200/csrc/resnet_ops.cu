// CUDA-core kernels specific to the ResNet family (tfimm/architectures/resnet.py):
//   grouped_conv        Conv2D(k x k, groups = cardinality) of ResNeXt bottlenecks (resnet.py:230-238):
//                       4..32 input channels per group is far too thin for a tensor-core tile, so each
//                       thread produces one pixel's outputs of one group from registers.
//   eca_gate            EcaModule (tfimm/layers/attention.py:120-130): mean -> Conv1D over the channel
//                       axis (zero padded) -> sigmoid.
//   scale_add_act       x = act(x * gate + shortcut): tail of SE / ECA residual blocks
//                       (resnet.py:182-188, 284-291).
#include "common.cuh"

namespace tfimm {
namespace {

// wgt: [ks*ks][CG_IN][Cout] fp32 == TF grouped kernel (kh, kw, Cin/groups, Cout); bias folded BN.
// One thread: one output pixel x one group (CG_OUT outputs).  Requires CG_IN == CG_OUT == CG.
template <typename T, int CG>
__global__ void grouped_conv_kernel(const T* __restrict__ x, const float* __restrict__ wgt,
                                    const float* __restrict__ bias, T* __restrict__ out, int B, int H, int W,
                                    int C, int Ho, int Wo, int ks, int stride, int pad, int act) {
  const int groups = C / CG;
  const long total = (long)B * Ho * Wo * groups;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    const long m = idx / groups;
    const int ox = (int)(m % Wo);
    const long t = m / Wo;
    const int oy = (int)(t % Ho);
    const long b = t / Ho;
    float acc[CG];
#pragma unroll
    for (int o = 0; o < CG; ++o) acc[o] = bias != nullptr ? bias[g * CG + o] : 0.f;
    for (int ky = 0; ky < ks; ++ky) {
      const int iy = oy * stride + ky - pad;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < ks; ++kx) {
        const int ix = ox * stride + kx - pad;
        if (ix < 0 || ix >= W) continue;
        const T* px = x + ((b * H + iy) * W + ix) * (long)C + g * CG;
        const float* wp = wgt + ((long)(ky * ks + kx) * CG) * C + g * CG;
        float in[CG];
#pragma unroll
        for (int i = 0; i < CG; ++i) in[i] = ld_as_float(px + i);
#pragma unroll
        for (int i = 0; i < CG; ++i) {
#pragma unroll
          for (int o = 0; o < CG; ++o) acc[o] = fmaf(in[i], __ldg(wp + (long)i * C + o), acc[o]);
        }
      }
    }
    T* po = out + m * C + g * CG;
#pragma unroll
    for (int o = 0; o < CG; ++o) st_from_float(po + o, apply_act<true>(acc[o], act));
  }
}

__global__ void eca_gate_kernel(const float* __restrict__ mean, const float* __restrict__ w, float* __restrict__ gate,
                                int B, int C, int ks) {
  const int pad = (ks - 1) / 2;
  const long total = (long)B * C;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long b = idx / C;
    float acc = 0.f;
    for (int j = 0; j < ks; ++j) {
      const int cc = c + j - pad;
      if (cc >= 0 && cc < C) acc = fmaf(w[j], mean[b * C + cc], acc);
    }
    gate[idx] = 1.0f / (1.0f + expf(-acc));
  }
}

template <typename T>
__global__ void scale_add_act_kernel(T* __restrict__ x, const float* __restrict__ gate, const T* __restrict__ shortcut,
                                     long total_chunks, int HW, int C, int act) {
  const int cpr = C >> 3;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total_chunks;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % cpr);
    const long row = idx / cpr;
    const long b = row / HW;
    float v[8], g[8], s[8];
    ld8(x + row * C + ch * 8, v);
    ld8(gate + b * C + ch * 8, g);
    ld8(shortcut + row * C + ch * 8, s);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = apply_act<true>(fmaf(v[j], g[j], s[j]), act);
    st8(x + row * C + ch * 8, v);
  }
}

inline unsigned rgrid(long total, int threads) {
  long blocks = (total + threads - 1) / threads;
  const long cap = (long)sm_count() * 32;
  return (unsigned)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// ---- GroupNormalization (tfimm/layers/norm.py:22-101), NHWC, groups of C/G consecutive channels --------------
// Pass 1: one CTA per (image, group): mean and rstd over HW x (C/G) values (two sweeps: mean, then centred
// second moment -- the second sweep hits L2).  Pass 2: elementwise normalise + per-channel affine (+ residual,
// activation).  Only resnet50_gn uses it, so the kernels favour simplicity over the last GB/s.
template <typename T>
__global__ void __launch_bounds__(256)
group_norm_stats_kernel(const T* __restrict__ x, float* __restrict__ stats /*[B][G][2]*/, int HW, int C, int G,
                        float eps) {
  const int b = blockIdx.x / G, g = blockIdx.x % G;
  const int cg = C / G;
  const T* base = x + (long)b * HW * C + g * cg;
  const long n = (long)HW * cg;
  __shared__ float red[8];
  __shared__ float s_mean;
  auto block_sum = [&](float v) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    return t;
  };
  float s = 0.f;
  for (long i = threadIdx.x; i < n; i += 256) s += ld_as_float(base + (i / cg) * C + (i % cg));
  const float mean = block_sum(s) / (float)n;
  float q = 0.f;
  for (long i = threadIdx.x; i < n; i += 256) {
    const float d = ld_as_float(base + (i / cg) * C + (i % cg)) - mean;
    q = fmaf(d, d, q);
  }
  const float var = block_sum(q) / (float)n;
  if (threadIdx.x == 0) {
    stats[(long)blockIdx.x * 2] = mean;
    stats[(long)blockIdx.x * 2 + 1] = rsqrtf(var + eps);
  }
}

template <typename T>
__global__ void group_norm_apply_kernel(const T* __restrict__ x, const float* __restrict__ stats,
                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                        const T* __restrict__ residual, T* __restrict__ out, long total, int HW, int C,
                                        int G, int act) {
  const int cg = C / G;
  const int chunks = C >> 3;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % chunks) * 8;
    const long pix = idx / chunks;
    const long b = pix / HW;
    float v[8], r[8];
    ld8(x + pix * C + c0, v);
    if (residual != nullptr) ld8(residual + pix * C + c0, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      const float* st = stats + (b * G + c / cg) * 2;
      float y = (v[j] - st[0]) * st[1] * __ldg(gamma + c) + __ldg(beta + c);
      if (residual != nullptr) y += r[j];
      v[j] = apply_act<true>(y, act);
    }
    st8(out + pix * C + c0, v);
  }
}

// ---- BlurPool2D (tfimm/layers/blurpool.py:54-62): REFLECT pad 1, 3x3 [1 2 1]x[1 2 1]/16, stride s ------------
template <typename T>
__global__ void blur_pool_kernel(const T* __restrict__ x, T* __restrict__ out, long total, int H, int W, int C, int Ho,
                                 int Wo, int stride) {
  const int chunks = C >> 3;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c0 = (int)(idx % chunks) * 8;
    long t = idx / chunks;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const long b = t / Ho;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      int iy = oy * stride + ky - 1;
      iy = iy < 0 ? -iy : (iy >= H ? 2 * H - 2 - iy : iy);  // REFLECT (no edge repeat)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        int ix = ox * stride + kx - 1;
        ix = ix < 0 ? -ix : (ix >= W ? 2 * W - 2 - ix : ix);
        const float wgt = (float)((ky == 1 ? 2 : 1) * (kx == 1 ? 2 : 1)) * (1.0f / 16.0f);
        float v[8];
        ld8(x + ((b * H + iy) * W + ix) * (long)C + c0, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(wgt, v[j], acc[j]);
      }
    }
    st8(out + ((b * Ho + oy) * Wo + ox) * (long)C + c0, acc);
  }
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_grouped_conv(const void* x, int dtype, const float* wgt, const float* bias, void* out, int B, int H,
                            int W, int C, int cg, int ks, int stride, int pad, int Ho, int Wo, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && C > 0 && cg > 0 && C % cg == 0, "grouped_conv: bad channel grouping (C=%d cg=%d)", C, cg);
  TFIMM_CHECK_ARG(dtype == kBF16 || dtype == kF32, "grouped_conv: dtype must be bf16 or f32");
  const long total = (long)B * Ho * Wo * (C / cg);
  const unsigned grid = rgrid(total, 128);
#define TFIMM_GC(T, CG)                                                                                   \
  grouped_conv_kernel<T, CG><<<grid, 128, 0, stream>>>(reinterpret_cast<const T*>(x), wgt, bias,           \
                                                       reinterpret_cast<T*>(out), B, H, W, C, Ho, Wo, ks, \
                                                       stride, pad, act)
#define TFIMM_GC_T(T)                          \
  do {                                         \
    if (cg == 4) TFIMM_GC(T, 4);               \
    else if (cg == 8) TFIMM_GC(T, 8);          \
    else if (cg == 16) TFIMM_GC(T, 16);        \
    else if (cg == 32) TFIMM_GC(T, 32);        \
    else {                                     \
      set_last_error("grouped_conv: channels per group must be 4, 8, 16 or 32 (got %d)", cg); \
      return kUnsupported;                     \
    }                                          \
  } while (0)
  if (dtype == kBF16) TFIMM_GC_T(__nv_bfloat16);
  else TFIMM_GC_T(float);
#undef TFIMM_GC_T
#undef TFIMM_GC
  TFIMM_LAUNCH_OK("grouped_conv_kernel");
  return kOk;
}

int tfimm_b200_eca_gate(const float* mean, const float* w, float* gate, int B, int C, int ks, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && C > 0 && ks > 0 && (ks & 1), "eca_gate: need an odd kernel size");
  eca_gate_kernel<<<rgrid((long)B * C, 256), 256, 0, stream>>>(mean, w, gate, B, C, ks);
  TFIMM_LAUNCH_OK("eca_gate_kernel");
  return kOk;
}

int tfimm_b200_scale_add_act(void* x, int dtype, const float* gate, const void* shortcut, int B, int HW, int C, int act,
                             void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && HW > 0 && C % 8 == 0, "scale_add_act: need C%%8==0 (C=%d)", C);
  const long total = (long)B * HW * (C / 8);
  if (dtype == kBF16)
    scale_add_act_kernel<<<rgrid(total, 256), 256, 0, stream>>>(
        reinterpret_cast<__nv_bfloat16*>(x), gate, reinterpret_cast<const __nv_bfloat16*>(shortcut), total, HW, C, act);
  else if (dtype == kF32)
    scale_add_act_kernel<<<rgrid(total, 256), 256, 0, stream>>>(reinterpret_cast<float*>(x), gate,
                                                               reinterpret_cast<const float*>(shortcut), total, HW, C, act);
  else {
    set_last_error("scale_add_act: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("scale_add_act_kernel");
  return kOk;
}

int tfimm_b200_group_norm(const void* x, int dtype, const float* gamma, const float* beta, const void* residual,
                          void* out, float* stats, int B, int HW, int C, int groups, float eps, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && HW > 0 && groups > 0 && C % groups == 0 && C % 8 == 0,
                  "group_norm: need C%%groups==0 and C%%8==0 (C=%d groups=%d)", C, groups);
  const long total = (long)B * HW * (C / 8);
#define TFIMM_GN(T)                                                                                               \
  group_norm_stats_kernel<T><<<B * groups, 256, 0, stream>>>(reinterpret_cast<const T*>(x), stats, HW, C, groups, eps); \
  group_norm_apply_kernel<T><<<rgrid(total, 256), 256, 0, stream>>>(                                              \
      reinterpret_cast<const T*>(x), stats, gamma, beta, reinterpret_cast<const T*>(residual),                      \
      reinterpret_cast<T*>(out), total, HW, C, groups, act)
  if (dtype == kBF16) { TFIMM_GN(__nv_bfloat16); }
  else if (dtype == kF32) { TFIMM_GN(float); }
  else {
    set_last_error("group_norm: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
#undef TFIMM_GN
  TFIMM_LAUNCH_OK("group_norm kernels");
  return kOk;
}

int tfimm_b200_blur_pool(const void* x, int dtype, void* out, int B, int H, int W, int C, int stride, int Ho, int Wo,
                         void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 1 && W > 1 && C % 8 == 0 && stride > 0, "blur_pool: need H,W>1 and C%%8==0 (C=%d)", C);
  const long total = (long)B * Ho * Wo * (C / 8);
  if (dtype == kBF16)
    blur_pool_kernel<<<rgrid(total, 256), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                           reinterpret_cast<__nv_bfloat16*>(out), total, H, W, C, Ho, Wo, stride);
  else if (dtype == kF32)
    blur_pool_kernel<<<rgrid(total, 256), 256, 0, stream>>>(reinterpret_cast<const float*>(x),
                                                           reinterpret_cast<float*>(out), total, H, W, C, Ho, Wo, stride);
  else {
    set_last_error("blur_pool: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("blur_pool_kernel");
  return kOk;
}

}  // extern "C"
