// Shared device/host helpers for the tfimm_b200 kernel library (sm_90a).
//
// Everything in here is a thin wrapper over a PTX instruction or a small
// utility used by more than one translation unit.  No torch types, no
// allocation: the C ABI in include/tfimm_b200.h only ever sees raw device
// pointers owned by the caller.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "tfimm_b200.h"

namespace tfimm {

// ----------------------------------------------------------------------------
// Status / error reporting (thread-local message, C ABI returns int status).
// ----------------------------------------------------------------------------
enum Status : int {
  kOk = TFIMM_OK,
  kInvalidArgument = TFIMM_ERR_INVALID_ARGUMENT,
  kCudaError = TFIMM_ERR_CUDA,
  kUnsupported = TFIMM_ERR_UNSUPPORTED,
};

void set_last_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define TFIMM_CHECK_ARG(cond, ...)                \
  do {                                            \
    if (!(cond)) {                                \
      ::tfimm::set_last_error(__VA_ARGS__);       \
      return ::tfimm::kInvalidArgument;           \
    }                                             \
  } while (0)

#define TFIMM_CUDA_OK(expr)                                   \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) return ::tfimm::cuda_fail(_e, #expr); \
  } while (0)

#define TFIMM_LAUNCH_OK(name)                                  \
  do {                                                         \
    cudaError_t _e = cudaGetLastError();                       \
    if (_e != cudaSuccess) return ::tfimm::cuda_fail(_e, name); \
  } while (0)

enum DType : int { kF32 = TFIMM_F32, kBF16 = TFIMM_BF16, kU8 = TFIMM_U8 };

enum Act : int {
  kActNone = TFIMM_ACT_NONE,
  kActGelu = TFIMM_ACT_GELU,    // exact erf form (Keras "gelu")
  kActSwish = TFIMM_ACT_SWISH,  // x * sigmoid(x)
  kActRelu = TFIMM_ACT_RELU,
  kActRelu6 = TFIMM_ACT_RELU6,
  kActTanh = TFIMM_ACT_TANH,
  kActSigmoid = TFIMM_ACT_SIGMOID,
};

// The C entry points take the stream as void* (the header is plain C).
inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

int sm_count();  // of the CURRENT device (cached per device)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device setting: `devs` (one static per kernel
// instantiation) records the devices it has been set on.  A device is recorded only once the call has succeeded, so no
// thread launches before the attribute is in place, and a failed call is tried again on the next launch.
// nonportable_cluster: also allow cluster sizes above 8 (cudaFuncAttributeNonPortableClusterSizeAllowed).
template <typename Kernel>
cudaError_t set_max_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>& devs,
                                 bool nonportable_cluster = false) {
  int dev = 0;
  const bool known = cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev <= 63;
  const unsigned long long bit = known ? 1ull << dev : 0;
  if (known && (devs.load(std::memory_order_acquire) & bit)) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && nonportable_cluster)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (e == cudaSuccess) devs.fetch_or(bit, std::memory_order_release);
  return e;
}

// tmap.cu: TMA descriptors (SWIZZLE_128B, zero OOB fill)
int make_tmap(CUtensorMap* map, const void* ptr, int dtype, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, const char* what, int swizzle_bytes = 128,
              const uint32_t* elem_strides = nullptr);
int make_tmap_2d(CUtensorMap* map, const void* ptr, int dtype, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols, const char* what, int swizzle_bytes = 128);

// ----------------------------------------------------------------------------
// Small device math
// ----------------------------------------------------------------------------
constexpr float kLog2e = 1.4426950408889634f;

#if defined(__CUDACC__)

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// a / l, correctly rounded, given inv = 1.0f / l (itself correctly rounded): q = a inv is within an ulp of a / l, the
// remainder a - q l is exact in one fma, and q + remainder * inv rounds to the correctly rounded quotient (Markstein).
// Attention normalises every output of a row by its row sum l: the plain product a * inv would carry the one rounding
// error of inv into all of them alike, a bias that decides the bf16 rounding of every output near a tie the same way.
__device__ __forceinline__ float div_rn_by(float a, float l, float inv) {
  const float q = a * inv;
  return fmaf(fmaf(-q, l, a), inv, q);
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// GELU (exact erf form) for GEMM epilogues: x * Phi(x) with
//   erfc(z) ~= t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2),  t = 1 / (1 + p z),  z = |x| / sqrt(2)
// (Abramowitz & Stegun 7.1.26, |abs err| < 1.5e-7 on erfc).  Written on the erfc side so there is no
// cancellation for negative x.  Two MUFU ops (rcp, ex2) + ~14 FMA-pipe ops per element.
__device__ __forceinline__ float gelu_fast(float x) {
  const float ax = fabsf(x);
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678f, ax, 1.0f));
  float p = 1.061405429f;
  p = fmaf(p, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  // exp(-x^2 / 2) = exp2(-x^2 * log2(e) / 2)
  const float e = ex2_approx(ax * ax * -0.72134752044448170368f);
  const float h = 0.5f * ax * (p * t * e);  // |x| * Phi(-|x|)
  return x > 0.f ? x - h : -h;
}

// ---- fp32 pairs: two values carried in one 64-bit register pair, operated on element by element ----
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ uint64_t splat2(float v) { return pack2(v, v); }
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}

// ---- accurate activations for the tensor-core epilogues (packed pairs, groups of FOUR elements) ----
// The bf16 parity budget (tests/test_parity_budget_gpu.py) needs every value to be right to ~1e-5 BEFORE it is rounded
// to bf16: a pre-rounding error d flips the rounding of a fraction d/ulp of the elements by a whole ulp, i.e. it adds
// noise of variance d*ulp against the ulp^2/12 inherent to bf16 storage -- tanh.approx (2^-11) would DOUBLE the noise
// (one-MUFU tanh.approx forms put 12-25 % of the stored values off by an ulp).
// Both activations are written as x * sigma with sigma = 1 / (1 + 2^u): one MUFU.EX2 (rel. error 2^-22) and one
// MUFU.RCP per element.
// kSharedRcp: ONE MUFU.RCP for four elements -- 1 / (d0 d1 d2 d3), the four quotients recovered with nine
// multiplications (u clamped to 28 so that the product stays below 2^127) -- 1.25 MUFU per element instead of 2, for
// kernels whose activation warps are bound by the MUFU pipe (16 lanes / clk / SM) rather than by issue slots.
template <bool kSharedRcp = false>
__device__ __forceinline__ void sigma4_from_log2(uint64_t u01, uint64_t u23, uint64_t& s01, uint64_t& s23) {
  float u0, u1, u2, u3;
  unpack2(u01, u0, u1);
  unpack2(u23, u2, u3);
  const uint64_t one2 = splat2(1.0f);
  float d0, d1, d2, d3;
  if constexpr (kSharedRcp) {
    unpack2(add2(pack2(ex2_approx(fminf(u0, 28.f)), ex2_approx(fminf(u1, 28.f))), one2), d0, d1);
    unpack2(add2(pack2(ex2_approx(fminf(u2, 28.f)), ex2_approx(fminf(u3, 28.f))), one2), d2, d3);
    const float p01 = d0 * d1, p23 = d2 * d3;
    const float inv = rcp_approx(p01 * p23);
    const float r01 = inv * p23, r23 = inv * p01;  // 1 / (d0 d1), 1 / (d2 d3)
    s01 = mul2(pack2(d1, d0), splat2(r01));        // (1/d0, 1/d1)
    s23 = mul2(pack2(d3, d2), splat2(r23));
  } else {
    unpack2(add2(pack2(ex2_approx(u0), ex2_approx(u1)), one2), d0, d1);
    unpack2(add2(pack2(ex2_approx(u2), ex2_approx(u3)), one2), d2, d3);
    s01 = pack2(rcp_approx(d0), rcp_approx(d1));   // 2^u = +inf -> rcp = +0: no clamp needed
    s23 = pack2(rcp_approx(d2), rcp_approx(d3));
  }
}
// swish(x) = x * sigmoid(x), sigmoid(x) = 1 / (1 + 2^(-x log2 e)).
template <bool kSharedRcp = false>
__device__ __forceinline__ void swish4(uint64_t& x01, uint64_t& x23) {
  const uint64_t nl2e = splat2(-1.4426950408889634f);
  uint64_t s01, s23;
  sigma4_from_log2<kSharedRcp>(mul2(x01, nl2e), mul2(x23, nl2e), s01, s23);
  x01 = mul2(x01, s01);
  x23 = mul2(x23, s23);
}
// erf-GELU: Phi(x) = 1 / (1 + 2^(-x q(x^2))) holds exactly for x q(x^2) ln 2 = logit(Phi(x)); q is a degree-4
// polynomial in x^2 fitted on |x| <= 5.5.  Max |error| of x Phi(x) against the exact erf form, evaluated in fp32:
// 3.6e-6 (tools/fit_gelu.py), i.e. < 1/500 of a bf16 ulp for |y| >= 0.5.  No clamp: beyond the fitted range q stays
// positive and increasing (q(30.25) = 5.4, leading coefficient > 0), so u keeps the sign of -x and grows, Phi is 0 / 1
// to 1e-9 there anyway, and overflow of the Horner chain ends in +inf (every later step adds a finite constant).
__device__ __forceinline__ uint64_t gelu_neg_log2_odds(uint64_t x) {
  const uint64_t t = mul2(x, x);
  uint64_t q = fma2(splat2(3.2899208690650994e-06f), t, splat2(-8.927415183279663e-05f));
  q = fma2(q, t, splat2(-0.0003550456603989005f));
  q = fma2(q, t, splat2(0.10521824657917023f));
  q = fma2(q, t, splat2(2.3020482063293457f));
  return mul2(mul2(x, splat2(-1.0f)), q);
}
template <bool kSharedRcp = false>
__device__ __forceinline__ void gelu4(uint64_t& x01, uint64_t& x23) {
  uint64_t s01, s23;
  sigma4_from_log2<kSharedRcp>(gelu_neg_log2_odds(x01), gelu_neg_log2_odds(x23), s01, s23);
  x01 = mul2(x01, s01);
  x23 = mul2(x23, s23);
}

template <bool kPrecise>
__device__ __forceinline__ float gelu_erf(float x) {
  if constexpr (kPrecise) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
  } else {
    return gelu_fast(x);
  }
}

template <bool kPrecise>
__device__ __forceinline__ float sigmoidf_(float x) {
  if constexpr (kPrecise) {
    return 1.0f / (1.0f + expf(-x));
  } else {
    return rcp_approx(1.0f + ex2_approx(-x * 1.4426950408889634f));
  }
}

template <bool kPrecise>
__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case kActGelu: return gelu_erf<kPrecise>(v);
    case kActSwish: return v * sigmoidf_<kPrecise>(v);
    case kActRelu: return fmaxf(v, 0.0f);
    case kActRelu6: return fminf(fmaxf(v, 0.0f), 6.0f);
    case kActTanh: return tanhf(v);
    case kActSigmoid: return sigmoidf_<kPrecise>(v);
    default: return v;
  }
}

// Activation over a register array with the switch hoisted out of the element loop.
template <bool kPrecise, int N>
__device__ __forceinline__ void apply_act_array(float (&v)[N], int act) {
  switch (act) {
    case kActGelu:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = gelu_erf<kPrecise>(v[j]);
      break;
    case kActSwish:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = v[j] * sigmoidf_<kPrecise>(v[j]);
      break;
    case kActRelu:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = fmaxf(v[j], 0.0f);
      break;
    case kActRelu6:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = fminf(fmaxf(v[j], 0.0f), 6.0f);
      break;
    case kActTanh:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = tanhf(v[j]);
      break;
    case kActSigmoid:
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = sigmoidf_<kPrecise>(v[j]);
      break;
    default:
      break;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(h);
}

// Typed scalar load/store helpers used by templated kernels.
__device__ __forceinline__ float ld_as_float(const float* p) { return *p; }
__device__ __forceinline__ float ld_as_float(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float ld_as_float(const uint8_t* p) { return (float)(*p); }
__device__ __forceinline__ void st_from_float(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_from_float(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// Load 8 consecutive elements as floats (16B-aligned for bf16, 32B for f32).
__device__ __forceinline__ void ld8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  float2 f;
  f = unpack_bf16x2(a.x); v[0] = f.x; v[1] = f.y;
  f = unpack_bf16x2(a.y); v[2] = f.x; v[3] = f.y;
  f = unpack_bf16x2(a.z); v[4] = f.x; v[5] = f.y;
  f = unpack_bf16x2(a.w); v[6] = f.x; v[7] = f.y;
}
__device__ __forceinline__ void ld8(const uint8_t* p, float (&v)[8]) {   // 8-byte aligned
  const uint2 a = *reinterpret_cast<const uint2*>(p);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    v[j] = (float)((a.x >> (8 * j)) & 0xffu);
    v[4 + j] = (float)((a.y >> (8 * j)) & 0xffu);
  }
}
__device__ __forceinline__ void st8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 a;
  a.x = pack_bf16x2(v[0], v[1]);
  a.y = pack_bf16x2(v[2], v[3]);
  a.z = pack_bf16x2(v[4], v[5]);
  a.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = a;
}

// ----------------------------------------------------------------------------
// PTX wrappers: shared-memory addresses, mbarrier, TMA, wgmma.
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// try_wait parks the thread in hardware until the phase completes or the time hint (ns; the hardware caps it) runs out,
// so a waiting warp issues a handful of instructions per microsecond instead of spinning in the issue slots of the
// warps that share its scheduler.
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
#ifdef TFIMM_TRYWAIT_NO_HINT
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
#else
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n"
#endif
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(1000000u)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug turns into a trap (reported as a CUDA error by the host) instead of a hung GPU: the
// cycle counter is read once on entry and then only every 256th poll, ~4e9 cycles is a couple of seconds.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 255u) == 0 && clock64() - t0 > 4000000000LL) __trap();
  }
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Named barrier kId (1..15; 0 is __syncthreads) over `threads` threads, a multiple of 32.  The id is an immediate so
// that ptxas reserves only the barriers a kernel names.
template <int kId>
__device__ __forceinline__ void named_bar_sync(int threads) {
  asm volatile("bar.sync %0, %1;" ::"n"(kId), "r"(threads) : "memory");
}

__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// 2D tiled TMA load: global (via tensor map) -> shared, completion on mbarrier.
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const void* tmap, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 2D tiled TMA store: shared -> global (via tensor map), bulk-group completion.
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t src_smem, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src_smem), "r"(c0), "r"(c1)
      : "memory");
}
// 3D variants (innermost coordinate first).
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const void* tmap, uint32_t bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst_smem, const void* tmap, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, uint32_t src_smem, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t src_smem, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---- wgmma (warpgroup MMA, sm_90a) -----------------------------------------
// Shared-memory matrix descriptor for a K-major bf16 tile whose rows are exactly one 128-byte swizzle span (64 bf16),
// written by TMA SWIZZLE_128B; the tile base must be 1024-byte aligned.
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   [32,46) stride byte offset >> 4 (8 rows * 128 B = 1024)   [62,64) layout: 1 = SWIZZLE_128B
// Advancing 16 elements along K inside the span is +32 bytes, i.e. +2 on the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// Descriptor for an MN-major bf16 B tile (wgmma imm-trans-b = 1) written by TMA SWIZZLE_128B as boxes of 64 MN
// elements (one 128-byte span) x 64 K rows: every K row is a 128-byte span, the swizzle atom is 64 MN x 8 K (1024 B).
// Here the two offsets mean something else than in the K-major form:
//   leading byte offset = stride between 64-element MN atoms (the next TMA box: 64 rows * 128 B = 8192)
//   stride byte offset  = stride between 8-row K groups (1024)
// Advancing 16 elements along K is 16 rows = 2048 bytes, i.e. +128 on the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)(8192 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// ---- thread-block clusters ----
__device__ __forceinline__ void cluster_arrive_release() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait_acquire() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// ---- cp.async / ldmatrix / mma.sync (used by the attention kernels) ---------
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                            uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1,
                                                  uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
// D(16x8, f32) += A(16x16, bf16, row) * B(16x8, bf16, col)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
      "{%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---- TF32 (precision="tf32") ----
// fp32 -> TF32 (10 explicit mantissa bits, low 13 bits of the result zero): round to nearest, ties away from zero.
// Finite values at the top of the range round up to +-inf; NaN and inf pass through.  Every TF32 operand is rounded by
// this instruction (the tensor core would otherwise use the low bits as it pleases), and the plan-time weight rounding
// (tfimm.backend.lib.round_tf32) is the same function.
__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
// D(16x8, f32) += A(16x8, tf32, row) * B(8x8, tf32, col)
__device__ __forceinline__ void mma_tf32_1688(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 "
      "{%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

#endif  // __CUDACC__

}  // namespace tfimm
