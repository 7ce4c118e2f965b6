// Depthwise k x k convolution + folded-BN bias + activation (+ fused squeeze sums) for the MBConv families:
// PadDepthwiseConv2D -> BatchNormalization -> act  [-> reduce_mean for SqueezeExcite]
// (tfimm/architectures/efficientnet_blocks.py:312-323, 393-404, 241-242; tfimm/layers/conv.py:91-148).
//
// HBM-bound by arithmetic (9-25 MACs per element); the first version of this kernel was *instruction* bound
// (ncu: 144 issued instructions per output pair, profiles/r01_*), so the design goals are memory-level
// parallelism and a lean inner loop:
//   * one warp = one output row x 64 channels; a lane owns a channel PAIR (4-byte bf16x2 accesses, 128 B per
//     warp instruction), its k*k taps stay in registers as packed fp32 pairs for the whole row
//   * the row is walked in strips of TW output pixels; the k x ((TW-1)*s + k) raw input window of strip i+1
//     is loaded into a second register buffer BEFORE strip i is computed (15-55 independent loads in flight)
//   * interior strips (whole window inside the image) take a branch-free path with per-row base pointers;
//     only border strips pay for bounds predicates
//   * activation on packed pairs; squeeze sums accumulate in registers: one atomic per channel per row
#include "common.cuh"

namespace tfimm {
namespace {

template <typename T>
struct RawPair;
template <>
struct RawPair<__nv_bfloat16> {
  using type = uint32_t;
  static __device__ __forceinline__ type load(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }
  static __device__ __forceinline__ type zero() { return 0u; }
  static __device__ __forceinline__ uint64_t to_f32x2(type u) {
    return pack2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
  }
};
template <>
struct RawPair<float> {
  using type = uint64_t;
  static __device__ __forceinline__ type load(const float* p) {
    const float2 f = *reinterpret_cast<const float2*>(p);
    return pack2(f.x, f.y);
  }
  static __device__ __forceinline__ type zero() { return pack2(0.f, 0.f); }
  static __device__ __forceinline__ uint64_t to_f32x2(type u) { return u; }
};

// Activation of a whole output strip.  bf16 mode: accurate swish on groups of four elements (common.cuh); fp32 mode
// (the 1e-5 structural-parity path): libm-exact scalar forms.
template <bool kBf16, int N>
__device__ __forceinline__ void act_strip(uint64_t (&acc)[N], int act) {
  if (act == kActNone) return;
  if (kBf16 && act == kActSwish && N % 2 == 0) {
#pragma unroll
    for (int i = 0; i < N; i += 2) {
      swish4(acc[i], acc[i + 1]);
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float a, b;
    unpack2(acc[i], a, b);
    acc[i] = pack2(apply_act<!kBf16>(a, act), apply_act<!kBf16>(b, act));
  }
}

template <typename T, int KS, int STRIDE, int TW>
__global__ void __launch_bounds__(128)
dwconv_act_pairs_kernel(const T* __restrict__ x, const float* __restrict__ wgt /*[KS*KS][C]*/,
                        const float* __restrict__ bias, T* __restrict__ out, float* __restrict__ pool_sum, int B,
                        int H, int W, int C, int Ho, int Wo, int pad_t, int pad_l, int act) {
  using RP = RawPair<T>;
  using Raw = typename RP::type;
  constexpr int IW = (TW - 1) * STRIDE + KS;  // input columns feeding one strip
  const int cgroups = (C + 63) >> 6;
  const long unit = (long)blockIdx.x * 4 + (threadIdx.x >> 5);
  const long units = (long)B * Ho * cgroups;
  if (unit >= units) return;
  const int lane = threadIdx.x & 31;
  const int cg = (int)(unit % cgroups);
  const long t = unit / cgroups;
  const int oy = (int)(t % Ho);
  const int b = (int)(t / Ho);
  const int c = cg * 64 + lane * 2;
  if (c >= C) return;

  uint64_t w[KS * KS];
#pragma unroll
  for (int i = 0; i < KS * KS; ++i) w[i] = pack2(__ldg(wgt + (size_t)i * C + c), __ldg(wgt + (size_t)i * C + c + 1));
  const uint64_t bv = bias != nullptr ? pack2(__ldg(bias + c), __ldg(bias + c + 1)) : pack2(0.f, 0.f);

  // per-tap-row base pointers (column 0 of the image row) and validity
  const T* rowp[KS];
  bool rowok[KS];
  bool rows_all_ok = true;
#pragma unroll
  for (int ky = 0; ky < KS; ++ky) {
    const int iy = oy * STRIDE + ky - pad_t;
    rowok[ky] = iy >= 0 && iy < H;
    rows_all_ok = rows_all_ok && rowok[ky];
    rowp[ky] = x + (((long)b * H + (rowok[ky] ? iy : 0)) * W) * C + c;
  }

  auto load_window = [&](int ox0, Raw (&buf)[KS][IW]) {
    const int gx0 = ox0 * STRIDE - pad_l;
    if (rows_all_ok && gx0 >= 0 && gx0 + IW <= W) {
      // interior: no predicates, one pointer bump per column
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
        const T* p = rowp[ky] + (long)gx0 * C;
#pragma unroll
        for (int ix = 0; ix < IW; ++ix) buf[ky][ix] = RP::load(p + (long)ix * C);
      }
    } else {
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
#pragma unroll
        for (int ix = 0; ix < IW; ++ix) {
          const int gx = gx0 + ix;
          buf[ky][ix] = (rowok[ky] && gx >= 0 && gx < W) ? RP::load(rowp[ky] + (long)gx * C) : RP::zero();
        }
      }
    }
  };

  uint64_t ps = pack2(0.f, 0.f);
  T* orow = out + (((long)b * Ho + oy) * Wo) * C + c;
  Raw nxt[KS][IW];
  load_window(0, nxt);
#pragma unroll 1
  for (int ox0 = 0; ox0 < Wo; ox0 += TW) {
    Raw cur[KS][IW];
#pragma unroll
    for (int ky = 0; ky < KS; ++ky)
#pragma unroll
      for (int ix = 0; ix < IW; ++ix) cur[ky][ix] = nxt[ky][ix];
    if (ox0 + TW < Wo) load_window(ox0 + TW, nxt);  // in flight while this strip is computed

    uint64_t acc[TW];
#pragma unroll
    for (int i = 0; i < TW; ++i) acc[i] = bv;
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
#pragma unroll
      for (int ix = 0; ix < IW; ++ix) {
        const uint64_t v = RP::to_f32x2(cur[ky][ix]);
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          if ((ix - kx) >= 0 && (ix - kx) % STRIDE == 0 && (ix - kx) / STRIDE < TW)
            acc[(ix - kx) / STRIDE] = fma2(v, w[ky * KS + kx], acc[(ix - kx) / STRIDE]);
        }
      }
    }
    act_strip<sizeof(T) == 2>(acc, act);
#pragma unroll
    for (int i = 0; i < TW; ++i) {
      if (ox0 + i < Wo) {
        const uint64_t a = acc[i];
        float a0, a1;
        unpack2(a, a0, a1);
        T* dst = orow + (long)(ox0 + i) * C;
        if constexpr (sizeof(T) == 2) {
          const uint32_t packed = pack_bf16x2(a0, a1);
          *reinterpret_cast<uint32_t*>(dst) = packed;
          // squeeze sums see what the next layer actually reads (bf16-rounded)
          if (pool_sum != nullptr) ps = add2(ps, RP::to_f32x2(packed));
        } else {
          *reinterpret_cast<float2*>(dst) = make_float2(a0, a1);
          ps = add2(ps, a);
        }
      }
    }
  }
  if (pool_sum != nullptr) {
    float p0, p1;
    unpack2(ps, p0, p1);
    atomicAdd(pool_sum + (long)b * C + c, p0);
    atomicAdd(pool_sum + (long)b * C + c + 1, p1);
  }
}

}  // namespace

int dwconv_bias_act_pairs(const void* x, int dtype, const float* wgt, const float* bias, void* out, float* pool_sum,
                          int B, int H, int W, int C, int ks, int stride, int pad_t, int pad_l, int Ho, int Wo,
                          int act, cudaStream_t stream) {
  if (C % 2 != 0 || !(ks == 3 || ks == 5) || !(stride == 1 || stride == 2)) return kUnsupported;
  const long units = (long)B * Ho * ((C + 63) / 64);
  const unsigned grid = (unsigned)((units + 3) / 4);
#define TFIMM_DWP(T, KS, ST, TW)                                                                             \
  dwconv_act_pairs_kernel<T, KS, ST, TW><<<grid, 128, 0, stream>>>(reinterpret_cast<const T*>(x), wgt, bias, \
                                                                  reinterpret_cast<T*>(out), pool_sum, B, H, W, C, \
                                                                  Ho, Wo, pad_t, pad_l, act)
  // strip width: 8 outputs for the bf16 3x3/s1 case (window 10 columns x 3 rows per buffer), 4 otherwise --
  // chosen so that the two raw-window register buffers + taps stay under 255 registers without spilling
#define TFIMM_DWP_T(T, TW31)                             \
  do {                                                   \
    if (ks == 3 && stride == 1) TFIMM_DWP(T, 3, 1, TW31); \
    else if (ks == 3) TFIMM_DWP(T, 3, 2, 4);             \
    else if (stride == 1) TFIMM_DWP(T, 5, 1, 4);         \
    else TFIMM_DWP(T, 5, 2, 4);                          \
  } while (0)
  if (dtype == kBF16) TFIMM_DWP_T(__nv_bfloat16, 8);
  else if (dtype == kF32) TFIMM_DWP_T(float, 4);
  else return kUnsupported;
#undef TFIMM_DWP_T
#undef TFIMM_DWP
  TFIMM_LAUNCH_OK("dwconv_act_pairs_kernel");
  return kOk;
}

}  // namespace tfimm
