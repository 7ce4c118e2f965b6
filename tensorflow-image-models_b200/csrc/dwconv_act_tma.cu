// Depthwise k x k convolution (k in {3,5}, stride 1/2) + folded-BN bias + activation (+ fused squeeze sums) for the
// MBConv families, bf16 NHWC: PadDepthwiseConv2D -> BatchNormalization -> act [-> reduce_mean for SqueezeExcite]
// (tfimm/architectures/efficientnet_blocks.py:312-323, 393-404, 241-242; tfimm/layers/conv.py:91-148).
//
// HBM-bound by arithmetic (9-25 MACs per element), but the register-window kernel (dwconv_act.cu) was bound by
// its own address arithmetic: 81 issued instructions per output channel pair, 46 % of them integer ops for global
// addresses with a runtime channel stride (ncu: profiles/r01_ncu_full_dwconv_act_pairs.txt).  Here the input goes
// through shared memory, where every offset is a compile-time immediate:
//   * one CTA = TH x TW output pixels x 64 channels; its input halo ((TH-1)s+k) x ((TW-1)s+k) x 64 bf16 arrives as
//     ONE 4-D TMA box; the TF-"SAME" / symmetric zero padding (tfimm/layers/conv.py:15-28) and the channel tail are
//     the TMA out-of-bounds fill -- no predicates in the load path
//   * lane = channel pair (one 4-byte LDS per pixel, 128 B per warp instruction, conflict-free), warp = strips of 8
//     outputs along a row; k*k taps of the pair in registers as packed fp32 pairs; ~30 instructions per
//     output pair for 3x3
//   * squeeze sums: per-lane packed accumulation -> cross-warp reduction in shared memory -> one atomic per channel
//     per CTA
// Several CTAs are resident per SM (44-85 KB of shared memory each), so one CTA's TMA load overlaps the others' math.
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kSlab = 64;        // channels per CTA
constexpr int kStrip = 8;        // outputs per strip
constexpr int kWarps = 8;

// SHAPE: output tile per CTA.  0: 8 x 32 (stride 1) / 8 x 16 (stride 2) for large maps; 1: half as wide; 2: half as
// wide and 4 rows -- EfficientNet's late stages run on 24 x 24 and 12 x 12 maps, where the large tile computes 1.3x /
// 3.6x more pixels than exist (B4 @ 380: the 12 x 12 x 1632 depthwise launches ran at 0.7 TB/s).
template <int KS, int STRIDE, int SHAPE>
struct DwTmaCfg {
  static constexpr int TH = SHAPE == 2 ? 4 : 8;
  static constexpr int TW = (STRIDE == 1 ? 32 : 16) / (SHAPE == 0 ? 1 : 2);
  static constexpr int IH = (TH - 1) * STRIDE + KS;
  static constexpr int IW = (TW - 1) * STRIDE + KS;
  static constexpr int kHaloBytes = IH * IW * kSlab * 2;
  static constexpr int kSmemBytes = ((kHaloBytes + 15) / 16) * 16 + kWarps * kSlab * 4 + 16;
  static constexpr int kStrips = TH * (TW / kStrip);
};

__device__ __forceinline__ uint64_t bf16x2_as_f32x2(uint32_t u) {
  return pack2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

template <int KS, int STRIDE, int SHAPE>
__global__ void __launch_bounds__(kWarps * 32)
dwconv_act_tma_kernel(const __grid_constant__ CUtensorMap tmap_x, const float* __restrict__ wgt /*[KS*KS][C]*/,
                      const float* __restrict__ bias, __nv_bfloat16* __restrict__ out, float* __restrict__ pool_sum,
                      int C, int Ho, int Wo, int pad_t, int pad_l, int tiles_x, int tiles_y, int cslabs, int act) {
  using Cfg = DwTmaCfg<KS, STRIDE, SHAPE>;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t* halo = reinterpret_cast<const uint32_t*>(smem);                       // [IH][IW][32] bf16x2
  float* red = reinterpret_cast<float*>(smem + ((Cfg::kHaloBytes + 15) / 16) * 16);     // [kWarps][64]
  const uint32_t bar = smem_u32(red + kWarps * kSlab);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // channel slab fastest: concurrently running CTAs touch the same pixels' neighbouring channels
  int t = blockIdx.x;
  const int cs = t % cslabs; t /= cslabs;
  const int tx = t % tiles_x; t /= tiles_x;
  const int ty = t % tiles_y;
  const int b = t / tiles_y;
  const int oy0 = ty * Cfg::TH, ox0 = tx * Cfg::TW;
  const int c = cs * kSlab + 2 * lane;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_x);
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_expect_tx(bar, Cfg::kHaloBytes);
    tma_load_4d(smem_u32(smem), &tmap_x, bar, cs * kSlab, ox0 * STRIDE - pad_l, oy0 * STRIDE - pad_t, b);
  }
  // taps and bias of this lane's channel pair while the halo is in flight
  const bool c_ok = c < C;
  const int cl = c_ok ? c : 0;
  uint64_t w[KS * KS];
#pragma unroll
  for (int i = 0; i < KS * KS; ++i) w[i] = pack2(__ldg(wgt + (size_t)i * C + cl), __ldg(wgt + (size_t)i * C + cl + 1));
  const uint64_t bv = bias != nullptr ? pack2(__ldg(bias + cl), __ldg(bias + cl + 1)) : pack2(0.f, 0.f);
  __syncthreads();  // barrier init visible to the waiters
  mbar_wait(bar, 0);

  uint64_t ps = pack2(0.f, 0.f);
#pragma unroll 1
  for (int s = warp; s < Cfg::kStrips; s += kWarps) {
    const int ry = s / (Cfg::TW / kStrip), sx = (s % (Cfg::TW / kStrip)) * kStrip;
    const int oy = oy0 + ry;
    if (oy >= Ho || ox0 + sx >= Wo) continue;
    uint64_t acc[kStrip];
#pragma unroll
    for (int i = 0; i < kStrip; ++i) acc[i] = bv;
    constexpr int IWS = (kStrip - 1) * STRIDE + KS;  // input columns feeding one strip
    const uint32_t* base = halo + ((size_t)(ry * STRIDE) * Cfg::IW + sx * STRIDE) * 32 + lane;
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
#pragma unroll
      for (int ix = 0; ix < IWS; ++ix) {
        const uint64_t v = bf16x2_as_f32x2(base[(ky * Cfg::IW + ix) * 32]);
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          if ((ix - kx) >= 0 && (ix - kx) % STRIDE == 0 && (ix - kx) / STRIDE < kStrip)
            acc[(ix - kx) / STRIDE] = fma2(v, w[ky * KS + kx], acc[(ix - kx) / STRIDE]);
        }
      }
    }
    // activation on the whole strip (kStrip = 8 pairs): accurate swish on groups of four elements (common.cuh)
    if (act == kActSwish) {
#pragma unroll
      for (int i = 0; i < kStrip; i += 2) {
        swish4(acc[i], acc[i + 1]);
      }
    } else if (act != kActNone) {
#pragma unroll
      for (int i = 0; i < kStrip; ++i) {
        float a0, a1;
        unpack2(acc[i], a0, a1);
        acc[i] = pack2(apply_act<false>(a0, act), apply_act<false>(a1, act));
      }
    }
    if (c_ok) {
      __nv_bfloat16* orow = out + (((long)b * Ho + oy) * Wo + ox0 + sx) * C + c;
#pragma unroll
      for (int i = 0; i < kStrip; ++i) {
        if (ox0 + sx + i < Wo) {
          const uint64_t a = acc[i];
          float a0, a1;
          unpack2(a, a0, a1);
          const uint32_t packed = pack_bf16x2(a0, a1);
          *reinterpret_cast<uint32_t*>(orow + (long)i * C) = packed;
          // squeeze sums see what the next layer actually reads (bf16-rounded)
          if (pool_sum != nullptr) ps = add2(ps, bf16x2_as_f32x2(packed));
        }
      }
    }
  }
  if (pool_sum != nullptr) {
    float p0, p1;
    unpack2(ps, p0, p1);
    red[warp * kSlab + 2 * lane] = p0;
    red[warp * kSlab + 2 * lane + 1] = p1;
    __syncthreads();
    if (threadIdx.x < kSlab && cs * kSlab + (int)threadIdx.x < C) {
      float sum = 0.f;
#pragma unroll
      for (int wi = 0; wi < kWarps; ++wi) sum += red[wi * kSlab + threadIdx.x];
      atomicAdd(pool_sum + (long)b * C + cs * kSlab + threadIdx.x, sum);
    }
  }
}

template <int KS, int STRIDE, int SHAPE>
int launch_dw_tma(const void* x, const float* wgt, const float* bias, void* out, float* pool_sum, int B, int H, int W,
                  int C, int pad_t, int pad_l, int Ho, int Wo, int act, cudaStream_t stream) {
  using Cfg = DwTmaCfg<KS, STRIDE, SHAPE>;
  CUtensorMap tmap;
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
  const uint32_t box[4] = {(uint32_t)kSlab, (uint32_t)Cfg::IW, (uint32_t)Cfg::IH, 1u};
  int rc = make_tmap(&tmap, x, kBF16, 4, dims, strides, box, "dwconv input", /*swizzle_bytes=*/0);
  if (rc != kOk) return rc;
  auto kernel = dwconv_act_tma_kernel<KS, STRIDE, SHAPE>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Cfg::kSmemBytes, attr_devs));
  const int tiles_x = (Wo + Cfg::TW - 1) / Cfg::TW, tiles_y = (Ho + Cfg::TH - 1) / Cfg::TH;
  const int cslabs = (C + kSlab - 1) / kSlab;
  const long grid = (long)B * tiles_y * tiles_x * cslabs;
  if (grid > 0x7fffffffL) return kUnsupported;
  kernel<<<(unsigned)grid, kWarps * 32, Cfg::kSmemBytes, stream>>>(tmap, wgt, bias, reinterpret_cast<__nv_bfloat16*>(out),
                                                                  pool_sum, C, Ho, Wo, pad_t, pad_l, tiles_x, tiles_y,
                                                                  cslabs, act);
  TFIMM_LAUNCH_OK("dwconv_act_tma_kernel");
  return kOk;
}

}  // namespace

// Returns kUnsupported (without setting an error) for shapes this formulation does not take.
int dwconv_bias_act_tma(const void* x, int dtype, const float* wgt, const float* bias, void* out, float* pool_sum,
                        int B, int H, int W, int C, int ks, int stride, int pad_t, int pad_l, int Ho, int Wo, int act,
                        cudaStream_t stream) {
  if (dtype != kBF16 || C % 8 != 0 || !(ks == 3 || ks == 5) || !(stride == 1 || stride == 2)) return kUnsupported;
  if ((reinterpret_cast<uintptr_t>(x) & 15u) != 0 || pad_t < 0 || pad_l < 0) return kUnsupported;
  // tile shape: the one that computes the fewest pixels beyond the map (ties: the larger tile)
  const int tw0 = stride == 1 ? 32 : 16;
  auto padded = [&](int th, int tw) { return (long)((Ho + th - 1) / th * th) * ((Wo + tw - 1) / tw * tw); };
  int shape = 0;
  long best = padded(8, tw0);
  if (padded(8, tw0 / 2) < best) { best = padded(8, tw0 / 2); shape = 1; }
  if (padded(4, tw0 / 2) < best) { best = padded(4, tw0 / 2); shape = 2; }
#define TFIMM_DWT(KS_, ST_)                                                                                          \
  do {                                                                                                               \
    if (shape == 0) return launch_dw_tma<KS_, ST_, 0>(x, wgt, bias, out, pool_sum, B, H, W, C, pad_t, pad_l, Ho, Wo, act, stream); \
    if (shape == 1) return launch_dw_tma<KS_, ST_, 1>(x, wgt, bias, out, pool_sum, B, H, W, C, pad_t, pad_l, Ho, Wo, act, stream); \
    return launch_dw_tma<KS_, ST_, 2>(x, wgt, bias, out, pool_sum, B, H, W, C, pad_t, pad_l, Ho, Wo, act, stream);     \
  } while (0)
  if (ks == 3 && stride == 1) TFIMM_DWT(3, 1);
  if (ks == 3) TFIMM_DWT(3, 2);
  if (stride == 1) TFIMM_DWT(5, 1);
  TFIMM_DWT(5, 2);
#undef TFIMM_DWT
}

}  // namespace tfimm
