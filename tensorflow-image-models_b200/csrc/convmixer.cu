// The ConvMixer token mixer (tfimm/architectures/convmixer.py:63-68) on the CUDA cores, with the previous BatchNorm
// folded in (include/tfimm_b200_convmixer.h):
//   x = s_in a + t_in (0 in the padding),   y = x + s1 act(depthwise_k(x) + bias) + t1,   k in {7, 9}
//
// At k = 9 an output costs 81 FMAs against 6 to 8 bytes of HBM traffic, so the FP32 pipe is the roof, not HBM.  The plan
// keeps the FMA pipe fed from registers and reads shared memory with 16-byte loads only:
//   - A CTA owns 32 channels (one per lane) of a TH x TW output tile of one image; its 8 warps split the tile's rows
//     (warp g: rows g, g + 8, ...).  Grid (tiles, C / 32, B).
//   - Fill: the tile plus its (k - 1) / 2 halo is read from a once, x = fmaf(s_in, a, t_in) is applied where the cell
//     lies inside the image and 0 is stored where it does not -- by position, never by value, since s_in 0 + t_in is
//     not 0 and an interior a can be exactly 0.  Shared memory is channel-major, [32][IH][IW] with IW = TW + k - 1
//     rounded up to 4 and the channel plane padded to PLANE = 4 (mod 8) floats.  A warp stores 8 channels x 4
//     consecutive cells per instruction: their banks 4 (c PLANE / 4 mod 8) + cell are all distinct.  Its global loads
//     are 4 runs of 8 consecutive channels (32 bytes each).
//   - Compute: each thread keeps its channel's k * k taps in registers (81 at k = 9) and TW fp32 accumulators for one
//     output row.  For each ky it streams the input row (IW floats, one LDS.128 per 4 cells: the lanes read 16 bytes at
//     channel stride PLANE, conflict-free for the same reason) and adds every cell into the accumulators it touches,
//     so only 4 input values are live at a time.  Shared memory is only read 16 bytes at a time, and each float read
//     feeds TW k / IW FMAs (6 at k = 9, TW = 16).
//   - Registers decide the tile: two CTAs of 256 threads per SM (so one CTA's fill overlaps the other's FMAs) allow
//     128 registers.  81 taps + 16 accumulators fit only if the taps need not survive a loop over rows, so at k = 9
//     each warp owns exactly one row of an 8 x 16 tile.  At k = 7 (49 taps) a warp owns two rows of a 16 x 16 tile.
//     With 16 x 16 tiles at k = 9 ptxas spills 28 bytes.
//   - Each accumulator sums its taps in (ky, kx) order starting from 0, then adds bias; the residual x is the centre
//     cell of the same shared tile.  No atomics: the output is bitwise reproducible.
// Tile shapes (rows x cols): k = 7: 16 x 16 (a 32 x 32 map is 4 tiles); k = 9: 8 x 16 (32 x 32 is 8 tiles, 16 x 16 is
// 2); and 8 x 8 when the map fits in it (1 x 1 up to 8 x 8 grids, from small inputs), where a larger tile would be
// mostly padding.
#include "common.cuh"
#include "tfimm_b200_convmixer.h"

namespace tfimm {
namespace {

constexpr int kCh = 32;       // channels per CTA, one per lane
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;

template <int K, int TH_, int TW_>
struct DwShape {
  static constexpr int P = (K - 1) / 2;
  static constexpr int TH = TH_, TW = TW_;
  static constexpr int IH = TH + K - 1;
  static constexpr int IW = (TW + K - 1 + 3) / 4 * 4;
  static constexpr int PLANE = IH * IW + ((IH * IW) % 8 == 0 ? 4 : 0);
  static constexpr int kSmem = kCh * PLANE * 4;
  static_assert(PLANE % 8 == 4, "channel planes must be an odd number of 16-byte units apart");
  static_assert(TH % kWarps == 0, "every warp owns the same number of rows");
  static_assert((IH * IW) % 8 == 0, "the fill splits the cells into quads shared by two warps");
};

__device__ __forceinline__ void store_out(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_out(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <int K, int TH, int TW, typename OutT>
__global__ void __launch_bounds__(kThreads, 2) convmixer_dwconv_kernel(
    const float* __restrict__ a, const float* __restrict__ s_in, const float* __restrict__ t_in,
    const float* __restrict__ taps, const float* __restrict__ bias, const float* __restrict__ s1,
    const float* __restrict__ t1, OutT* __restrict__ y, int H, int W, int C, int act) {
  using S = DwShape<K, TH, TW>;
  extern __shared__ float4 smem4[];
  float* xs = reinterpret_cast<float*>(smem4);
  const int tiles_w = (W + S::TW - 1) / S::TW;
  const int h0 = (blockIdx.x / tiles_w) * S::TH, w0 = (blockIdx.x % tiles_w) * S::TW;
  const int c0 = blockIdx.y * kCh, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long img = (long)b * H * W;

  // ---- fill: x of the tile and its halo, 0 outside the image.  Unrolled so that a thread has several global loads
  // in flight before its first shared store.
  {
    const int cl = 8 * (warp & 3) + (lane >> 2);  // 8 channels x 4 consecutive cells per warp instruction
    const float sg = __ldg(s_in + c0 + cl), tg = __ldg(t_in + c0 + cl);
    constexpr int kQuads = S::IH * S::IW / 4;
#pragma unroll 16
    for (int quad = warp >> 2; quad < kQuads; quad += kWarps / 4) {
      const int cell = quad * 4 + (lane & 3);
      const int r = cell / S::IW, col = cell - r * S::IW;
      const int h = h0 - S::P + r, w = w0 - S::P + col;
      float v = 0.f;
      if (h >= 0 && h < H && w >= 0 && w < W) v = fmaf(sg, __ldg(a + (img + (long)h * W + w) * C + c0 + cl), tg);
      xs[cl * S::PLANE + cell] = v;
    }
  }

  // ---- per-channel constants and taps (coalesced over the lanes)
  const int c = c0 + lane;
  float wt[K * K];
#pragma unroll
  for (int i = 0; i < K * K; ++i) wt[i] = __ldg(taps + (long)i * C + c);
  const float bc = __ldg(bias + c), s1c = __ldg(s1 + c), t1c = __ldg(t1 + c);
  __syncthreads();

  const float* plane = xs + lane * S::PLANE;
#pragma unroll 1
  for (int oh = warp; oh < S::TH; oh += kWarps) {
    const int h = h0 + oh;
    if (h >= H) break;
    float acc[S::TW];
#pragma unroll
    for (int i = 0; i < S::TW; ++i) acc[i] = 0.f;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
      const float4* row = reinterpret_cast<const float4*>(plane + (oh + ky) * S::IW);
#pragma unroll
      for (int j = 0; j < S::IW / 4; ++j) {
        const float4 v4 = row[j];
        const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = 4 * j + e;
#pragma unroll
          for (int kx = 0; kx < K; ++kx) {
            const int ow = col - kx;
            if (ow >= 0 && ow < S::TW) acc[ow] = fmaf(v[e], wt[ky * K + kx], acc[ow]);
          }
        }
      }
    }
    const float* xrow = plane + (oh + S::P) * S::IW + S::P;
    OutT* yrow = y + (img + (long)h * W + w0) * C + c;
#pragma unroll
    for (int ow = 0; ow < S::TW; ++ow) {
      if (w0 + ow < W) {
        const float z = apply_act<true>(acc[ow] + bc, act);
        store_out(yrow + (long)ow * C, xrow[ow] + fmaf(s1c, z, t1c));
      }
    }
  }
}

template <int K, int TH, int TW, typename OutT>
int launch(const float* a, const float* s_in, const float* t_in, const float* taps, const float* bias, const float* s1,
           const float* t1, OutT* y, int B, int H, int W, int C, int act, cudaStream_t stream) {
  using S = DwShape<K, TH, TW>;
  static std::atomic<unsigned long long> attr_devs{0};
  auto kernel = convmixer_dwconv_kernel<K, TH, TW, OutT>;
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, S::kSmem, attr_devs));
  const long tiles = (long)((H + S::TH - 1) / S::TH) * ((W + S::TW - 1) / S::TW);
  TFIMM_CHECK_ARG(tiles <= 0x7fffffffL, "convmixer_dwconv: %ld tiles exceed the grid", tiles);
  kernel<<<dim3((unsigned)tiles, C / kCh, B), kThreads, S::kSmem, stream>>>(a, s_in, t_in, taps, bias, s1, t1, y, H, W,
                                                                            C, act);
  TFIMM_LAUNCH_OK("convmixer_dwconv_kernel");
  return kOk;
}

template <typename OutT>
int dispatch(const float* a, const float* s_in, const float* t_in, const float* taps, const float* bias,
             const float* s1, const float* t1, OutT* y, int B, int H, int W, int C, int k, int act,
             cudaStream_t stream) {
  const bool small = H <= 8 && W <= 8;
  if (k == 7)
    return small ? launch<7, 8, 8>(a, s_in, t_in, taps, bias, s1, t1, y, B, H, W, C, act, stream)
                 : launch<7, 16, 16>(a, s_in, t_in, taps, bias, s1, t1, y, B, H, W, C, act, stream);
  return small ? launch<9, 8, 8>(a, s_in, t_in, taps, bias, s1, t1, y, B, H, W, C, act, stream)
               : launch<9, 8, 16>(a, s_in, t_in, taps, bias, s1, t1, y, B, H, W, C, act, stream);
}

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_convmixer_dwconv(const float* a, const float* s_in, const float* t_in, const float* taps,
                                const float* bias, const float* s1, const float* t1, void* y, int y_dtype, int B, int H,
                                int W, int C, int k, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0,
                  "convmixer_dwconv: need B, H, W, C > 0 (B=%d H=%d W=%d C=%d)", B, H, W, C);
  if (k != 7 && k != 9) {
    set_last_error("convmixer_dwconv: kernel size %d is not supported (7 or 9)", k);
    return kUnsupported;
  }
  if (C % kCh != 0) {
    set_last_error("convmixer_dwconv: C = %d is not a multiple of %d", C, kCh);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG(B <= 65535 && C / kCh <= 65535, "convmixer_dwconv: need B <= 65535 and C / 32 <= 65535");
  TFIMM_CHECK_ARG(y_dtype == kBF16 || y_dtype == kF32, "convmixer_dwconv: y_dtype must be bf16 or f32");
  TFIMM_CHECK_ARG(act >= kActNone && act <= kActSigmoid, "convmixer_dwconv: unknown activation code %d", act);
  TFIMM_CHECK_ARG(a != nullptr && s_in != nullptr && t_in != nullptr && taps != nullptr && bias != nullptr &&
                      s1 != nullptr && t1 != nullptr && y != nullptr,
                  "convmixer_dwconv: null pointer argument");
  TFIMM_CHECK_ARG(static_cast<const void*>(a) != y, "convmixer_dwconv: y must not alias a");
  if (y_dtype == kBF16)
    return dispatch(a, s_in, t_in, taps, bias, s1, t1, static_cast<__nv_bfloat16*>(y), B, H, W, C, k, act, stream);
  return dispatch(a, s_in, t_in, taps, bias, s1, t1, static_cast<float*>(y), B, H, W, C, k, act, stream);
}

}  // extern "C"
