// Kernels of the PVT v2 family (tfimm/architectures/pvt_v2.py): the block's ConvFFN fused into one kernel, and
// spatial-reduction attention at head dim 32 (pvt_v2_b0).  Everything else -- the overlapping patch embeddings (im2col
// with zero padding + GEMM), the LayerNorms, the q / kv / proj GEMMs, head-dim-64 attention (pvt.cu) and the token mean
// -- runs on the existing paths.
//
// pvt_v2_conv_mlp_kernel<C>  the ConvFFN of one block, in place on the fp32 residual stream:
//     out = residual + act(dwconv3x3(bf16(h W1^T + b1)) + b_dw) W2^T + b2        h: (B gh gw, C) bf16, row-major grid
//   The (tokens, hidden) activations never reach HBM.  A CTA owns a kTH x kTW (8 x 16) tile of one image's output grid,
//   8 warps.
//   - The LN2 output of the (kTH + 2) x (kTW + 2) halo is copied once (cp.async, zero-filled off the map), 180 rows
//     padded to 192.  Per chunk of 64 hidden channels, W1 rows and W2 columns go through a two-stage cp.async ring.
//   - fc1: the 12 x 2 (16 halo rows, 32 channels) tiles of the chunk, three per warp, on mma.sync m16n8k16 in fp32;
//     + b1, rounded to bf16 into shared memory -- as the unfused fc1 GEMM stores it -- except that halo cells off the
//     map are stored as 0: the depthwise convolution's zero padding is applied by position, not by value (fc1 of a
//     zero row would be b1).
//   - Warp w owns output row w of the tile (16 outputs).  Each thread builds its own fc2 A fragments: per element
//     b_dw + the 9 taps in fixed (ky, kx) order as fp32 fmas, the activation (common.cuh's apply_act<false>, the
//     bf16 form that dwconv_bias_act uses), rounded to bf16.  That is the arithmetic of dwconv_act_pairs_kernel
//     (dwconv_act.cu), element by element.
//   - fc2: mma.sync with those A fragments against the W2 chunk, accumulating (16, C) fp32 over the chunks; at the end
//     + b2, + residual, fp32 stores of the outputs that are on the map.
//   Shapes: C in {32, 64, 128}, hidden % 64 == 0.  No instance spills.
//
// pvt_sr_attention_{bf16,f32}_kernel<32>  spatial-reduction attention at head dim 32 (pvt_sr_attention.cuh).
#include "common.cuh"
#include "pvt_sr_attention.cuh"
#include "tfimm_b200_pvt_v2.h"

namespace tfimm {
namespace {

constexpr int kTH = 8, kTW = 16;                  // output tile
constexpr int kHW = kTW + 2;                      // halo width
constexpr int kHalo = (kTH + 2) * kHW;            // 180 halo cells
constexpr int kHaloRows = (kHalo + 15) / 16 * 16; // 192: whole m16 tiles
constexpr int kHC = 64;                           // hidden chunk
constexpr int kCmWarps = kTH;                     // one output row per warp
constexpr int kCmThreads = kCmWarps * 32;
constexpr int kHidBytes = (kHC + 8) * 2;          // shared row of a hidden chunk / of W2: 9 chunks, conflict-free

template <int C>
struct ConvMlpCfg {
  static constexpr int kRowBytes = (C + 8) * 2;   // shared row of h and W1: 5, 9 or 17 chunks
  static constexpr int kHBytes = kHaloRows * kRowBytes;
  static constexpr int kW1Bytes = kHC * kRowBytes;
  static constexpr int kW2Bytes = C * kHidBytes;
  static constexpr int kStageBytes = kW1Bytes + kW2Bytes;
  static constexpr int kSmem = kHBytes + 2 * kStageBytes + kHalo * kHidBytes;
};

__device__ __forceinline__ uint64_t bf16x2_to_f32x2(uint32_t u) {
  return pack2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

template <int C>
__global__ void __launch_bounds__(kCmThreads, 1)
pvt_v2_conv_mlp_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w1,
                       const float* __restrict__ b1, const float* __restrict__ wdw, const float* __restrict__ bdw,
                       const __nv_bfloat16* __restrict__ w2, const float* __restrict__ b2,
                       const float* residual, float* out, int gh, int gw, int hidden, int tiles_x, int act) {
  using Cfg = ConvMlpCfg<C>;
  constexpr int RB = Cfg::kRowBytes, CH = C / 8;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sH = smem_u32(smem);
  const uint32_t sStages = sH + Cfg::kHBytes;
  const uint32_t sHid = sStages + 2 * Cfg::kStageBytes;
  uint8_t* hid = smem + Cfg::kHBytes + 2 * Cfg::kStageBytes;

  const int b = blockIdx.y;
  const int y0 = (blockIdx.x / tiles_x) * kTH, x0 = (blockIdx.x % tiles_x) * kTW;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long img = (long)b * gh * gw;
  const int n_chunks = hidden / kHC;

  // halo cell p = (hy, hx) is grid cell (y0 - 1 + hy, x0 - 1 + hx)
  auto on_map = [&](int p, long& tok) {
    const int y = y0 - 1 + p / kHW, x = x0 - 1 + p % kHW;
    tok = img + (long)y * gw + x;
    return p < kHalo && y >= 0 && y < gh && x >= 0 && x < gw;
  };
  // one commit group per call (empty past the last chunk), so that wait_group counts stay uniform
  auto load_chunk = [&](int j) {
    if (j < n_chunks) {
      const uint32_t sW1 = sStages + (j & 1) * Cfg::kStageBytes, sW2 = sW1 + Cfg::kW1Bytes;
      for (int idx = tid; idx < kHC * CH; idx += kCmThreads) {
        const int r = idx / CH, c = idx - r * CH;
        cp_async_16(sW1 + r * RB + c * 16, w1 + (long)(j * kHC + r) * C + c * 8, true);
      }
      for (int idx = tid; idx < C * (kHC / 8); idx += kCmThreads) {
        const int r = idx / (kHC / 8), c = idx - r * (kHC / 8);
        cp_async_16(sW2 + r * kHidBytes + c * 16, w2 + (long)r * hidden + j * kHC + c * 8, true);
      }
    }
    cp_async_commit();
  };

  for (int idx = tid; idx < kHaloRows * CH; idx += kCmThreads) {
    const int p = idx / CH, c = idx - p * CH;
    long tok;
    const bool valid = on_map(p, tok);
    cp_async_16(sH + p * RB + c * 16, h + (valid ? tok : 0L) * C + c * 8, valid);
  }
  load_chunk(0);   // with the halo
  load_chunk(1);

  // this thread's fc1 stores: halo rows of its three (m16, n32) tiles, masked by position
  float acc2[C / 8][4];
#pragma unroll
  for (int i = 0; i < C / 8; ++i) acc2[i][0] = acc2[i][1] = acc2[i][2] = acc2[i][3] = 0.f;

#pragma unroll 1
  for (int j = 0; j < n_chunks; ++j) {
    cp_async_wait<1>();   // chunk j (and the halo) has landed for this thread
    __syncthreads();      // for every thread
    const uint32_t sW1 = sStages + (j & 1) * Cfg::kStageBytes, sW2 = sW1 + Cfg::kW1Bytes;

    // ---- fc1 over the halo: tile u = (m16 tile u / 2, channels 32 (u % 2) ..)
#pragma unroll 1
    for (int u = warp; u < 2 * (kHaloRows / 16); u += kCmWarps) {
      const int m = u >> 1, nh = u & 1;
      float s[4][4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < C / 16; ++ks) {
        uint32_t a[4];
        ldmatrix_x4(sH + (m * 16 + (lane & 15)) * RB + (ks * 2 + (lane >> 4)) * 16, a[0], a[1], a[2], a[3]);
#pragma unroll
        for (int np = 0; np < 2; ++np) {
          const int row = nh * 32 + np * 16 + (lane >> 4) * 8 + (lane & 7);
          uint32_t k0, k1, k2, k3;
          ldmatrix_x4(sW1 + row * RB + (ks * 2 + ((lane >> 3) & 1)) * 16, k0, k1, k2, k3);
          mma_bf16_16816(s[2 * np], a, k0, k1);
          mma_bf16_16816(s[2 * np + 1], a, k2, k3);
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int p = m * 16 + g + 8 * r;
        long tok;
        const bool valid = on_map(p, tok);
        if (p < kHalo) {
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int col = nh * 32 + nt * 8 + 2 * t;
            const float2 bb = __ldg(reinterpret_cast<const float2*>(b1 + j * kHC + col));
            *reinterpret_cast<uint32_t*>(hid + p * kHidBytes + col * 2) =
                valid ? pack_bf16x2(s[nt][2 * r] + bb.x, s[nt][2 * r + 1] + bb.y) : 0u;
          }
        }
      }
    }
    __syncthreads();   // the hidden chunk of the whole halo is in shared memory

    // ---- depthwise 3x3 + b_dw + act -> bf16 A fragments of fc2, one k16 step at a time
#pragma unroll
    for (int ks = 0; ks < kHC / 16; ++ks) {
      uint32_t a[4];
#pragma unroll
      for (int hi = 0; hi < 2; ++hi) {   // channels 16 ks + 2 t (+ 8 hi)
        const int col = ks * 16 + hi * 8 + 2 * t;
        const int ch = j * kHC + col;
        uint64_t wv[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const float2 w = __ldg(reinterpret_cast<const float2*>(wdw + (long)k * hidden + ch));
          wv[k] = pack2(w.x, w.y);
        }
        const float2 bd = __ldg(reinterpret_cast<const float2*>(bdw + ch));
#pragma unroll
        for (int r = 0; r < 2; ++r) {    // output (warp, g + 8 r) of the tile
          uint64_t acc = pack2(bd.x, bd.y);
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int p = (warp + ky) * kHW + g + 8 * r + kx;
              const uint32_t v = *reinterpret_cast<const uint32_t*>(hid + p * kHidBytes + col * 2);
              acc = fma2(bf16x2_to_f32x2(v), wv[ky * 3 + kx], acc);
            }
          float lo, hi2;
          unpack2(acc, lo, hi2);
          a[2 * hi + r] = pack_bf16x2(apply_act<false>(lo, act), apply_act<false>(hi2, act));
        }
      }
      // ---- fc2: acc2 += A (16, k16) W2[:, chunk k16]^T
#pragma unroll
      for (int np = 0; np < C / 16; ++np) {
        const int row = np * 16 + (lane >> 4) * 8 + (lane & 7);
        uint32_t k0, k1, k2, k3;
        ldmatrix_x4(sW2 + row * kHidBytes + (ks * 2 + ((lane >> 3) & 1)) * 16, k0, k1, k2, k3);
        mma_bf16_16816(acc2[2 * np], a, k0, k1);
        mma_bf16_16816(acc2[2 * np + 1], a, k2, k3);
      }
    }
    __syncthreads();      // every warp is done with the hidden chunk and with stage j & 1
    load_chunk(j + 2);
  }
  cp_async_wait<0>();     // only empty groups can be pending here

  // ---- epilogue: + b2, + residual, rows on the map
  const int y = y0 + warp;
  if (y >= gh) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int x = x0 + g + 8 * r;
    if (x >= gw) continue;
    const long row = (img + (long)y * gw + x) * C;
#pragma unroll
    for (int nt = 0; nt < C / 8; ++nt) {
      const int col = nt * 8 + 2 * t;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(b2 + col));
      const float2 res = *reinterpret_cast<const float2*>(residual + row + col);
      *reinterpret_cast<float2*>(out + row + col) =
          make_float2((acc2[nt][2 * r] + bb.x) + res.x, (acc2[nt][2 * r + 1] + bb.y) + res.y);
    }
  }
}

template <int C>
int launch_conv_mlp(const void* h, const void* w1, const float* b1, const float* wdw, const float* bdw, const void* w2,
                    const float* b2, const float* residual, float* out, int B, int gh, int gw, int hidden, int act,
                    cudaStream_t stream) {
  auto kernel = pvt_v2_conv_mlp_kernel<C>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, ConvMlpCfg<C>::kSmem, attr_devs));
  const int tiles_x = (gw + kTW - 1) / kTW, tiles_y = (gh + kTH - 1) / kTH;
  kernel<<<dim3(tiles_x * tiles_y, B), kCmThreads, ConvMlpCfg<C>::kSmem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(h), reinterpret_cast<const __nv_bfloat16*>(w1), b1, wdw, bdw,
      reinterpret_cast<const __nv_bfloat16*>(w2), b2, residual, out, gh, gw, hidden, tiles_x, act);
  TFIMM_LAUNCH_OK("pvt_v2_conv_mlp_kernel");
  return kOk;
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

constexpr int kDH = 32;
using Sra = PvtSra<kDH>;

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_pvt_v2_conv_mlp_bf16(const void* h, const void* w1, const float* b1, const float* wdw, const float* bdw,
                                    const void* w2, const float* b2, const float* residual, float* out, int B, int gh,
                                    int gw, int C, int hidden, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  if ((C != 32 && C != 64 && C != 128) || hidden <= 0 || hidden % kHC != 0) {
    set_last_error("pvt_v2_conv_mlp_bf16: needs C in {32, 64, 128} and hidden %% 64 == 0 (got C=%d hidden=%d)", C,
                   hidden);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && B <= 65535, "pvt_v2_conv_mlp_bf16: bad shape B=%d gh=%d gw=%d", B, gh,
                  gw);
  const long tiles = (long)((gh + kTH - 1) / kTH) * ((gw + kTW - 1) / kTW);
  TFIMM_CHECK_ARG(tiles <= 0x7fffffffL, "pvt_v2_conv_mlp_bf16: grid too large (%d x %d)", gh, gw);
  TFIMM_CHECK_ARG(h != nullptr && w1 != nullptr && w2 != nullptr && aligned(h, 16) && aligned(w1, 16) &&
                      aligned(w2, 16),
                  "pvt_v2_conv_mlp_bf16: h, w1 and w2 must be 16-byte aligned");
  TFIMM_CHECK_ARG(b1 != nullptr && wdw != nullptr && bdw != nullptr && b2 != nullptr && residual != nullptr &&
                      out != nullptr && aligned(b1, 8) && aligned(wdw, 8) && aligned(bdw, 8) && aligned(b2, 8) &&
                      aligned(residual, 8) && aligned(out, 8),
                  "pvt_v2_conv_mlp_bf16: b1, wdw, bdw, b2, residual and out must be 8-byte aligned");
  switch (C) {
    case 32: return launch_conv_mlp<32>(h, w1, b1, wdw, bdw, w2, b2, residual, out, B, gh, gw, hidden, act, stream);
    case 64: return launch_conv_mlp<64>(h, w1, b1, wdw, bdw, w2, b2, residual, out, B, gh, gw, hidden, act, stream);
    default: return launch_conv_mlp<128>(h, w1, b1, wdw, bdw, w2, b2, residual, out, B, gh, gw, hidden, act, stream);
  }
}

int tfimm_b200_pvt_v2_sr_attention_bf16(const void* q, const void* kv, void* out, int B, int N, int Nk, int H, int dh,
                                        float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_v2_sr_attention_bf16: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_v2_sr_attention_bf16: head_dim must be 32 (got %d)", dh);
  TFIMM_CHECK_ARG(B <= 65535 && H <= 65535, "pvt_v2_sr_attention_bf16: need B, H <= 65535 (B=%d H=%d)", B, H);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_v2_sr_attention_bf16: q, kv and out must be 16-byte aligned");
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

int tfimm_b200_pvt_v2_sr_attention_f32(const float* q, const float* kv, float* out, int B, int N, int Nk, int H,
                                       int dh, float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_v2_sr_attention_f32: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_v2_sr_attention_f32: head_dim must be 32 (got %d)", dh);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_v2_sr_attention_f32: q, kv and out must be 16-byte aligned");
  const long rows = (long)B * H * N;
  const long blocks = (rows + kF32Warps - 1) / kF32Warps;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pvt_v2_sr_attention_f32: problem too large (%ld blocks)", blocks);
  pvt_sr_attention_f32_kernel<kDH><<<(unsigned)blocks, kF32Warps * 32, 0, stream>>>(q, kv, out, rows, N, Nk, H, scale);
  TFIMM_LAUNCH_OK("pvt_sr_attention_f32_kernel");
  return kOk;
}

}  // extern "C"
