// Swin (shifted-)window attention on mma.sync, bf16, head_dim 32: tokens per window N <= 64, or N <= 144 (the 12 x 12
// windows of the *_window12_384 models) in a second instantiation.  Two entry points share the kernel: one takes the
// bias as [H][N][N] and the shift mask as per-token region labels, the other (kPadded, what the model uses for 7 x 7
// windows) the bias as a padded [H][64][64] table and the mask as one 64-bit word per query row.
//
// Reference: WindowAttention.call (tfimm/architectures/swin.py:159-198) wrapped by
// SwinTransformerBlock.call's tf.roll -> window_partition -> ... -> window_reverse -> tf.roll
// (swin.py:299-313).  Those five full-tensor copies are pure row permutations, so here they are a
// row-index table (row_map): each warp gathers the q/k/v rows of its (window, head) straight from the
// token-ordered qkv projection and scatters the result rows back to the same tokens.
//
// One warp per (window, head): q/k/v (N x 32 bf16 each, zero-padded to ROWS = 64 / 144 rows) staged in swizzled
// shared memory with cp.async; S = q k^T on mma.sync m16n8k16 (ROWS / 16 query tiles x ROWS / 8 key tiles), then
// + relative-position bias[h] (+ -100 between tokens of different shift regions), fp32 softmax in
// registers, P (bf16) V on mma.sync, O / l correctly rounded (RowNorm), 4-byte stores of the 16 x 32 output tile.
#include "attention_mma.cuh"
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kWDH = 32;      // head dim
constexpr int kWWarps = 4;

// 64-byte rows: 4 chunks of 16 B; XOR with (row >> 1) & 3 spreads 8 consecutive rows over all banks.
__device__ __forceinline__ uint32_t wswz(int row, int chunk) {
  return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4));
}

template <int ROWS, bool kPadded>   // padded tokens per window: 64 or 144
__global__ void __launch_bounds__(kWWarps * 32)
window_attention_bf16_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                             const float* __restrict__ bias, const int* __restrict__ row_map,
                             const int* __restrict__ labels, const unsigned long long* __restrict__ maskbits,
                             long total_pairs, int nw_img, int N, int H, float scale) {
  static_assert(!kPadded || ROWS == 64, "the padded bias / mask-bit format is 64 x 64");
  constexpr int kWRows = ROWS;
  constexpr int kTileBytes = ROWS * kWDH * 2;   // 4 / 9 KB per q / k / v tile
  constexpr int NT = ROWS / 8;                  // key tiles of 8
  extern __shared__ __align__(128) uint8_t smem[];  // kWWarps * 3 * kTileBytes
  __shared__ int s_rows[kWWarps][kWRows];
  __shared__ int s_lab[kWWarps][kWRows];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long pair = (long)blockIdx.x * kWWarps + warp;
  if (pair >= total_pairs) return;
  const int h = (int)(pair % H);
  const long w = pair / H;                 // global window index
  const int wi = (int)(w % nw_img);        // window inside its image
  const long img = w / nw_img;
  const int L = nw_img * N;
  const long ld = 3L * H * kWDH;
  const uint32_t sQ = smem_u32(smem) + (uint32_t)(warp * 3) * kTileBytes;
  const uint32_t sK = sQ + kTileBytes, sV = sK + kTileBytes;

  for (int p = lane; p < kWRows; p += 32) {
    s_rows[warp][p] = p < N ? row_map[wi * N + p] : 0;
    s_lab[warp][p] = (p < N && labels != nullptr) ? labels[wi * N + p] : 0;
  }
  __syncwarp();
  const __nv_bfloat16* base = qkv + img * L * ld + (long)h * kWDH;
  for (int idx = lane; idx < kWRows * 4; idx += 32) {
    const int r = idx >> 2, c = idx & 3;
    const bool valid = r < N;
    const __nv_bfloat16* src = base + (long)s_rows[warp][r] * ld + c * 8;
    const uint32_t off = wswz(r, c);
    cp_async_16(sQ + off, src, valid);
    cp_async_16(sK + off, src + H * kWDH, valid);
    cp_async_16(sV + off, src + 2 * H * kWDH, valid);
  }
  cp_async_commit();

  const int g = lane >> 2, t = lane & 3;
  const int bias_ld = kPadded ? 64 : N;
  const float* bias_h = bias + (long)h * bias_ld * bias_ld;
  cp_async_wait<0>();
  __syncwarp();

  const int mtiles = (N + 15) >> 4;
  const int ntiles = (N + 7) >> 3;   // key tiles with at least one valid key (<= NT)

#pragma unroll 1
  for (int mt = 0; mt < mtiles; ++mt) {
    uint32_t qf[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int row = mt * 16 + (lane & 15);
      const int chunk = ks * 2 + (lane >> 4);
      ldmatrix_x4(sQ + wswz(row, chunk), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
    float s[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      if (nt < ntiles) {
        const int row = nt * 8 + (lane & 7);
        const int chunk = lane >> 3;
        uint32_t k0, k1, k2, k3;
        ldmatrix_x4(sK + wswz(row, chunk), k0, k1, k2, k3);
        mma_bf16_16816(s[nt], qf[0], k0, k1);
        mma_bf16_16816(s[nt], qf[1], k2, k3);
      }
    }
    // logits = scale * qk + bias + mask; rows g and g+8 of this tile
    const int r0 = mt * 16 + g, r1 = r0 + 8;
    const int lab0 = s_lab[warp][r0], lab1 = s_lab[warp][r1];
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = nt * 8 + 2 * t + (e & 1);
        const int row = (e >> 1) ? r1 : r0;
        float val = -INFINITY;
        if (key < N && row < N) {
          val = fmaf(s[nt][e], scale, __ldg(bias_h + (long)row * bias_ld + key));   // L1 / L2-resident table
          if constexpr (kPadded) {
            if (maskbits != nullptr && ((__ldg(maskbits + wi * 64 + row) >> key) & 1ull)) val += -100.0f;
          } else {
            if (labels != nullptr && s_lab[warp][key] != ((e >> 1) ? lab1 : lab0)) val += -100.0f;
          }
        } else if (key < N) {
          val = 0.f;  // padded query rows: keep finite, result is discarded
        }
        s[nt][e] = val * kLog2e;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
      }
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) mx[r] = quad_max(mx[r]);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nt][e] - mx[e >> 1]);
        s[nt][e] = pv;
        sum[e >> 1] += pv;
      }
    }
    const RowNorm nrm[2] = {RowNorm(sum[0]), RowNorm(sum[1])};
    float o[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    pv_bf16(o, s, ntiles, lane, [&](int row, int chunk) { return sV + wswz(row, chunk); });
    __nv_bfloat16* obase = out + img * L * ((long)H * kWDH) + (long)h * kWDH;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      if (r0 < N)
        *reinterpret_cast<uint32_t*>(obase + (long)s_rows[warp][r0] * ((long)H * kWDH) + nt * 8 + 2 * t) =
            pack_bf16x2(nrm[0](o[nt][0]), nrm[0](o[nt][1]));
      if (r1 < N)
        *reinterpret_cast<uint32_t*>(obase + (long)s_rows[warp][r1] * ((long)H * kWDH) + nt * 8 + 2 * t) =
            pack_bf16x2(nrm[1](o[nt][2]), nrm[1](o[nt][3]));
    }
  }
}

template <int ROWS, bool kPadded>
int launch_window_attention(const void* qkv, void* out, const float* bias, const int* row_map, const int* labels,
                            const unsigned long long* maskbits, int B, int nw_img, int N, int H, float scale,
                            cudaStream_t stream) {
  const long pairs = (long)B * nw_img * H;
  const unsigned grid = (unsigned)((pairs + kWWarps - 1) / kWWarps);
  constexpr int smem = kWWarps * 3 * ROWS * kWDH * 2;   // 48 KB / 108 KB (two CTAs per SM)
  auto kernel = window_attention_bf16_kernel<ROWS, kPadded>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, smem, attr_devs));
  kernel<<<grid, kWWarps * 32, smem, stream>>>(reinterpret_cast<const __nv_bfloat16*>(qkv),
                                               reinterpret_cast<__nv_bfloat16*>(out), bias, row_map, labels, maskbits,
                                               pairs, nw_img, N, H, scale);
  TFIMM_LAUNCH_OK("window_attention_bf16_kernel");
  return kOk;
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_window_attention_bf16(const void* qkv, void* out, const float* bias, const int* row_map,
                                     const int* labels, int B, int nw_img, int N, int H, int dh, float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && nw_img > 0 && N > 0 && H > 0, "window_attention: bad shape");
  TFIMM_CHECK_ARG(bias != nullptr && row_map != nullptr, "window_attention: bias and row_map are required");
  if (dh != kWDH || N > 144) {
    set_last_error("window_attention: bf16 kernel supports head_dim 32 and <= 144 tokens per window (got dh=%d N=%d)", dh, N);
    return kUnsupported;
  }
  if (N <= 64)
    return launch_window_attention<64, false>(qkv, out, bias, row_map, labels, nullptr, B, nw_img, N, H, scale, stream);
  return launch_window_attention<144, false>(qkv, out, bias, row_map, labels, nullptr, B, nw_img, N, H, scale, stream);
}

// bias_pad: [H][64][64] fp32 (rows / columns beyond N are ignored); maskbits: [nw_img][64] uint64, bit j of entry
// (wi, i) set when tokens i and j of window wi lie in different shift regions (null for unshifted blocks).
int tfimm_b200_window_attention_tc_bf16(const void* qkv, void* out, const float* bias_pad, const int* row_map,
                                        const void* maskbits, int B, int nw_img, int N, int H, int dh, float scale,
                                        void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && nw_img > 0 && N > 0 && H > 0, "window_attention: bad shape");
  TFIMM_CHECK_ARG(bias_pad != nullptr && row_map != nullptr, "window_attention: bias and row_map are required");
  if (dh != kWDH || N > 52) {
    set_last_error("window_attention: the padded-table entry takes head_dim 32 and <= 52 tokens per window (got dh=%d N=%d)",
                   dh, N);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(bias_pad) & 15u) == 0,
                  "window_attention: qkv / out / bias must be 16-byte aligned");
  return launch_window_attention<64, true>(qkv, out, bias_pad, row_map, nullptr,
                                           static_cast<const unsigned long long*>(maskbits), B, nw_img, N, H, scale,
                                           stream);
}

}  // extern "C"
