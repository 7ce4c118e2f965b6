// Fused MLP block of the narrow stages on sm_90a:
//
//     out = residual + gamma * (act(A @ W1^T + b1) @ W2^T + b2)          A:[M,C] bf16, out / residual fp32
//
// Replaces MLP.call (tfimm/layers/transformers.py:208-214) + layer scale + shortcut in ConvNeXtBlock.call
// (tfimm/architectures/convnext.py:219-228) and the MLP half of SwinTransformerBlock.call (swin.py:315-318) for
// C in {96, 128, 192, 256}.  The [M, hidden] activations never reach HBM.
//
// One CTA per 128 rows, two warpgroups of 64 rows each.  Thread 0 also issues the TMA loads: the CTA's A rows once
// (resident), then per hidden chunk of 64 the W1 rows [64][C] and the W2 columns [C][64] into a two-stage ring, the
// next chunk's as soon as both warpgroups have released its stage (no separate producer warp: a ninth warp would cap
// the register file at 168 per thread, and the C = 256 accumulators need more).  Per chunk:
//                 fc1  wgmma m64n64k16 over C (A and W1 from smem) -> 64 x 64 fp32 in registers
//                 + b1, activation, rounded to bf16 -- the accumulator fragment IS the register A-operand fragment of
//                 the next product, so the hidden chunk goes straight back into the tensor core:
//                 fc2  wgmma m64nCk16 (A from registers, W2 from smem) accumulating 64 x C fp32 over the chunks
//               then + b2, * gamma, + residual, fp32 stores (gemm_epilogue.cuh).
// The rounding points are those of the two-GEMM form (bf16 hidden, fp32 accumulation in ascending k).
#include "gemm_epilogue.cuh"
#include "wgmma.cuh"

namespace tfimm {
namespace {

constexpr int kMlpRows = 128;
constexpr int kHC = 64;   // hidden chunk
constexpr int kMlpStages = 2;
constexpr int kMlpThreads = 256;

template <int C>
struct MlpCfg {
  static constexpr int kKB = (C + 63) / 64;               // 64-wide k-blocks of the fc1 contraction
  static constexpr int kABytes = kKB * kMlpRows * 128;    // resident A: kKB boxes of [128 rows][64]
  static constexpr int kW1Bytes = kKB * kHC * 128;        // W1 chunk: kKB boxes of [64 rows][64]
  static constexpr int kW2Bytes = C * 128;                // W2 chunk: [C rows][64]
  static constexpr int kStageBytes = kW1Bytes + kW2Bytes;
  static constexpr int kSmemBytes = kABytes + kMlpStages * kStageBytes + (1 + 2 * kMlpStages) * 8 + 1024;
};

template <int C>
__global__ void __launch_bounds__(kMlpThreads, 1)
mlp_fused_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w1,
                       const __grid_constant__ CUtensorMap tmap_w2, const float* __restrict__ b1, int hidden, int act,
                       const GemmParams p) {
  using Cfg = MlpCfg<C>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = smem_base;
  const uint32_t sStages = sA + Cfg::kABytes;
  const uint32_t bars = sStages + kMlpStages * Cfg::kStageBytes;
  const uint32_t a_bar = bars;
  auto full_bar = [&](int s) { return bars + 8u * (1 + s); };
  auto empty_bar = [&](int s) { return bars + 8u * (1 + kMlpStages + s); };
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x;
  const int n_chunks = hidden / kHC;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_w1);
    prefetch_tmap(&tmap_w2);
    mbar_init(a_bar, 1);
    for (int s = 0; s < kMlpStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  // chunk j goes to stage j % kMlpStages; its load waits until both warpgroups have released chunk j - kMlpStages
  auto load_chunk = [&](int j) {
    const int s = j % kMlpStages;
    if (j >= kMlpStages) mbar_wait(empty_bar(s), (uint32_t)((j / kMlpStages - 1) & 1));
    const uint32_t sw1 = sStages + s * Cfg::kStageBytes, sw2 = sw1 + Cfg::kW1Bytes;
    mbar_expect_tx(full_bar(s), Cfg::kStageBytes);
    for (int kb = 0; kb < Cfg::kKB; ++kb) tma_load_2d(sw1 + kb * (kHC * 128), &tmap_w1, full_bar(s), kb * 64, j * kHC);
    tma_load_2d(sw2, &tmap_w2, full_bar(s), j * kHC, 0);
  };
  if (threadIdx.x == 0) {
    mbar_expect_tx(a_bar, Cfg::kABytes);
    for (int kb = 0; kb < Cfg::kKB; ++kb)
      tma_load_2d(sA + kb * (kMlpRows * 128), &tmap_a, a_bar, kb * 64, m_blk * kMlpRows);
    for (int j = 0; j < kMlpStages && j < n_chunks; ++j) load_chunk(j);
  }

  const int wg = warp_idx >> 2;
  const bool releaser = (threadIdx.x & 127) == 0;
  float acc2[C / 2];
#pragma unroll
  for (int i = 0; i < C / 2; ++i) acc2[i] = 0.f;
  mbar_wait(a_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
#pragma unroll 1
  for (int j = 0; j < n_chunks; ++j) {
    mbar_wait(full_bar(stage), phase);
    const uint32_t sw1 = sStages + stage * Cfg::kStageBytes, sw2 = sw1 + Cfg::kW1Bytes;
    float acc1[kHC / 2];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < Cfg::kKB; ++kb) {
      const uint64_t da = gmma_desc_k_sw128(sA + kb * (kMlpRows * 128) + wg * (64 * 128));
      const uint64_t db = gmma_desc_k_sw128(sw1 + kb * (kHC * 128));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (kb * 64 + k * 16 >= C) break;   // C = 96 / 192: the last k-block is half used
        wgmma_ss<kHC>(acc1, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    // hidden = bf16(act(acc1 + b1)), packed as the m64k16 A fragments of the four k16 steps of fc2
    uint32_t a[kHC / 16][4];
#pragma unroll
    for (int s = 0; s < kHC / 16; ++s) {
      uint64_t v[4];
#pragma unroll
      for (int q = 0; q < 2; ++q) {   // 8-column group 2 s + q: rows r and r + 8
        const int n = j * kHC + s * 16 + q * 8 + 2 * (lane & 3);
        const float2 b = __ldg(reinterpret_cast<const float2*>(b1 + n));
        const uint64_t bb = pack2(b.x, b.y);
        v[2 * q] = add2(pack2(acc1[8 * s + 4 * q], acc1[8 * s + 4 * q + 1]), bb);
        v[2 * q + 1] = add2(pack2(acc1[8 * s + 4 * q + 2], acc1[8 * s + 4 * q + 3]), bb);
      }
      apply_act_pairs(v, act);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float lo, hi;
        unpack2(v[e], lo, hi);
        a[s][e] = pack_bf16x2(lo, hi);
      }
    }
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < kHC / 16; ++s)
      wgmma_rs<C>(acc2, a[s], gmma_desc_k_sw128(sw2) + (uint64_t)(2 * s), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (releaser) mbar_arrive(empty_bar(stage));
    if (threadIdx.x == 0 && j + kMlpStages < n_chunks) load_chunk(j + kMlpStages);
    if (++stage == kMlpStages) { stage = 0; phase ^= 1u; }
  }
  epilogue_frag<float, C>(p, acc2, m_blk, 0, wg * 64);
}

template <int C>
int launch_mlp(const void* A, int lda, const void* W1, int ldw1, const float* b1, const void* W2, int ldw2, int hidden,
               int act, const GemmParams& p, cudaStream_t stream) {
  using Cfg = MlpCfg<C>;
  CUtensorMap ta, tw1, tw2;
  int st;
  if ((st = make_tmap_2d(&ta, A, kBF16, p.M, C, lda, kMlpRows, 64, "A")) != kOk) return st;
  if ((st = make_tmap_2d(&tw1, W1, kBF16, hidden, C, ldw1, kHC, 64, "W1")) != kOk) return st;
  if ((st = make_tmap_2d(&tw2, W2, kBF16, C, hidden, ldw2, C, 64, "W2")) != kOk) return st;
  auto kernel = mlp_fused_wgmma_kernel<C>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Cfg::kSmemBytes, attr_devs));
  const int tiles = (p.M + kMlpRows - 1) / kMlpRows;
  kernel<<<tiles, kMlpThreads, Cfg::kSmemBytes, stream>>>(ta, tw1, tw2, b1, hidden, act, p);
  TFIMM_LAUNCH_OK("mlp_fused_wgmma_kernel");
  return kOk;
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

// Returns kUnsupported for shapes outside the kernel (the caller then runs the two GEMMs).
int tfimm_b200_mlp_bf16(const void* A, int lda, const void* W1, int ldw1, const float* b1, const void* W2, int ldw2,
                        const float* b2, const float* gamma, const void* residual, int ldr, void* out, int ldc, int M,
                        int C, int H, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  if ((C != 96 && C != 128 && C != 192 && C != 256) || H % 128 != 0 || H < 256 || M < 1) {
    set_last_error("mlp_fused: needs C in {96, 128, 192, 256} and hidden %% 128 == 0, >= 256 (got C=%d hidden=%d)", C, H);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG(b1 != nullptr && (reinterpret_cast<uintptr_t>(b1) & 7u) == 0, "mlp_fused: b1 must be 8-byte aligned");
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15u) == 0 && ldc % 4 == 0 &&
                      (residual == nullptr || ((reinterpret_cast<uintptr_t>(residual) & 15u) == 0 && ldr % 4 == 0)),
                  "mlp_fused: out / residual must be 16-byte aligned with row strides a multiple of 4");
  GemmParams p{};
  p.M = M;
  p.N = C;
  p.K = H;
  p.bias = b2;
  p.gamma = gamma;
  p.act = kActNone;
  p.has_res = residual != nullptr;
  p.c = out;
  p.res = residual;
  p.ldc = ldc;
  p.ldr = ldr;
  switch (C) {
    case 96: return launch_mlp<96>(A, lda, W1, ldw1, b1, W2, ldw2, H, act, p, stream);
    case 128: return launch_mlp<128>(A, lda, W1, ldw1, b1, W2, ldw2, H, act, p, stream);
    case 192: return launch_mlp<192>(A, lda, W1, ldw1, b1, W2, ldw2, H, act, p, stream);
    default: return launch_mlp<256>(A, lda, W1, ldw1, b1, W2, ldw2, H, act, p, stream);
  }
}

}  // extern "C"
