// Dense layer with a SHORT contraction (K <= 64): a streaming kernel, not a tile pipeline.
//
//     C[M,N] = act(A[M,K] @ W[N,K]^T + bias[N]) + residual[M,N]        bf16 in / bf16 out, fp32 accumulate
//
// Call sites: the 1x1 convolutions of EfficientNet's first stages and stems -- (K, N) = (27->32, 48), (48, 24),
// (24, 144), (32, 192), (56, 336) with M up to 9.2 M pixels at 380 px -- and the patch-embedding GEMMs (K = 48) of
// Swin / ConvNeXt (tfimm/architectures/efficientnet_blocks.py:412-434, layers/transformers.py:131-139).  At K <= 64
// the work is ~40 flop per byte: HBM-bound, with the activation (one MUFU.EX2 per element) as the second term.  A tile
// pipeline (TMA -> tensor core -> epilogue) pays a barrier round trip per 128 x 64 tile on such shapes.  Here the whole weight matrix sits in shared memory for the life of the CTA, warps stream 16-row slices of A through
// cp.async double buffers, multiply on mma.sync (HMMA -- the tensor pipe is idle either way at this intensity) and
// store their fragments directly; occupancy (up to 24 warps / SM), not a pipeline, hides the latency.
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kSkM = 128;        // rows per CTA step (8 warps x 16)
constexpr int kSkWarps = 8;
constexpr int kSkNMax = 512;
constexpr int kSkRowBytes = 128; // smem pitch of A / W rows: 64 bf16, zero-padded past K, 16-byte chunks XOR-swizzled

__device__ __forceinline__ uint32_t sk_off(int row, int chunk) {
  return (uint32_t)(row * kSkRowBytes + ((chunk ^ (row & 7)) << 4));
}

__global__ void __launch_bounds__(kSkWarps * 32, 3)
gemm_bf16_skinny_kernel(const __nv_bfloat16* __restrict__ A, int lda, const __nv_bfloat16* __restrict__ W, int ldw,
                        const float* __restrict__ bias, const __nv_bfloat16* __restrict__ residual, int ldr,
                        __nv_bfloat16* __restrict__ C, int ldc, int M, int N, int K, int act, int n_rows_w,
                        const float* __restrict__ gate, int rows_per_img, int imgs) {
  extern __shared__ __align__(128) uint8_t smem[];
  // [W: n_rows_w x 128 B][A buffers: 2 x 128 x 128 B][bias: n_rows_w floats]
  const uint32_t sW = smem_u32(smem);
  const uint32_t sA = sW + (uint32_t)n_rows_w * kSkRowBytes;
  float* s_bias = reinterpret_cast<float*>(smem + (size_t)n_rows_w * kSkRowBytes + 2 * kSkM * kSkRowBytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kchunks = (K + 7) >> 3;           // 16-byte chunks per row that hold data
  const int ksteps = (K + 15) >> 4;           // mma k-steps (<= 4)
  const int num_tiles = (M + kSkM - 1) / kSkM;

  // weights and bias: once per CTA
  for (int idx = tid; idx < n_rows_w * 8; idx += kSkWarps * 32) {
    const int r = idx >> 3, c = idx & 7;
    const bool valid = r < N && c < kchunks;
    cp_async_16(sW + sk_off(r, c), W + (long)(valid ? r : 0) * ldw + (valid ? c : 0) * 8, valid);
  }
  for (int n = tid; n < n_rows_w; n += kSkWarps * 32) s_bias[n] = (bias != nullptr && n < N) ? bias[n] : 0.f;
  auto load_a = [&](int tile, int buf) {
    const long row0 = (long)tile * kSkM;
    for (int idx = tid; idx < kSkM * 8; idx += kSkWarps * 32) {
      const int r = idx >> 3, c = idx & 7;
      const bool valid = row0 + r < M && c < kchunks;
      cp_async_16(sA + (uint32_t)buf * (kSkM * kSkRowBytes) + sk_off(r, c),
                  A + (valid ? (row0 + r) * (long)lda + c * 8 : 0), valid);
    }
  };
  int tile = blockIdx.x;
  if (tile < num_tiles) load_a(tile, 0);
  cp_async_commit();

  const int g = lane >> 2, t = lane & 3;
  int it = 0;
  for (; tile < num_tiles; tile += gridDim.x, ++it) {
    const int buf = it & 1;
    if (tile + (int)gridDim.x < num_tiles) load_a(tile + gridDim.x, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();      // this tile's A (and, the first time, W) has landed
    __syncthreads();
    const uint32_t a_base = sA + (uint32_t)buf * (kSkM * kSkRowBytes);
    const long row0 = (long)tile * kSkM + warp * 16;
    if (row0 < M) {
      uint32_t af[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (ks < ksteps) {
          const int row = warp * 16 + (lane & 15);
          ldmatrix_x4(a_base + sk_off(row, ks * 2 + (lane >> 4)), af[ks][0], af[ks][1], af[ks][2], af[ks][3]);
        }
      }
      if (gate != nullptr) {
        // squeeze-excite gate on the A fragments: element (row, k) *= gate[row / rows_per_img][k], rounded to bf16 like
        // the separate scale pass.  A lane holds rows g, g + 8 and k = 16 ks + 2 t + {0, 1, 8, 9} of every k-step.
        long i0 = (row0 + g) / rows_per_img, i1 = (row0 + g + 8) / rows_per_img;
        i0 = i0 < imgs ? i0 : imgs - 1;
        i1 = i1 < imgs ? i1 : imgs - 1;
        const float* g0 = gate + i0 * K + 2 * t;
        const float* g1 = gate + i1 * K + 2 * t;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          if (ks < ksteps) {
            const int k = ks * 16;
            const bool lo_ok = k + 2 * t < K, hi_ok = k + 8 + 2 * t < K;   // K % 8 == 0: a pair is in or out as a whole
            const float2 z = make_float2(0.f, 0.f);
            const float2 a_lo = lo_ok ? __ldg(reinterpret_cast<const float2*>(g0 + k)) : z;
            const float2 a_hi = hi_ok ? __ldg(reinterpret_cast<const float2*>(g0 + k + 8)) : z;
            const float2 b_lo = lo_ok ? __ldg(reinterpret_cast<const float2*>(g1 + k)) : z;
            const float2 b_hi = hi_ok ? __ldg(reinterpret_cast<const float2*>(g1 + k + 8)) : z;
            float2 x;
            x = unpack_bf16x2(af[ks][0]); af[ks][0] = pack_bf16x2(x.x * a_lo.x, x.y * a_lo.y);
            x = unpack_bf16x2(af[ks][1]); af[ks][1] = pack_bf16x2(x.x * b_lo.x, x.y * b_lo.y);
            x = unpack_bf16x2(af[ks][2]); af[ks][2] = pack_bf16x2(x.x * a_hi.x, x.y * a_hi.y);
            x = unpack_bf16x2(af[ks][3]); af[ks][3] = pack_bf16x2(x.x * b_hi.x, x.y * b_hi.y);
          }
        }
      }
      const bool r0_ok = row0 + g < M, r1_ok = row0 + g + 8 < M;
      __nv_bfloat16* c0 = C + (row0 + g) * (long)ldc + 2 * t;
      __nv_bfloat16* c1 = c0 + 8 * (long)ldc;
      const __nv_bfloat16* q0 = residual != nullptr ? residual + (row0 + g) * (long)ldr + 2 * t : nullptr;
      const __nv_bfloat16* q1 = residual != nullptr ? q0 + 8 * (long)ldr : nullptr;
      // one 8-column tile at a time: 16 x 8 results = one group of four per lane (rows g, g+8 x columns 2t, 2t+1),
      // written as two 4-byte stores (eight rows x 16 contiguous bytes per instruction; L2 merges the sectors)
#pragma unroll 2
      for (int n0 = 0; n0 < N; n0 += 8) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        const int row = n0 + (lane & 7);
        {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(sW + sk_off(row, lane >> 3), b0, b1, b2, b3);
          mma_bf16_16816(acc, af[0], b0, b1);
          if (ksteps > 1) mma_bf16_16816(acc, af[1], b2, b3);
        }
        if (ksteps > 2) {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(sW + sk_off(row, 4 + (lane >> 3)), b0, b1, b2, b3);
          mma_bf16_16816(acc, af[2], b0, b1);
          if (ksteps > 3) mma_bf16_16816(acc, af[3], b2, b3);
        }
        const float2 bb = *reinterpret_cast<const float2*>(s_bias + n0 + 2 * t);
        uint64_t lo = pack2(acc[0] + bb.x, acc[1] + bb.y), hi = pack2(acc[2] + bb.x, acc[3] + bb.y);
        if (act == kActSwish) swish4(lo, hi);
        else if (act == kActGelu) gelu4(lo, hi);
        else if (act != kActNone) {
          float a0, a1, a2, a3;
          unpack2(lo, a0, a1);
          unpack2(hi, a2, a3);
          lo = pack2(apply_act<false>(a0, act), apply_act<false>(a1, act));
          hi = pack2(apply_act<false>(a2, act), apply_act<false>(a3, act));
        }
        float a0, a1, a2, a3;
        unpack2(lo, a0, a1);
        unpack2(hi, a2, a3);
        if (residual != nullptr) {   // may alias C: each element is read and written by the same thread
          if (r0_ok) {
            const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q0 + n0));
            a0 += r.x;
            a1 += r.y;
          }
          if (r1_ok) {
            const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q1 + n0));
            a2 += r.x;
            a3 += r.y;
          }
        }
        if (r0_ok) *reinterpret_cast<uint32_t*>(c0 + n0) = pack_bf16x2(a0, a1);
        if (r1_ok) *reinterpret_cast<uint32_t*>(c1 + n0) = pack_bf16x2(a2, a3);
      }
    }
    __syncthreads();   // every warp is done with A buffer `buf` before the next iteration's prefetch overwrites it
  }
  cp_async_wait<0>();
}

}  // namespace

// Returns kUnsupported (without setting an error) for shapes outside this kernel: the caller uses the wgmma path.
int gemm_bf16_skinny(const void* A, int lda, const void* W, int ldw, const float* bias, const void* residual, int ldr,
                     void* C, int ldc, int M, int N, int K, int act, cudaStream_t stream, const float* gate,
                     int rows_per_img, int imgs) {
  if (K > 64 || K % 8 != 0 || N % 8 != 0 || N > kSkNMax || M < 4096) return kUnsupported;
  if (lda % 8 != 0 || ldw % 8 != 0 || ldc % 8 != 0) return kUnsupported;
  if (residual != nullptr && (ldr % 2 != 0 || (reinterpret_cast<uintptr_t>(residual) & 3u))) return kUnsupported;
  if ((reinterpret_cast<uintptr_t>(A) & 15u) || (reinterpret_cast<uintptr_t>(W) & 15u) ||
      (reinterpret_cast<uintptr_t>(C) & 15u) || (bias != nullptr && (reinterpret_cast<uintptr_t>(bias) & 7u)))
    return kUnsupported;
  const int n_rows_w = (N + 7) / 8 * 8;
  const int smem = n_rows_w * kSkRowBytes + 2 * kSkM * kSkRowBytes + n_rows_w * 4;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(gemm_bf16_skinny_kernel, kSkNMax * kSkRowBytes + 2 * kSkM * kSkRowBytes + kSkNMax * 4,
                                     attr_devs));
  const int tiles = (M + kSkM - 1) / kSkM;
  const int per_sm = smem <= 56 * 1024 ? 3 : 2;   // co-resident CTAs (shared memory / 3 x 256 threads)
  const int max_ctas = per_sm * sm_count();
  const int grid = tiles < max_ctas ? tiles : max_ctas;
  gemm_bf16_skinny_kernel<<<grid, kSkWarps * 32, smem, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(A), lda, reinterpret_cast<const __nv_bfloat16*>(W), ldw, bias,
      reinterpret_cast<const __nv_bfloat16*>(residual), ldr, reinterpret_cast<__nv_bfloat16*>(C), ldc, M, N, K, act,
      n_rows_w, gate, rows_per_img, imgs);
  TFIMM_LAUNCH_OK("gemm_bf16_skinny_kernel");
  return kOk;
}

}  // namespace tfimm
