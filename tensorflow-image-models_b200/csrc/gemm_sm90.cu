// Dense contraction for the tfimm forward path on sm_90a:
//
//     C[M,N] = residual[M,N] + gamma[N] * act(A[M,K] @ W[N,K]^T + bias[N])
//
// This single kernel replaces every tf.keras.layers.Dense and 1x1 Conv2D the
// reference calls on the hot path (qkv/proj: tfimm/architectures/vit.py:142-146,
// swin.py:124-128; fc1/fc2: tfimm/layers/transformers.py:192-205; heads:
// vit.py:364-368, convnext.py:356-360; 1x1 convs: efficientnet_blocks.py:412-434,
// resnet.py:220-248) plus the patchify convolutions once their input has been
// gathered (layers/transformers.py:131-139, convnext.py:259-266,319-326).
//
// Design (one 128 x BLOCK_N output tile per CTA, warp-specialised):
//   warps 0..7  two consumer warpgroups, 64 tile rows each: wgmma m64 x BLOCK_N x k16 from the swizzled smem ring,
//               fp32 accumulators in registers, one wgmma group kept in flight (the stage of the group before it is
//               released as soon as it retires); then the epilogue (gemm_epilogue.cuh): staged through shared memory
//               with TMA residual load and output store (plain bf16 GEMM, BLOCK_N <= 128), or from the fragments
//   warp 8      TMA producer: A/W tiles -> 128B-swizzled smem ring (mbarrier full/empty); the residual tile of the
//               staged epilogue
//   warps 9..12 (A-transform instances only) rewrite the A tile in smem before the MMA reads it: the squeeze-excite
//               gate (bf16), or the TF32 rounding of fp32 activations (precision="tf32")
//
// gemm_persistent_kernel is the plain bf16 GEMM at 128 x 256 tiles with one CTA per SM walking the tiles (see there).
//
// Two more instances share the ring, barriers, producer/consumer split and epilogue plumbing (GemmMode):
//   kModeToken   token mixing, out[b][m][c] = epi(sum_n Wt[m][n] X[b][n][c]): the Dense layer that MLP-Mixer, ResMLP
//                and gMLP apply along the token axis of a transposed activation.  B is X where it is stored, read
//                MN-major (channels contiguous) as 3-D TMA boxes {64 channels, 64 tokens, 1 image} and fed to wgmma with
//                imm-trans-b = 1; the token axis is a bounded TMA dimension, so the K tail reads zeros and no tile
//                reads the next image.  Epilogue: epilogue_token (row bias, GLU on row pairs, multiplier).
//   kModeGluCols a plain GEMM whose epilogue writes value * act(gate) of interleaved column pairs at half width.
//
// Operands: bf16 (wgmma k16), or fp32 rounded to TF32 (wgmma k8).  Either way a tile row is 128 bytes -- one
// SWIZZLE_128B span of 64 bf16 or 32 fp32 contraction indices -- so stage bytes, descriptors and the 32-byte k-step are
// the same; only the TMA element type, the k-block width and the MMA instruction differ.
#include <type_traits>

#include "gemm_epilogue.cuh"
#include "wgmma.cuh"

namespace tfimm {

namespace {

constexpr int kBlockM = 128;
constexpr int kRowBytes = 128;   // one 128-byte swizzle span per tile row
constexpr int kConsumerThreads = 256;
constexpr int kProducerWarp = kConsumerThreads / 32;
constexpr int kNumGateWarps = 4;   // A-transform instances only

// What the A-transform warps do to each A tile between the TMA load and the MMA.
enum ATransform : int {
  kANone = 0,   // nothing: the consumers wait on the TMA barrier directly
  kAGate = 1,   // bf16 A: x * gate[image][k] in fp32, rounded back to bf16 (squeeze-excite)
  kATf32 = 2,   // fp32 A: cvt.rna.tf32 of every element (precision="tf32")
};
enum GemmMode : int { kModeGemm = 0, kModeToken = 1, kModeGluCols = 2 };

template <int AX>
using OperandT = std::conditional_t<AX == kATf32, float, __nv_bfloat16>;
template <int AX>
constexpr int block_k() { return kRowBytes / (int)sizeof(OperandT<AX>); }   // 64 bf16 / 32 fp32
template <int AX>
constexpr int dtype_code() { return AX == kATf32 ? kF32 : kBF16; }

// STAGED (plain bf16 GEMM at BLOCK_N 64 / 128, epilogue_staged): after the ring, a 128 x BLOCK_N OutT tile that takes
// the residual by TMA during the mainloop and holds the result for the TMA store, then the tile's bias and gamma.
// Shared memory per CTA (ring + tile + bias / gamma + barriers + alignment slack; the SM reserves 1 KB more per CTA,
// and has 228 KB in all):
//   BLOCK_N = 64:  4 stages = 96 KB, or 3 stages = 72 KB + 16 / 32 KB (bf16 / fp32 tile) when STAGED: two CTAs per SM
//                  either way (4 stages + a 16 KB tile would need 2 x 114.6 KB with the reserved 1 KB)
//   BLOCK_N = 128: 4 stages = 128 KB, + 32 / 64 KB when STAGED: one CTA per SM
//   BLOCK_N = 256: 4 stages = 192 KB, no room for a tile: fragment epilogue only
template <int BLOCK_N, typename OutT = float, bool STAGED = false>
struct GemmCfg {
  static constexpr int kABytes = kBlockM * kRowBytes;
  static constexpr int kBBytes = BLOCK_N * kRowBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = STAGED && BLOCK_N == 64 ? 3 : 4;
  static constexpr int kOutBytes = STAGED ? kBlockM * BLOCK_N * (int)sizeof(OutT) : 0;
  static constexpr int kVecBytes = STAGED ? 2 * BLOCK_N * 4 : 0;   // bias, gamma
  static constexpr int kNumBarriers = 3 * kStages + 1;   // full, empty, ready (A-transform instances), residual
  static constexpr int kSmemBytes =
      kStages * kStageBytes + kOutBytes + kVecBytes + kNumBarriers * 8 + 1024 /*alignment slack*/;
  static_assert(!STAGED || BLOCK_N <= 128, "the staged epilogue's tile does not fit next to a 256-wide ring");
};

// B operand descriptor: K-major, or MN-major for token mixing; one k16 step is 32 bytes (+2) or 16 MN-major rows (+128).
template <bool kMN>
__device__ __forceinline__ uint64_t gmma_desc_b(uint32_t smem_addr) {
  if constexpr (kMN) return gmma_desc_mn_sw128(smem_addr);
  else return gmma_desc_k_sw128(smem_addr);
}
template <bool kMN>
constexpr int kDescStepB = kMN ? 128 : 2;

template <int BLOCK_N, int AX>
constexpr int gemm_threads() { return kConsumerThreads + 32 + (AX != kANone ? 32 * kNumGateWarps : 0); }

// STAGED: epilogue_staged, with the output (tmap_c) and residual (tmap_r) tensor maps; otherwise they are unused and
// the epilogue works from the fragments.
template <int BLOCK_N, typename OutT, int AX = kANone, int MODE = kModeGemm, bool STAGED = false>
__global__ void __launch_bounds__(gemm_threads<BLOCK_N, AX>(), (BLOCK_N == 64 && AX == kANone) ? 2 : 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r,
                  const GemmParams p) {
  static_assert(!STAGED || (AX == kANone && MODE == kModeGemm), "staged epilogue: plain bf16 GEMM only");
  using Cfg = GemmCfg<BLOCK_N, OutT, STAGED>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kBlockK = block_k<AX>();

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_tiles = smem_base;
  const uint32_t smem_out = smem_base + kStages * Cfg::kStageBytes;
  const uint32_t smem_vec = smem_out + Cfg::kOutBytes;
  const uint32_t smem_bars = smem_vec + Cfg::kVecBytes;
  auto full_bar = [&](int s) { return smem_bars + 8u * s; };
  auto empty_bar = [&](int s) { return smem_bars + 8u * (kStages + s); };
  auto ready_bar = [&](int s) { return smem_bars + 8u * (2 * kStages + s); };
  const uint32_t res_bar = smem_bars + 8u * (3 * kStages);
  float* const s_bias = reinterpret_cast<float*>(smem_raw + (smem_vec - smem_u32(smem_raw)));
  float* const s_gamma = s_bias + BLOCK_N;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp_idx == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    if constexpr (STAGED) {
      prefetch_tmap(&tmap_c);
      if (p.has_res) prefetch_tmap(&tmap_r);
      mbar_init(res_bar, 1);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
      mbar_init(ready_bar(s), 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  int m_blk, n_blk, img = 0;
  if constexpr (MODE == kModeToken) {
    // token mixing: image-major tile order, tiles never cross images
    const int img_tiles = ((p.M + kBlockM - 1) / kBlockM) * num_n_tiles;
    img = (int)blockIdx.x / img_tiles;
    const int tile = (int)blockIdx.x - img * img_tiles;
    m_blk = tile / num_n_tiles; n_blk = tile % num_n_tiles;
  } else {
    m_blk = blockIdx.x / num_n_tiles; n_blk = blockIdx.x % num_n_tiles;
  }
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;

  if (warp_idx == kProducerWarp) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
        const uint32_t sb = sa + Cfg::kABytes;
        mbar_expect_tx(full_bar(stage), Cfg::kStageBytes);
        if (STAGED || p.conv == 0) {
          tma_load_2d(sa, &tmap_a, full_bar(stage), kb * kBlockK, m_blk * kBlockM);
        } else {
          // implicit convolution: tap (ky, kx) and a kBlockK-channel slice of the input patch; padding = OOB zero fill
          const int tap = kb / p.cv_cblocks, cb = kb - tap * p.cv_cblocks;
          const int ky = tap / p.cv_ks, kx = tap - ky * p.cv_ks;
          const int tx = m_blk % p.cv_tiles_x, tyb = m_blk / p.cv_tiles_x;
          const int ty = tyb % p.cv_tiles_y, tb = tyb / p.cv_tiles_y;
          tma_load_4d(sa, &tmap_a, full_bar(stage), cb * kBlockK, tx * p.cv_pw * p.cv_stride + kx - p.cv_pad,
                      ty * p.cv_ph * p.cv_stride + ky - p.cv_pad, tb * p.cv_pb);
        }
        if constexpr (MODE == kModeToken) {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 64; ++i)
            tma_load_3d(sb + i * 8192, &tmap_b, full_bar(stage), n_blk * BLOCK_N + i * 64, kb * kBlockK, img);
        } else {
          tma_load_2d(sb, &tmap_b, full_bar(stage), kb * kBlockK, n_blk * BLOCK_N);
        }
        if constexpr (STAGED) {
          // the residual tile, right behind the first k-block: its latency hides under the mainloop.  Boxes wholly
          // past M or N are not loaded (the tile exists, so box (0, 0) always is).
          if (kb == 0 && p.has_res) {
            constexpr int kCols = staged_chunk_cols<OutT>(), kChunks = BLOCK_N / kCols;
            const int row0 = m_blk * kBlockM, col0 = n_blk * BLOCK_N;
            const int rows = p.M - row0 > 64 ? 2 : 1, chunks = min(kChunks, (p.N - col0 + kCols - 1) / kCols);
            mbar_expect_tx(res_bar, (uint32_t)(rows * chunks * kStagedBoxBytes));
            for (int h = 0; h < rows; ++h)
              for (int ch = 0; ch < chunks; ++ch)
                tma_load_2d(smem_out + (uint32_t)((h * kChunks + ch) * kStagedBoxBytes), &tmap_r, res_bar,
                            col0 + ch * kCols, row0 + 64 * h);
          }
        }
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (AX != kANone && warp_idx > kProducerWarp) {
    // ------------------------------ A-tile transform ------------------------------
    // Each of the four warps owns every fourth k-block (a whole 128-row tile), so four stages are being rewritten at
    // any time.  lane = one 16-byte chunk column x 32 rows 4 apart; a quarter-warp touches one whole 128-byte row (no
    // bank conflicts under the 128B swizzle).  After the rewrite: the proxy fence that makes the generic-proxy writes
    // visible to the tensor core's async-proxy reads, and one arrive on the stage's "ready" barrier.
    //   kAGate: x * gate in fp32, back as bf16 -- the rounding of the separate scale pass (csrc/conv.cu,
    //           scale_channels_kernel).  A chunk is 8 contraction indices; the gate values of a lane change only when
    //           its rows cross into the next image.
    //   kATf32: every element rounded to TF32 (cvt.rna), in place: elementwise, so the swizzle does not matter.
    const int wt = warp_idx - kProducerWarp - 1;
    const int c = lane & 7, r0 = lane >> 3;
    auto load_gate = [&](int img, int k0, float4& ga, float4& gb) {
      const float* g = p.a_scale + (long)img * p.K + k0;
      ga = __ldg(reinterpret_cast<const float4*>(g));
      gb = __ldg(reinterpret_cast<const float4*>(g + 4));
    };
    int img0 = 0;
    long bound0 = 0;
    if constexpr (AX == kAGate) {
      const long row_first = (long)m_blk * kBlockM + r0;
      long im0 = row_first / p.a_rows_per_img;
      im0 = im0 < p.a_imgs ? im0 : p.a_imgs - 1;            // rows past M are zero-filled: any gate row will do
      img0 = (int)im0;
      bound0 = (im0 + 1) * p.a_rows_per_img - (long)m_blk * kBlockM;   // first tile row of the next image
    }
    int stage = 0, turn = 0;   // stage / owner of the NEXT k-block
    uint32_t phase = 0;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      if (turn == wt) {
        if constexpr (AX == kATf32) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
#pragma unroll 1
          for (int b8 = 0; b8 < 4; ++b8) {
            uint4 u[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int r = r0 + 4 * (8 * b8 + i);
              asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                           : "=r"(u[i].x), "=r"(u[i].y), "=r"(u[i].z), "=r"(u[i].w)
                           : "r"(sa + (uint32_t)(r * 128 + (c << 4))));
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int r = r0 + 4 * (8 * b8 + i);
              asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(sa + (uint32_t)(r * 128 + (c << 4))),
                           "r"(tf32_rna(__uint_as_float(u[i].x))), "r"(tf32_rna(__uint_as_float(u[i].y))),
                           "r"(tf32_rna(__uint_as_float(u[i].z))), "r"(tf32_rna(__uint_as_float(u[i].w)))
                           : "memory");
            }
          }
        } else {
          const int k0 = kb * kBlockK + c * 8;
          const bool valid = k0 < p.K;                       // K % 8 == 0: a chunk is inside or outside as a whole
          float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), gb = ga;
          if (valid) load_gate(img0, k0, ga, gb);
          mbar_wait(full_bar(stage), phase);
          if (valid) {
            const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
            int cur = img0;
            long bound = bound0;
#pragma unroll 1
            for (int b8 = 0; b8 < 4; ++b8) {
              uint4 u[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int r = r0 + 4 * (8 * b8 + i);
                asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(u[i].x), "=r"(u[i].y), "=r"(u[i].z), "=r"(u[i].w)
                             : "r"(sa + (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4))));
              }
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int r = r0 + 4 * (8 * b8 + i);
                if (r >= bound && cur < p.a_imgs - 1) {
                  do { ++cur; bound += p.a_rows_per_img; } while (r >= bound && cur < p.a_imgs - 1);
                  load_gate(cur, k0, ga, gb);
                }
                const float2 x0 = unpack_bf16x2(u[i].x), x1 = unpack_bf16x2(u[i].y), x2 = unpack_bf16x2(u[i].z),
                             x3 = unpack_bf16x2(u[i].w);
                const uint32_t o0 = pack_bf16x2(x0.x * ga.x, x0.y * ga.y), o1 = pack_bf16x2(x1.x * ga.z, x1.y * ga.w);
                const uint32_t o2 = pack_bf16x2(x2.x * gb.x, x2.y * gb.y), o3 = pack_bf16x2(x3.x * gb.z, x3.y * gb.w);
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};"
                             ::"r"(sa + (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4))), "r"(o0), "r"(o1), "r"(o2), "r"(o3)
                             : "memory");
              }
            }
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(ready_bar(stage));
      }
      turn = turn + 1 == kNumGateWarps ? 0 : turn + 1;
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
  } else if (warp_idx < kProducerWarp) {
    // ------------------------------- consumers -------------------------------
    const int wg = warp_idx >> 2;   // warpgroup: tile rows 64 wg .. 64 wg + 63
    const bool releaser = (threadIdx.x & 127) == 0;
    if constexpr (STAGED) {
      // the tile's bias and gamma, once: the load's latency overlaps the first k-block's TMA; read after a barrier in
      // epilogue_staged.  Columns past N get neutral values (the store clips them anyway).
      const int t = threadIdx.x, n = n_blk * BLOCK_N + (t % BLOCK_N);
      if (t < BLOCK_N && p.bias != nullptr) s_bias[t] = n < p.N ? __ldg(p.bias + n) : 0.f;
      if (t >= BLOCK_N && t < 2 * BLOCK_N && p.gamma != nullptr) s_gamma[t - BLOCK_N] = n < p.N ? __ldg(p.gamma + n) : 1.f;
    }
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      // A-transform instances: the A tile has been rewritten
      mbar_wait(AX != kANone ? ready_bar(stage) : full_bar(stage), phase);
      const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
      const uint64_t da = gmma_desc_k_sw128(sa + (uint32_t)wg * (64 * 128));
      const uint64_t db = gmma_desc_b<MODE == kModeToken>(sa + Cfg::kABytes);
      wgmma_fence();
      // four 32-byte k-steps per 128-byte row (k16 bf16 / k8 tf32): +2 on the descriptors each
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (AX == kATf32)
          wgmma_ss_tf32<BLOCK_N>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
        else
          wgmma_ss<BLOCK_N, MODE == kModeToken>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(kDescStepB<MODE == kModeToken> * k),
                                                (uint32_t)((kb | k) != 0));
      }
      wgmma_commit();
      // the group issued one k-block ago has retired: its stage may be refilled
      wgmma_wait<1>();
      if (kb > 0 && releaser) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    if (releaser) mbar_arrive(empty_bar(prev));
    if constexpr (MODE == kModeToken) epilogue_token<OutT, BLOCK_N>(p, acc, img, m_blk, n_blk, wg * 64);
    else if constexpr (MODE == kModeGluCols) epilogue_glu_cols<OutT, BLOCK_N>(p, acc, m_blk, n_blk, wg * 64);
    else if constexpr (STAGED)
      epilogue_staged<OutT, BLOCK_N>(p, acc, m_blk, n_blk, wg, smem_out, s_bias, s_gamma, res_bar, &tmap_c);
    else epilogue_frag<OutT, BLOCK_N>(p, acc, m_blk, n_blk, wg * 64);
  }
}

// ---------------------- persistent 128 x 256 instance ----------------------
// The plain bf16 GEMM with the staged epilogue, one CTA per SM: CTA c takes tiles c, c + gridDim.x, ... in the n-fastest
// order of the per-tile grid.  A 128 x 256 tile loads half the operand bytes per MAC of a 128 x 64 one.  The producer's
// ring stage and phase run on across tiles, so it fills the next tile's first k-blocks while the consumers run the
// epilogue, and the tensor cores restart on a full ring.
// Shared memory: 3 stages of 48 KB, a 64 KB staging buffer of four 8 KB boxes per warpgroup (the whole bf16 tile, or
// one 128-column half of the fp32 tile), bias and gamma of two tiles (one warpgroup may still read tile i's while the
// other writes tile i + 1's), and the barriers: 213 KB.
struct PersistentCfg {
  static constexpr int kBlockN = 256;
  static constexpr int kABytes = kBlockM * kRowBytes;
  static constexpr int kStageBytes = kABytes + kBlockN * kRowBytes;
  static constexpr int kStages = 3;
  static constexpr int kBoxes = 4;   // staged boxes per warpgroup
  static constexpr int kOutBytes = 2 * kBoxes * kStagedBoxBytes;
  static constexpr int kVecBytes = 2 * 2 * kBlockN * 4;
  static constexpr int kNumBarriers = 2 * kStages + 2;   // full, empty, one residual barrier per warpgroup
  static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + kVecBytes + kNumBarriers * 8 + 1024;
};

// Each warpgroup's leader thread (its thread 0) moves the warpgroup's staged rows: it loads the residual span into them
// by TMA and stores the result from them.  Before the next residual load or epilogue reuses the boxes, it waits until
// the previous store has read them (cp.async.bulk.wait_group.read); for a tile's first span that wait and the residual
// load are issued right after the tile's first k-block, so both hide under the mainloop.  fp32 output takes two spans of
// 128 columns: the second span's residual is loaded once the first span's store has been read out.  In place is safe:
// tiles are disjoint, and a span is stored after its own residual has landed.
template <typename OutT>
__global__ void __launch_bounds__(kConsumerThreads + 32, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r,
                       const GemmParams p) {
  using Cfg = PersistentCfg;
  constexpr int BN = Cfg::kBlockN, kStages = Cfg::kStages, kBlockK = 64;
  constexpr int kCols = staged_chunk_cols<OutT>(), kSpan = Cfg::kBoxes * kCols;   // 256 bf16 / 128 fp32 columns

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_tiles = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_out = smem_tiles + kStages * Cfg::kStageBytes;
  const uint32_t smem_vec = smem_out + Cfg::kOutBytes;
  const uint32_t smem_bars = smem_vec + Cfg::kVecBytes;
  auto full_bar = [&](int s) { return smem_bars + 8u * s; };
  auto empty_bar = [&](int s) { return smem_bars + 8u * (kStages + s); };
  float* const s_vec = reinterpret_cast<float*>(smem_raw + (smem_vec - smem_u32(smem_raw)));

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (warp_idx == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    prefetch_tmap(&tmap_c);
    if (p.has_res) prefetch_tmap(&tmap_r);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    mbar_init(smem_bars + 8u * (2 * kStages), 1);
    mbar_init(smem_bars + 8u * (2 * kStages + 1), 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int num_n_tiles = (p.N + BN - 1) / BN;
  const int tiles = ((p.M + kBlockM - 1) / kBlockM) * num_n_tiles;
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;

  if (warp_idx == kProducerWarp) {
    // ------------------------------ TMA producer ------------------------------
    if (threadIdx.x == kProducerWarp * 32) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int m_blk = t / num_n_tiles, n_blk = t % num_n_tiles;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
          mbar_expect_tx(full_bar(stage), Cfg::kStageBytes);
          tma_load_2d(sa, &tmap_a, full_bar(stage), kb * kBlockK, m_blk * kBlockM);
          tma_load_2d(sa + Cfg::kABytes, &tmap_b, full_bar(stage), kb * kBlockK, n_blk * BN);
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ------------------------------- consumers -------------------------------
  const int wg = warp_idx >> 2;   // warpgroup: tile rows 64 wg .. 64 wg + 63
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t s_wg = smem_out + (uint32_t)(wg * Cfg::kBoxes * kStagedBoxBytes);
  const uint32_t res_bar = smem_bars + 8u * (2 * kStages + wg);
  int stage = 0, prev = 0, buf = 0;
  uint32_t phase = 0, res_phase = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x, buf ^= 1) {
    const int m_blk = t / num_n_tiles, n_blk = t % num_n_tiles;
    const int row0 = m_blk * kBlockM + wg * 64;
    // span h of this warpgroup's rows has a residual to load (uniform over the warpgroup)
    auto has_res_span = [&](int h) { return p.has_res && row0 < p.M && n_blk * BN + h * kSpan < p.N; };
    auto load_res_span = [&](int h) {   // leader only
      const int col0 = n_blk * BN + h * kSpan, chunks = min(Cfg::kBoxes, (p.N - col0 + kCols - 1) / kCols);
      mbar_expect_tx(res_bar, (uint32_t)(chunks * kStagedBoxBytes));
      for (int ch = 0; ch < chunks; ++ch)
        tma_load_2d(s_wg + (uint32_t)(ch * kStagedBoxBytes), &tmap_r, res_bar, col0 + ch * kCols, row0);
    };
    // the tile's bias and gamma (columns past N get neutral values): loaded here, written to shared memory once the
    // first k-block's MMAs are issued, so the load's latency does not delay them; read after a barrier in the epilogue
    float* const s_bias = s_vec + buf * 2 * BN;
    float* const s_gamma = s_bias + BN;
    const int n_own = n_blk * BN + threadIdx.x;
    const float bias_own = p.bias != nullptr && n_own < p.N ? __ldg(p.bias + n_own) : 0.f;
    const float gamma_own = p.gamma != nullptr && n_own < p.N ? __ldg(p.gamma + n_own) : 1.f;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_tiles + stage * Cfg::kStageBytes;
      const uint64_t da = gmma_desc_k_sw128(sa + (uint32_t)wg * (64 * 128));
      const uint64_t db = gmma_desc_k_sw128(sa + Cfg::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<BN, false>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
      wgmma_commit();
      if (kb == 0) {
        s_bias[threadIdx.x] = bias_own;
        s_gamma[threadIdx.x] = gamma_own;
      }
      // halfway through the mainloop, the previous tile's store has long read the staged boxes: the leader's wait
      // (which holds up its warpgroup's next MMAs) is short, and the residual has the other half to land
      if (kb == num_k_blocks / 2 && leader) {
        tma_store_wait_read<0>();
        if (has_res_span(0)) load_res_span(0);
      }
      wgmma_wait<1>();
      if (kb > 0 && leader) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    if (leader) mbar_arrive(empty_bar(prev));

    // ------------------------------- epilogue -------------------------------
    named_bar_sync<1>(256);   // s_bias / s_gamma were written by both consumer warpgroups
    auto span = [&](auto h_const) {
      constexpr int h = decltype(h_const)::value;
      if (n_blk * BN + h * kSpan >= p.N) return;
      if constexpr (h > 0) {
        // the boxes hold the previous span until its store has read them
        if (leader) {
          tma_store_wait_read<0>();
          if (has_res_span(h)) load_res_span(h);
        }
        warpgroup_bar_sync(wg);
      }
      if (has_res_span(h)) {
        mbar_wait(res_bar, res_phase);
        res_phase ^= 1u;
      }
      staged_apply<OutT, BN, h * kSpan, kSpan>(p, acc, s_wg, s_bias, s_gamma);
      // generic-proxy writes -> visible to the TMA engine, then the leader stores the span
      fence_proxy_async_smem();
      warpgroup_bar_sync(wg);
      if (leader && row0 < p.M) staged_store<OutT, Cfg::kBoxes>(p, &tmap_c, s_wg, row0, n_blk * BN + h * kSpan);
    };
    span(std::integral_constant<int, 0>{});
    if constexpr (kSpan < BN) span(std::integral_constant<int, 1>{});
  }
  if (leader) tma_store_wait_read<0>();   // the CTA's shared memory must outlive the last store's reads
}

// ------------------------------ host side -----------------------------------
// Output / residual: 16-byte aligned base and row stride (vector epilogue accesses, as the layout of every caller).
int check_out(const void* C, long ldc, const void* residual, long ldr, int esize) {
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(C) & 15u) == 0 && (ldc * esize) % 16 == 0,
                  "gemm: C must be 16-byte aligned with a row stride of a multiple of 16 bytes");
  TFIMM_CHECK_ARG(residual == nullptr || ((reinterpret_cast<uintptr_t>(residual) & 15u) == 0 && (ldr * esize) % 16 == 0),
                  "gemm: residual must be 16-byte aligned with a row stride of a multiple of 16 bytes");
  return kOk;
}

// Every launch of a gemm_wgmma_kernel instance: the shared-memory attribute, one CTA per 128 x BLOCK_N output tile (per
// image for token mixing), the launch and its error check.
// tc / tr: output and residual maps of the STAGED instances (unused otherwise).
template <int BLOCK_N, typename OutT, int AX, int MODE, bool STAGED = false>
int launch_wgmma(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, const char* what,
                 cudaStream_t stream, const CUtensorMap& tc = CUtensorMap{}, const CUtensorMap& tr = CUtensorMap{}) {
  using Cfg = GemmCfg<BLOCK_N, OutT, STAGED>;
  auto kernel = gemm_wgmma_kernel<BLOCK_N, OutT, AX, MODE, STAGED>;
  static std::atomic<unsigned long long> attr_devs{0};  // per instantiation
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Cfg::kSmemBytes, attr_devs));
  const long imgs = MODE == kModeToken ? p.tk_imgs : 1;
  const long tiles = imgs * ((p.M + kBlockM - 1) / kBlockM) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  kernel<<<(unsigned)tiles, gemm_threads<BLOCK_N, AX>(), Cfg::kSmemBytes, stream>>>(ta, tb, tc, tr, p);
  TFIMM_LAUNCH_OK(what);
  return kOk;
}

// Calls launch(std::integral_constant<int, BLOCK_N>{}) for the tile width bn.  kMaxN = 128 for the instances with
// A-transform warps, which leave the consumers too few registers for a 256-wide accumulator.
template <int kMaxN, typename F>
int with_block_n(int bn, const char* unsupported_fmt, F&& launch) {
  if constexpr (kMaxN >= 256) {
    if (bn == 256) return launch(std::integral_constant<int, 256>{});
  }
  if (bn == 128) return launch(std::integral_constant<int, 128>{});
  if (bn == 64) return launch(std::integral_constant<int, 64>{});
  set_last_error(unsupported_fmt, bn);
  return kInvalidArgument;
}

// The persistent 128 x 256 instance: one CTA per SM, or one per tile when there are fewer tiles.
template <typename OutT>
int launch_persistent(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr,
                      const GemmParams& p, cudaStream_t stream) {
  using Cfg = PersistentCfg;
  auto kernel = gemm_persistent_kernel<OutT>;
  static std::atomic<unsigned long long> attr_devs{0};  // per instantiation
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Cfg::kSmemBytes, attr_devs));
  const long tiles = (long)((p.M + kBlockM - 1) / kBlockM) * ((p.N + Cfg::kBlockN - 1) / Cfg::kBlockN);
  const int grid = (int)std::min<long>(tiles, sm_count());
  kernel<<<grid, kConsumerThreads + 32, Cfg::kSmemBytes, stream>>>(ta, tb, tc, tr, p);
  TFIMM_LAUNCH_OK("gemm_persistent_kernel (bf16)");
  return kOk;
}

// PERSISTENT (BLOCK_N = 256, plain bf16 GEMM): the persistent instance instead of the per-tile one.
template <int BLOCK_N, typename OutT, int AX = kANone, int MODE = kModeGemm, bool PERSISTENT = false>
int launch_gemm(const void* A, int lda, const void* W, int ldw, const void* residual, int ldr, void* C, int ldc,
                GemmParams p, cudaStream_t stream) {
  static_assert(!PERSISTENT || (BLOCK_N == PersistentCfg::kBlockN && AX == kANone && MODE == kModeGemm),
                "the persistent instance is the plain bf16 GEMM at 256 columns");
  const int M = p.M, N = p.N, K = p.K;
  constexpr int kBlockK = block_k<AX>();
  CUtensorMap ta, tb;
  int st;
  if ((st = check_out(C, ldc, residual, ldr, (int)sizeof(OutT))) != kOk) return st;
  if ((st = make_tmap_2d(&ta, A, dtype_code<AX>(), M, K, lda, kBlockM, kBlockK, "A")) != kOk) return st;
  if ((st = make_tmap_2d(&tb, W, dtype_code<AX>(), N, K, ldw, BLOCK_N, kBlockK, "W")) != kOk) return st;
  p.c = C; p.res = residual; p.ldc = ldc; p.ldr = ldr;
  // The plain bf16 GEMM at 64 / 128 columns and the persistent instance stage their epilogue through shared memory.  The
  // output and residual maps have the real extents (N, M) and their own row strides, in 64-row boxes of one 128-byte
  // span.  The TMA store clips a row only at a 16-byte boundary: with N * sizeof(OutT) % 16 != 0 (bf16 out, N % 8 != 0)
  // it would overwrite the elements after column N up to that boundary, so those shapes keep the fragment epilogue.
  constexpr bool kStaged = AX == kANone && MODE == kModeGemm && (BLOCK_N <= 128 || PERSISTENT);
  if constexpr (kStaged) {
    if ((long)N * (long)sizeof(OutT) % 16 != 0)
      return launch_wgmma<BLOCK_N, OutT, AX, MODE>(ta, tb, p, "gemm_wgmma_kernel (bf16)", stream);
    constexpr int es = (int)sizeof(OutT), dt = es == 2 ? kBF16 : kF32;
    CUtensorMap tc, tr{};
    if ((st = make_tmap_2d(&tc, C, dt, M, N, ldc, 64, staged_chunk_cols<OutT>(), "C")) != kOk) return st;
    if (residual != nullptr &&
        (st = make_tmap_2d(&tr, residual, dt, M, N, ldr, 64, staged_chunk_cols<OutT>(), "residual")) != kOk)
      return st;
    if constexpr (PERSISTENT) return launch_persistent<OutT>(ta, tb, tc, tr, p, stream);
    else return launch_wgmma<BLOCK_N, OutT, AX, MODE, true>(ta, tb, p, "gemm_wgmma_kernel (bf16)", stream, tc, tr);
  }
  return launch_wgmma<BLOCK_N, OutT, AX, MODE>(
      ta, tb, p,
      AX == kATf32 ? "gemm_wgmma_kernel (tf32)"
                   : (MODE == kModeGluCols ? "gemm_wgmma_kernel (bf16 glu)" : "gemm_wgmma_kernel (bf16)"),
      stream);
}

// Token mixing (kModeToken): A = Wt[M][K] (K-major, row stride ldw), B = X[imgs][K][N] (row stride ldx, image stride
// img_x), both bf16.
template <int BLOCK_N, typename OutT>
int launch_token(const void* Wt, int ldw, const void* X, long ldx, long img_x, GemmParams p, cudaStream_t stream) {
  CUtensorMap ta, tb;
  int st;
  if ((st = check_out(p.c, p.ldc, p.res, p.ldr, (int)sizeof(OutT))) != kOk) return st;
  if ((st = make_tmap_2d(&ta, Wt, kBF16, p.M, p.K, ldw, kBlockM, 64, "token Wt")) != kOk) return st;
  {
    const uint64_t dims[3] = {(uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.tk_imgs};
    const uint64_t strides[2] = {(uint64_t)ldx * 2, (uint64_t)img_x * 2};
    const uint32_t box[3] = {64u, 64u, 1u};
    if ((st = make_tmap(&tb, X, kBF16, 3, dims, strides, box, "token X")) != kOk) return st;
  }
  return launch_wgmma<BLOCK_N, OutT, kANone, kModeToken>(ta, tb, p, "gemm_wgmma_kernel (bf16 token mixing)", stream);
}

// Implicit k x k convolution on the tensor cores: same kernel, A tensor map = the NHWC input (rank 4, traversal
// stride = conv stride), C / residual = the NHWC output.  See GemmParams::conv.
template <int BLOCK_N, typename OutT, int AX = kANone>
int launch_conv(const void* x, const void* W, int ldw, const void* residual, void* out, int B, int H, int Wd, int C,
                int Ho, int Wo, GemmParams p, cudaStream_t stream) {
  constexpr int kBlockK = block_k<AX>();
  constexpr uint64_t es = sizeof(OperandT<AX>);
  const int N = p.N, s = p.cv_stride;
  CUtensorMap ta, tb;
  int st;
  if ((st = check_out(out, N, residual, N, (int)sizeof(OutT))) != kOk) return st;
  {
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)Wd, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)C * es, (uint64_t)Wd * C * es, (uint64_t)H * Wd * C * es};
    const uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)(p.cv_pw * s), (uint32_t)(p.cv_ph * s), (uint32_t)p.cv_pb};
    const uint32_t estr[4] = {1u, (uint32_t)s, (uint32_t)s, 1u};
    if ((st = make_tmap(&ta, x, dtype_code<AX>(), 4, dims, strides, box, "conv input", 128, estr)) != kOk) return st;
  }
  if ((st = make_tmap_2d(&tb, W, dtype_code<AX>(), N, p.K, ldw, BLOCK_N, kBlockK, "conv weights")) != kOk) return st;
  p.c = out; p.res = residual; p.ldc = N; p.ldr = N;
  p.cv_B = B; p.cv_Ho = Ho; p.cv_Wo = Wo;
  return launch_wgmma<BLOCK_N, OutT, AX, kModeGemm>(
      ta, tb, p,
      AX == kATf32 ? "gemm_wgmma_kernel (tf32 implicit convolution)" : "gemm_wgmma_kernel (bf16 implicit convolution)",
      stream);
}

int pick_block_n(int M, int N) {
  const int sms = sm_count() > 0 ? sm_count() : 132;  // no device (host-side shape queries): H100 SXM
  const int mt = (M + kBlockM - 1) / kBlockM;
  int best = 256;
  double best_cost = 1e30;
  for (int bn : {256, 128, 64}) {
    const int nt = (N + bn - 1) / bn;
    const long tiles = (long)mt * nt;
    // BLOCK_N = 64 runs two CTAs per SM
    const int slots = bn == 64 ? 2 * sms : sms;
    const long waves = (tiles + slots - 1) / slots;
    // time ~ waves * per-tile MMA time (prop. to bn, halved per CTA when two share an SM); small preference for wide
    // tiles, which load less operand data per MMA
    const double cost = (double)waves * (bn == 64 ? 2 * bn : bn) * (bn == 256 ? 1.0 : (bn == 128 ? 1.04 : 1.10));
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

// Tile width of the plain bf16 GEMM (tfimm_b200_gemm_bf16), fitted to measurements of its kernels (profiles/gemm_h100.md).
// The other instances keep pick_block_n: their kernels (A-transform warps, TF32 k-blocks, token mixing) were not measured
// against this rule.
// The persistent 128 x 256 instance, when its TMA store applies (not bf16 output with N % 8 != 0), its tiles fill every
// SM, and N > 256.  It measured fastest at every ViT-B, ConvNeXt-B and Swin-B shape with more than 256 columns, by
// 10-40 %, down to K = 128.  At N <= 256 (Swin-B's stage 1 and 2 proj: fp32 residual, bound by HBM) it was 2-8 % slower
// than the 64-wide tile; with N = 128 half of each 256-wide tile is empty.  Below one tile per SM it was not measured.
// Otherwise, from a wave count and a per-wave time:
//   BLOCK_N = 128, one CTA per SM: the epilogue runs after the mainloop with the tensor cores idle, so a wave costs
//     ~ 128 * (K + kEpilogueK).
//   BLOCK_N = 64, two CTAs per SM: one CTA's epilogue runs under the other's mainloop, so a wave of two tiles per SM
//     costs ~ kPairWidth * K.
// The constants were fitted with the fragment epilogue.  With the staged one, 128 ties 64 at the bias-only K = 768 ViT-B
// shapes, loses to it by 10-15 % with the GELU epilogue (fc1) and wins by 20-25 % at K = 3072 (fc2): the choices this
// model makes at those shapes, so it is kept until shapes where it chooses wrongly are measured.
// The per-tile BLOCK_N = 256 instance is not chosen: it was the slowest width at every measured shape (force_block_n
// still selects it).
constexpr int kPersistent = 1;   // force_block_n / pick_block_n_bf16 value of the persistent 128 x 256 instance

int pick_block_n_bf16(int M, int N, int K, int out_dtype) {
  constexpr double kEpilogueK = 926.0, kPairWidth = 184.0;
  const int sms = sm_count() > 0 ? sm_count() : 132;  // no device (host-side shape queries): H100 SXM
  const long mt = (M + kBlockM - 1) / kBlockM;
  if (N > 256 && (out_dtype == kF32 || N % 8 == 0) && mt * ((N + 255) / 256) >= sms) return kPersistent;
  const long waves128 = (mt * ((N + 127) / 128) + sms - 1) / sms;
  const long waves64 = (mt * ((N + 63) / 64) + 2 * sms - 1) / (2 * sms);
  return (double)waves64 * kPairWidth * K < (double)waves128 * 128.0 * (K + kEpilogueK) ? 64 : 128;
}

}  // namespace

int gemm_bf16_skinny(const void* A, int lda, const void* W, int ldw, const float* bias, const void* residual, int ldr,
                     void* C, int ldc, int M, int N, int K, int act, cudaStream_t stream, const float* gate = nullptr,
                     int rows_per_img = 1, int imgs = 1);

// k x k convolution (stride 1 or 2, symmetric padding (k-1)/2... given as `pad`) + bias + activation (+ residual),
// NHWC bf16 in, NHWC bf16/fp32 out, W[N][k*k*C] in (ky, kx, c) order: implicit GEMM, no im2col matrix in HBM.
// Geometry of an implicit convolution (shared by the bf16 and TF32 entry points); `cblock` = channels per k-block.
int conv_setup(GemmParams& p, const float* bias, const void* residual, int B, int H, int Wd, int C, int N, int ks,
               int stride, int pad, int act, int act_post, int cblock, int& Ho, int& Wo) {
  TFIMM_CHECK_ARG(B > 0 && H > 0 && Wd > 0 && C > 0 && C % cblock == 0, "conv: C must be a multiple of %d (got %d)",
                  cblock, C);
  TFIMM_CHECK_ARG(ks >= 1 && ks <= 7 && (stride == 1 || stride == 2) && pad >= 0 && pad < ks, "conv: bad geometry");
  TFIMM_CHECK_ARG(N > 0 && N % 8 == 0, "conv: N must be a multiple of 8 (got %d)", N);
  TFIMM_CHECK_ARG(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15u) == 0, "conv: bias must be 16-byte aligned");
  Ho = (H + 2 * pad - ks) / stride + 1;
  Wo = (Wd + 2 * pad - ks) / stride + 1;
  TFIMM_CHECK_ARG(Ho > 0 && Wo > 0, "conv: empty output");
  p = GemmParams{};
  p.N = N; p.K = ks * ks * C;
  p.bias = bias; p.act = act; p.has_res = residual != nullptr ? 1 : 0; p.act_post = act_post;
  p.conv = 1; p.cv_cblocks = C / cblock; p.cv_ks = ks; p.cv_stride = stride; p.cv_pad = pad;
  // 128-pixel output patch: 8 x 16 pixels of one image, or 8 x 8 pixels of two images for small feature maps
  if (Wo > 8) { p.cv_pb = 1; p.cv_ph = 8; p.cv_pw = 16; }
  else { p.cv_pb = 2; p.cv_ph = 8; p.cv_pw = 8; }
  p.cv_tiles_x = (Wo + p.cv_pw - 1) / p.cv_pw;
  p.cv_tiles_y = (Ho + p.cv_ph - 1) / p.cv_ph;
  const int tiles_b = (B + p.cv_pb - 1) / p.cv_pb;
  p.M = tiles_b * p.cv_tiles_y * p.cv_tiles_x * kBlockM;  // padded row count: every tile is a full patch
  return kOk;
}

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_gemm_bf16(const void* A, int lda, const void* W, int ldw, const float* bias, const float* gamma,
                         const void* residual, int ldr, void* C, int ldc, int M, int N, int K, int act, int act_post,
                         int out_dtype, int force_block_n, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: M, N, K must be positive (got %d %d %d)", M, N, K);
  TFIMM_CHECK_ARG(out_dtype == kBF16 || out_dtype == kF32, "gemm: out_dtype must be bf16 or f32");
  TFIMM_CHECK_ARG(K % 8 == 0, "gemm: K must be a multiple of 8 (got %d)", K);
  TFIMM_CHECK_ARG(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15u) == 0, "gemm: bias must be 16-byte aligned");
  TFIMM_CHECK_ARG(gamma == nullptr || (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0, "gemm: gamma must be 16-byte aligned");
  if (force_block_n == 0 && K <= 64 && out_dtype == kBF16 && gamma == nullptr && act_post == 0) {
    // short contraction: streaming mma.sync kernel (gemm_skinny.cu); kUnsupported = shape outside its envelope
    const int st = gemm_bf16_skinny(A, lda, W, ldw, bias, residual, ldr, C, ldc, M, N, K, act, stream);
    if (st != kUnsupported) return st;
  }
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.gamma = gamma; p.act = act; p.has_res = residual != nullptr ? 1 : 0; p.act_post = act_post;
  // force_block_n: 0 = choose; 64/128/256 = that tile width; 2 = the widest tile (256); 1 = the persistent instance
  const int bn =
      force_block_n == 2 ? 256 : (force_block_n > 0 ? force_block_n : pick_block_n_bf16(M, N, K, out_dtype));
  if (bn == kPersistent)
    return out_dtype == kBF16
               ? launch_gemm<256, __nv_bfloat16, kANone, kModeGemm, true>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream)
               : launch_gemm<256, float, kANone, kModeGemm, true>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream);
  return with_block_n<256>(bn, "gemm: unsupported block_n %d", [&](auto n) {
    constexpr int BN = decltype(n)::value;
    return out_dtype == kBF16 ? launch_gemm<BN, __nv_bfloat16>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream)
                              : launch_gemm<BN, float>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream);
  });
}

// Dense layer whose input rows are first multiplied by a per-image channel gate (squeeze-excite): the projection
// convolutions after SEModule (tfimm/layers/attention.py, efficientnet_blocks.py:241-248, 438-453).  bf16 out.
int tfimm_b200_gemm_bf16_gated(const void* A, int lda, const float* gate, int rows_per_img, int imgs, const void* W,
                               int ldw, const float* bias, const void* residual, int ldr, void* C, int ldc, int M,
                               int N, int K, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0 && K % 8 == 0, "gemm_gated: need K %% 8 == 0 (got M=%d N=%d K=%d)", M, N, K);
  TFIMM_CHECK_ARG(gate != nullptr && rows_per_img > 0 && imgs > 0 && (reinterpret_cast<uintptr_t>(gate) & 15u) == 0,
                  "gemm_gated: gate [imgs][K] fp32, 16-byte aligned");
  TFIMM_CHECK_ARG(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15u) == 0, "gemm_gated: bias must be 16-byte aligned");
  if (K <= 64) {   // short contraction: the streaming kernel scales its A fragments in registers
    const int st = gemm_bf16_skinny(A, lda, W, ldw, bias, residual, ldr, C, ldc, M, N, K, act, stream, gate, rows_per_img,
                                    imgs);
    if (st != kUnsupported) return st;
  }
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.act = act; p.has_res = residual != nullptr ? 1 : 0;
  p.a_scale = gate; p.a_rows_per_img = rows_per_img; p.a_imgs = imgs;
  return with_block_n<128>(pick_block_n(M, N) == 64 ? 64 : 128, "gemm_gated: unsupported block_n %d", [&](auto n) {
    return launch_gemm<decltype(n)::value, __nv_bfloat16, kAGate>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream);
  });
}

int tfimm_b200_conv_bf16(const void* x, const void* W, int ldw, const float* bias, const void* residual, void* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act, int act_post,
                         int out_dtype, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(out_dtype == kBF16 || out_dtype == kF32, "conv: out_dtype must be bf16 or f32");
  GemmParams p;
  int Ho, Wo, st;
  if ((st = conv_setup(p, bias, residual, B, H, Wd, C, N, ks, stride, pad, act, act_post, 64, Ho, Wo)) != kOk)
    return st;
  return with_block_n<256>(N >= 256 ? 256 : (N >= 128 ? 128 : 64), "conv: unsupported block_n %d", [&](auto n) {
    constexpr int BN = decltype(n)::value;
    return out_dtype == kBF16 ? launch_conv<BN, __nv_bfloat16>(x, W, ldw, residual, out, B, H, Wd, C, Ho, Wo, p, stream)
                              : launch_conv<BN, float>(x, W, ldw, residual, out, B, H, Wd, C, Ho, Wo, p, stream);
  });
}

// ---- precision="tf32": fp32 operands, TF32 tensor-core products, fp32 out ----
// W must already be TF32-representable (low 13 bits zero: rounded once at plan time); the A tiles are rounded in shared
// memory by the transform warps.  At most 128 columns: the transform warps leave the consumers too few registers for a
// 256-wide accumulator (as in the gated instances).
int tfimm_b200_gemm_tf32(const float* A, int lda, const float* W, int ldw, const float* bias, const float* gamma,
                         const float* residual, int ldr, float* C, int ldc, int M, int N, int K, int act, int act_post,
                         int force_block_n, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm_tf32: M, N, K must be positive (got %d %d %d)", M, N, K);
  TFIMM_CHECK_ARG(K % 4 == 0, "gemm_tf32: K must be a multiple of 4 (got %d)", K);
  TFIMM_CHECK_ARG(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15u) == 0, "gemm_tf32: bias must be 16-byte aligned");
  TFIMM_CHECK_ARG(gamma == nullptr || (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0,
                  "gemm_tf32: gamma must be 16-byte aligned");
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.gamma = gamma; p.act = act; p.has_res = residual != nullptr ? 1 : 0; p.act_post = act_post;
  // force_block_n: 0 = choose; 64 / 128 = that tile width; 2 = the widest tile (128)
  const int bn = force_block_n == 2 ? 128 : (force_block_n > 0 ? force_block_n : (pick_block_n(M, N) == 64 ? 64 : 128));
  return with_block_n<128>(bn, "gemm_tf32: unsupported block_n %d (64 or 128)", [&](auto n) {
    return launch_gemm<decltype(n)::value, float, kATf32>(A, lda, W, ldw, residual, ldr, C, ldc, p, stream);
  });
}

// k x k convolution as tfimm_b200_conv_bf16, fp32 NHWC in / out with TF32 products; C % 32 == 0 (one 32-channel fp32 box
// per k-block).
int tfimm_b200_conv_tf32(const float* x, const float* W, int ldw, const float* bias, const float* residual, float* out,
                         int B, int H, int Wd, int C, int N, int ks, int stride, int pad, int act, int act_post,
                         void* s) {
  const cudaStream_t stream = as_stream(s);
  GemmParams p;
  int Ho, Wo, st;
  if ((st = conv_setup(p, bias, residual, B, H, Wd, C, N, ks, stride, pad, act, act_post, 32, Ho, Wo)) != kOk)
    return st;
  return with_block_n<128>(N >= 128 ? 128 : 64, "conv: unsupported block_n %d", [&](auto n) {
    return launch_conv<decltype(n)::value, float, kATf32>(x, W, ldw, residual, out, B, H, Wd, C, Ho, Wo, p, stream);
  });
}

// ---- MLP-Mixer family (tfimm.backend.mixer_ops) ----
// Token mixing: out[b][m][c] = epi(sum_n Wt[m][n] X[b][n][c]), see GemmParams (kModeToken) for the epilogue.
// Wt: bf16 [M][K], row stride ldw % 8 == 0 (rows padded at plan time); X: bf16, row stride ldx and image stride img_x,
// both multiples of 8 elements.  out / residual / mul: bf16 or fp32 (out_dtype), rows of N elements.
int tfimm_b200_token_gemm_bf16(const void* Wt, int ldw, const void* X, long ldx, long img_x, const float* bias,
                               const float* gamma, const void* residual, long ldr, long img_r, const void* mul,
                               long ld_mul, long img_mul, void* out, long ldc, long img_c, int imgs, int M, int N,
                               int K, int m_out, int act, int glu, int out_dtype, int force_block_n, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(imgs > 0 && M > 0 && N > 0 && K > 0 && m_out > 0, "token_gemm: empty shape (imgs %d M %d N %d K %d)",
                  imgs, M, N, K);
  TFIMM_CHECK_ARG(out_dtype == kBF16 || out_dtype == kF32, "token_gemm: out_dtype must be bf16 or f32");
  TFIMM_CHECK_ARG(ldw % 8 == 0 && ldw >= K && ldx % 8 == 0 && img_x % 8 == 0 && ldx >= N,
                  "token_gemm: Wt / X strides must be multiples of 8 elements");
  TFIMM_CHECK_ARG(glu ? (M % 16 == 0 && m_out <= M / 2) : m_out <= M, "token_gemm: m_out %d does not fit M %d (glu %d)",
                  m_out, M, glu);
  TFIMM_CHECK_ARG(N % 2 == 0 && (gamma == nullptr || (reinterpret_cast<uintptr_t>(gamma) & 7u) == 0),
                  "token_gemm: N must be even and gamma 8-byte aligned");
  const int es = out_dtype == kBF16 ? 2 : 4;
  TFIMM_CHECK_ARG(mul == nullptr || ((reinterpret_cast<uintptr_t>(mul) & 15u) == 0 && (ld_mul * es) % 16 == 0 &&
                                     (img_mul * es) % 16 == 0),
                  "token_gemm: mul must be 16-byte aligned with strides of multiples of 16 bytes");
  TFIMM_CHECK_ARG((img_c * es) % 16 == 0 && (residual == nullptr || (img_r * es) % 16 == 0),
                  "token_gemm: image strides must be multiples of 16 bytes");
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.gamma = gamma; p.act = act; p.has_res = residual != nullptr ? 1 : 0;
  p.c = out; p.res = residual; p.ldc = ldc; p.ldr = ldr;
  p.tk_imgs = imgs; p.m_out = m_out; p.glu = glu; p.img_c = img_c; p.img_r = img_r;
  p.mul = mul; p.ld_mul = ld_mul; p.img_mul = img_mul;
  const int bn = force_block_n > 0 ? force_block_n : pick_block_n(imgs * ((M + kBlockM - 1) / kBlockM) * kBlockM, N);
  return with_block_n<256>(bn, "token_gemm: unsupported block_n %d", [&](auto n) {
    constexpr int BN = decltype(n)::value;
    return out_dtype == kBF16 ? launch_token<BN, __nv_bfloat16>(Wt, ldw, X, ldx, img_x, p, stream)
                              : launch_token<BN, float>(Wt, ldw, X, ldx, img_x, p, stream);
  });
}

// Channel GLU (gMixer's mlp_channels fc1): W rows 2j / 2j + 1 are value / gate feature j (interleaved at plan time),
// bias likewise; out[M][N / 2] = (A W_value^T + b) * act(A W_gate^T + b), bf16.  The full-width hidden tensor is never
// written.
int tfimm_b200_gemm_glu_bf16(const void* A, int lda, const void* W, int ldw, const float* bias, void* C, int ldc, int M,
                             int N, int K, int act, int force_block_n, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(M > 0 && N > 0 && K > 0 && K % 8 == 0 && N % 2 == 0,
                  "gemm_glu: need K %% 8 == 0 and an even N (got M=%d N=%d K=%d)", M, N, K);
  TFIMM_CHECK_ARG(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 7u) == 0, "gemm_glu: bias must be 8-byte aligned");
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.bias = bias; p.act = act;
  const int bn = force_block_n > 0 ? force_block_n : pick_block_n(M, N);
  return with_block_n<256>(bn, "gemm_glu: unsupported block_n %d", [&](auto n) {
    return launch_gemm<decltype(n)::value, __nv_bfloat16, kANone, kModeGluCols>(A, lda, W, ldw, nullptr, 0, C, ldc, p,
                                                                               stream);
  });
}

}  // extern "C"
