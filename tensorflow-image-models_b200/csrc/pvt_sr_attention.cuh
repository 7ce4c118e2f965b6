// Spatial-reduction attention kernels of the PVT families, templated on the head dim DH (32 or 64): pvt.cu
// instantiates DH = 64 (PVT v1, PVT v2 b1-b5), pvt_v2.cu DH = 32 (PVT v2 b0).
//
// pvt_sr_attention_bf16_kernel<DH>  out = softmax(scale q k^T) v, N queries against N' keys per image.  q is the
//   (B N, H DH) output of the q GEMM; kv the (B N', 2 H DH) output of the kv GEMM, k of head h at column DH h and v at
//   H DH + DH h.  One CTA owns one (image, head) and `tiles` consecutive 64-query tiles of it.
//   - 4 warps, 16 query rows each.  Per tile the same arithmetic as pit_attention_bf16_kernel<DH> (pit.cu): Q held as
//     mma.sync A fragments, 64-key blocks, attention_mma.cuh's qk_bf16 / OnlineSoftmax<true> with raw scores / pv_bf16,
//     the normalised tile staged through the warp's own Q rows and stored as 16-byte chunks, rows past N not stored.
//     Keys past N' are zero-filled by the copy and set to -inf.  So with N' = N and q / kv cut from one packed qkv,
//     the output equals pit_attention_bf16's bit for bit.
//   - Shared-memory rows are DH + 8 bf16 wide: an odd number of 16-byte chunks (9 at DH 64, 5 at DH 32), so ldmatrix
//     is conflict-free.
//   - K / V go through a ring of kStages stages of 64 keys.  When N' fits in the ring (N' <= 192: every PVT stage at
//     224 px has N' <= 50), they are loaded once and stay resident while the CTA walks its query tiles; Q tiles are
//     double-buffered, the next one copied while the current one computes all its key blocks.  Past 192 keys the
//     ring streams K / V anew for every tile, as PiT's kernel does, and a CTA takes one tile.
//   - The tile count per CTA is chosen at launch (pvt_tiles_per_cta): several tiles share one K / V load while the
//     grid still fills the GPU for a few waves.
// pvt_sr_attention_f32_kernel<DH>  the same operation on fp32 q / kv: one warp per query row, keys in blocks of 32 (one
//   per lane: score = (scale q) . k by DH fmas), an online softmax with expf (m the running maximum, l the running sum
//   of the unrounded p, O and l rescaled by expf(m_old - m_new)), lane d accumulating output column d (and d + 32 at
//   DH 64); at the end out = O / l.
#pragma once

#include "attention_mma.cuh"
#include "common.cuh"

#ifndef TFIMM_PVT_MAX_TILES
#define TFIMM_PVT_MAX_TILES 8   // query tiles per CTA at most (profiles/pvt_h100.md)
#endif

namespace tfimm {
namespace {

template <int DH>
struct PvtSra {
  static constexpr int kWarps = 4;
  static constexpr int kRows = kWarps * 16;          // queries per tile
  static constexpr int kKeys = 64;                   // keys per ring stage
  static constexpr int kStages = 3;
  static constexpr int kChunks = DH / 8;             // 16-byte chunks of a row of q, k or v
  static constexpr int kRowBytes = (DH + 8) * 2;     // padded shared-memory row: an odd number of chunks
  static constexpr int kQBytes = kRows * kRowBytes;
  static constexpr int kStageBytes = 2 * kKeys * kRowBytes;
  static constexpr int kSmem = 2 * kQBytes + kStages * kStageBytes;
  // CTAs of this footprint that fit in an SM's 228 KB of shared memory (1 KB of it reserved per CTA): 3 at DH 64, 5 at
  // DH 32
  static constexpr int kCtasPerSm = (228 * 1024) / (kSmem + 1024);
};

template <int DH>
__global__ void __launch_bounds__(PvtSra<DH>::kWarps * 32)
pvt_sr_attention_bf16_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                             __nv_bfloat16* __restrict__ out, int N, int Nk, int H, int tiles_per_cta,
                             float scale_log2) {
  using S = PvtSra<DH>;
  constexpr int kWarps = S::kWarps, kRows = S::kRows, kKeys = S::kKeys, kStages = S::kStages;
  constexpr int kQBytes = S::kQBytes, kStageBytes = S::kStageBytes;
  constexpr int RB = S::kRowBytes, CH = S::kChunks;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sRing = sQ + 2 * kQBytes;

  const int b = blockIdx.z, h = blockIdx.y;
  const int tile0 = blockIdx.x * tiles_per_cta;
  const int tiles = min(tiles_per_cta, (N + kRows - 1) / kRows - tile0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long ldq = (long)H * DH, ldkv = 2L * H * DH;
  const __nv_bfloat16* qbase = q + (long)b * N * ldq + h * DH;
  const __nv_bfloat16* kbase = kv + (long)b * Nk * ldkv + h * DH;
  const int nblocks = (Nk + kKeys - 1) / kKeys;
  const bool resident = nblocks <= kStages;
  const int nsteps = tiles * nblocks;   // (tile, key block) pairs, in that order

  // one commit group per call, empty when there is nothing to copy, so that wait_group counts stay uniform.  Resident
  // K / V: block kb lives in stage kb and is copied once; streamed: step j's block goes to stage j % kStages.
  auto load_step = [&](int j) {
    if (j < nsteps && (!resident || j < nblocks)) {
      const int kb = j % nblocks;
      const uint32_t sK = sRing + (resident ? kb : j % kStages) * kStageBytes;
      const uint32_t sV = sK + kKeys * RB;
      for (int idx = tid; idx < kKeys * CH; idx += kWarps * 32) {
        const int r = idx / CH, c = idx - r * CH;
        const int key = kb * kKeys + r;
        const bool valid = key < Nk;
        const __nv_bfloat16* src = kbase + (long)(valid ? key : 0) * ldkv + c * 8;
        cp_async_16(sK + r * RB + c * 16, src, valid);
        cp_async_16(sV + r * RB + c * 16, src + H * DH, valid);
      }
    }
    cp_async_commit();
  };
  auto load_q = [&](int tl) {
    const uint32_t dst = sQ + (tl & 1) * kQBytes;
    for (int idx = tid; idx < kRows * CH; idx += kWarps * 32) {
      const int r = idx / CH, c = idx - r * CH;
      const int row = (tile0 + tl) * kRows + r;
      const bool valid = row < N;
      cp_async_16(dst + r * RB + c * 16, qbase + (long)(valid ? row : 0) * ldq + c * 8, valid);
    }
    cp_async_commit();
  };

  load_q(0);
#pragma unroll
  for (int j = 0; j < kStages - 1; ++j) load_step(j);

  const int q0 = warp * 16;
  int step = 0;
#pragma unroll 1
  for (int tl = 0; tl < tiles; ++tl) {
    cp_async_wait<0>();   // this tile's Q (and everything copied so far) has landed
    __syncthreads();      // everyone's has, and every warp is done staging the previous tile in the other Q buffer
    if (tl + 1 < tiles) load_q(tl + 1);
    const int q_base = (tile0 + tl) * kRows;
    const bool active = q_base + q0 < N;
    const uint32_t sQt = sQ + (tl & 1) * kQBytes;
    uint32_t qf[DH / 16][4];
#pragma unroll
    for (int ks = 0; ks < DH / 16; ++ks) {
      const int row = q0 + (lane & 15);
      const int chunk = ks * 2 + (lane >> 4);
      ldmatrix_x4(sQt + row * RB + chunk * 16, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
    float o[DH / 8][4];
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    OnlineSoftmax<true> sm;

#pragma unroll 1
    for (int kb = 0; kb < nblocks; ++kb, ++step) {
      // this thread's copies of this step have landed.  Resident K / V after the first tile landed with the tile's
      // wait above, so the next tile's Q copy may stay in flight through every key block.
      if (!resident || tl == 0) cp_async_wait<kStages - 2>();
      __syncthreads();                // everyone's have, and every warp is done with the stage the next copy refills
      load_step(step + kStages - 1);
      if (!active) continue;
      const uint32_t sK = sRing + (resident ? kb : step % kStages) * kStageBytes;
      const uint32_t sV = sK + kKeys * RB;
      const int nvalid = min(kKeys, Nk - kb * kKeys);
      const int ntiles = (nvalid + 7) >> 3;   // 8-key tiles holding a key < N'

      float s[8][4];
      qk_bf16(s, qf, ntiles, lane, [&](int row, int chunk) { return sK + row * RB + chunk * 16; });
      if (nvalid < kKeys) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (nt * 8 + 2 * t + (e & 1) >= nvalid) s[nt][e] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
      }
      sm.update(s, o, mx, scale_log2);
      pv_bf16(o, s, ntiles, lane, [&](int row, int chunk) { return sV + row * RB + chunk * 16; });
    }
    if (!active) continue;

    const RowNorm n0 = sm.finish(0), n1 = sm.finish(1);
    uint8_t* tile = smem + (tl & 1) * kQBytes + q0 * RB;   // this warp's Q rows: read only by this warp, above
#pragma unroll
    for (int nt = 0; nt < DH / 8; ++nt) {
      *reinterpret_cast<uint32_t*>(tile + g * RB + nt * 16 + t * 4) = pack_bf16x2(n0(o[nt][0]), n0(o[nt][1]));
      *reinterpret_cast<uint32_t*>(tile + (g + 8) * RB + nt * 16 + t * 4) = pack_bf16x2(n1(o[nt][2]), n1(o[nt][3]));
    }
    __syncwarp();
    for (int idx = lane; idx < 16 * CH; idx += 32) {
      const int r = idx / CH, c = idx - r * CH;
      const int row = q_base + q0 + r;
      if (row < N)
        *reinterpret_cast<uint4*>(out + ((long)b * N + row) * ldq + h * DH + c * 8) =
            *reinterpret_cast<const uint4*>(tile + r * RB + c * 16);
    }
  }
  cp_async_wait<0>();   // only empty groups can be pending here
}

// Query tiles per CTA.  Streamed K / V: one.  Resident K / V: as many as keep at least kWaves waves of CTAs on the
// GPU (kCtasPerSm of them fit in shared memory), at most TFIMM_PVT_MAX_TILES, spread evenly over an image's tiles.
template <int DH>
int pvt_tiles_per_cta(int ntiles, int nblocks, int B, int H) {
  constexpr int kCtasPerSm = PvtSra<DH>::kCtasPerSm, kWaves = 4;
  if (nblocks > PvtSra<DH>::kStages) return 1;
  const long slots = (long)sm_count() * kCtasPerSm * kWaves;
  const long want = max(1L, min((long)TFIMM_PVT_MAX_TILES, (long)ntiles * B * H / slots));
  const long groups = (ntiles + want - 1) / want;
  return (int)((ntiles + groups - 1) / groups);
}

constexpr int kF32Warps = 4;
constexpr int kF32Keys = 32;   // keys per block of the fp32 online softmax: one per lane

template <int DH>
__global__ void __launch_bounds__(kF32Warps * 32)
pvt_sr_attention_f32_kernel(const float* __restrict__ q, const float* __restrict__ kv, float* __restrict__ out,
                            long rows, int N, int Nk, int H, float scale) {
  static_assert(DH == 32 || DH == 64, "lane d holds output column d, and d + 32 at DH 64");
  const int lane = threadIdx.x & 31;
  const long rid = (long)blockIdx.x * kF32Warps + (threadIdx.x >> 5);   // ((b H + h) N + n)
  if (rid >= rows) return;
  const int n = (int)(rid % N);
  const long bh = rid / N;
  const int h = (int)(bh % H);
  const long b = bh / H;
  const long ldq = (long)H * DH, ldkv = 2L * H * DH;
  float qs[DH];
  const float4* qr = reinterpret_cast<const float4*>(q + (b * N + n) * ldq + h * DH);
#pragma unroll
  for (int c = 0; c < DH / 4; ++c) {
    const float4 v = __ldg(qr + c);
    qs[4 * c] = v.x * scale; qs[4 * c + 1] = v.y * scale; qs[4 * c + 2] = v.z * scale; qs[4 * c + 3] = v.w * scale;
  }
  const float* kimg = kv + b * Nk * ldkv + h * DH;
  float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll 1
  for (int j0 = 0; j0 < Nk; j0 += kF32Keys) {
    const int j = j0 + lane;
    float s = -INFINITY;
    if (j < Nk) {
      const float4* kr = reinterpret_cast<const float4*>(kimg + (long)j * ldkv);
      s = 0.f;
#pragma unroll
      for (int c = 0; c < DH / 4; ++c) {
        const float4 k4 = __ldg(kr + c);
        s = fmaf(qs[4 * c], k4.x, s); s = fmaf(qs[4 * c + 1], k4.y, s);
        s = fmaf(qs[4 * c + 2], k4.z, s); s = fmaf(qs[4 * c + 3], k4.w, s);
      }
    }
    const float m_new = fmaxf(m, warp_max(s));   // finite: every block holds a key
    const float alpha = expf(m - m_new);
    const float p = expf(s - m_new);
    l = l * alpha + warp_sum(p);
    o0 *= alpha;
    if constexpr (DH == 64) o1 *= alpha;
    m = m_new;
    const int nvalid = min(kF32Keys, Nk - j0);
    const float* vr = kimg + (long)j0 * ldkv + H * DH;
#pragma unroll 4
    for (int jj = 0; jj < nvalid; ++jj) {
      const float pj = __shfl_sync(0xffffffffu, p, jj);
      o0 = fmaf(pj, __ldg(vr + (long)jj * ldkv + lane), o0);
      if constexpr (DH == 64) o1 = fmaf(pj, __ldg(vr + (long)jj * ldkv + lane + 32), o1);
    }
  }
  float* dst = out + (b * N + n) * ldq + h * DH;
  dst[lane] = o0 / l;
  if constexpr (DH == 64) dst[lane + 32] = o1 / l;
}

}  // namespace
}  // namespace tfimm
