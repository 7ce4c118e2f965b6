// Kernels of the PVT family (tfimm/architectures/pvt.py): spatial-reduction attention, whose keys and values come from
// a second, shorter sequence than the queries, in bf16 on the tensor cores and in fp32 on the CUDA cores; and the end of
// each stage's patch embedding (LayerNorm, position table, class row).  The blocks' LayerNorms and GEMMs, the patch and
// spatial-reduction convolutions (im2col + GEMM) run on the existing paths.
//
// pvt_sr_attention_bf16_kernel  out = softmax(scale q k^T) v, head dim 64, N queries against N' keys per image.  q is
//   the (B N, H 64) output of the q GEMM; kv the (B N', 2 H 64) output of the kv GEMM, k of head h at column 64 h and
//   v at H 64 + 64 h.  One CTA owns one (image, head) and `tiles` consecutive 64-query tiles of it.
//   - 4 warps, 16 query rows each.  Per tile the same arithmetic as pit_attention_bf16_kernel<64> (pit.cu): Q held as
//     mma.sync A fragments, 64-key blocks, attention_mma.cuh's qk_bf16 / OnlineSoftmax<true> with raw scores / pv_bf16,
//     the normalised tile staged through the warp's own Q rows and stored as 16-byte chunks, rows past N not stored.
//     Keys past N' are zero-filled by the copy and set to -inf.  So with N' = N and q / kv cut from one packed qkv,
//     the output equals pit_attention_bf16's bit for bit.
//   - K / V go through a ring of kStages stages of 64 keys.  When N' fits in the ring (N' <= 192: every PVT stage at
//     224 px has N' <= 50), they are loaded once and stay resident while the CTA walks its query tiles; Q tiles are
//     double-buffered, the next one copied while the current one computes all its key blocks.  Past 192 keys the
//     ring streams K / V anew for every tile, as PiT's kernel does, and a CTA takes one tile.
//   - The tile count per CTA is chosen at launch (pvt_tiles_per_cta): several tiles share one K / V load while the
//     grid still fills the GPU for a few waves.
// pvt_sr_attention_f32_kernel  the same operation on fp32 q / kv: one warp per query row, keys in blocks of 32 (one per
//   lane: score = (scale q) . k by 64 fmas), an online softmax with expf (m the running maximum, l the running sum of
//   the unrounded p, O and l rescaled by expf(m_old - m_new)), lane d accumulating output columns d and d + 32; at the
//   end out = O / l.
// pvt_embed_norm_kernel  out[b, ntok + p] = LayerNorm_eps(tok[b, p]) gamma + beta + pos[ntok + p] and, when ntok = 1,
//   out[b, 0] = cls + pos[0]: the fp32 residual stream of a stage.  The LayerNorm is layernorm_f32_rows_kernel's
//   (norm.cu, one row per warp) with the position row added after it.
#include "attention_mma.cuh"
#include "common.cuh"
#include "tfimm_b200_pvt.h"

#ifndef TFIMM_PVT_MAX_TILES
#define TFIMM_PVT_MAX_TILES 8   // query tiles per CTA at most (profiles/pvt_h100.md)
#endif

namespace tfimm {
namespace {

constexpr int kDH = 64;
constexpr int kWarps = 4;
constexpr int kRows = kWarps * 16;          // queries per tile
constexpr int kKeys = 64;                   // keys per ring stage
constexpr int kStages = 3;
constexpr int kChunks = kDH / 8;            // 16-byte chunks of a row of q, k or v
constexpr int kRowBytes = (kDH + 8) * 2;    // padded shared-memory row: 9 chunks, odd, so ldmatrix is conflict-free
constexpr int kQBytes = kRows * kRowBytes;
constexpr int kStageBytes = 2 * kKeys * kRowBytes;
constexpr int kSmem = 2 * kQBytes + kStages * kStageBytes;

__global__ void __launch_bounds__(kWarps * 32)
pvt_sr_attention_bf16_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                             __nv_bfloat16* __restrict__ out, int N, int Nk, int H, int tiles_per_cta,
                             float scale_log2) {
  constexpr int RB = kRowBytes, CH = kChunks;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sRing = sQ + 2 * kQBytes;

  const int b = blockIdx.z, h = blockIdx.y;
  const int tile0 = blockIdx.x * tiles_per_cta;
  const int tiles = min(tiles_per_cta, (N + kRows - 1) / kRows - tile0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long ldq = (long)H * kDH, ldkv = 2L * H * kDH;
  const __nv_bfloat16* qbase = q + (long)b * N * ldq + h * kDH;
  const __nv_bfloat16* kbase = kv + (long)b * Nk * ldkv + h * kDH;
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
        cp_async_16(sV + r * RB + c * 16, src + H * kDH, valid);
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
    uint32_t qf[kDH / 16][4];
#pragma unroll
    for (int ks = 0; ks < kDH / 16; ++ks) {
      const int row = q0 + (lane & 15);
      const int chunk = ks * 2 + (lane >> 4);
      ldmatrix_x4(sQt + row * RB + chunk * 16, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
    float o[kDH / 8][4];
#pragma unroll
    for (int i = 0; i < kDH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
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
    for (int nt = 0; nt < kDH / 8; ++nt) {
      *reinterpret_cast<uint32_t*>(tile + g * RB + nt * 16 + t * 4) = pack_bf16x2(n0(o[nt][0]), n0(o[nt][1]));
      *reinterpret_cast<uint32_t*>(tile + (g + 8) * RB + nt * 16 + t * 4) = pack_bf16x2(n1(o[nt][2]), n1(o[nt][3]));
    }
    __syncwarp();
    for (int idx = lane; idx < 16 * CH; idx += 32) {
      const int r = idx / CH, c = idx - r * CH;
      const int row = q_base + q0 + r;
      if (row < N)
        *reinterpret_cast<uint4*>(out + ((long)b * N + row) * ldq + h * kDH + c * 8) =
            *reinterpret_cast<const uint4*>(tile + r * RB + c * 16);
    }
  }
  cp_async_wait<0>();   // only empty groups can be pending here
}

// Query tiles per CTA.  Streamed K / V: one.  Resident K / V: as many as keep at least kWaves waves of CTAs on the
// GPU (kCtasPerSm of them fit in shared memory), at most TFIMM_PVT_MAX_TILES, spread evenly over an image's tiles.
int pvt_tiles_per_cta(int ntiles, int nblocks, int B, int H) {
  constexpr int kCtasPerSm = 3, kWaves = 4;
  if (nblocks > kStages) return 1;
  const long slots = (long)sm_count() * kCtasPerSm * kWaves;
  const long want = max(1L, min((long)TFIMM_PVT_MAX_TILES, (long)ntiles * B * H / slots));
  const long groups = (ntiles + want - 1) / want;
  return (int)((ntiles + groups - 1) / groups);
}

constexpr int kF32Warps = 4;
constexpr int kF32Keys = 32;   // keys per block of the fp32 online softmax: one per lane

__global__ void __launch_bounds__(kF32Warps * 32)
pvt_sr_attention_f32_kernel(const float* __restrict__ q, const float* __restrict__ kv, float* __restrict__ out,
                            long rows, int N, int Nk, int H, float scale) {
  const int lane = threadIdx.x & 31;
  const long rid = (long)blockIdx.x * kF32Warps + (threadIdx.x >> 5);   // ((b H + h) N + n)
  if (rid >= rows) return;
  const int n = (int)(rid % N);
  const long bh = rid / N;
  const int h = (int)(bh % H);
  const long b = bh / H;
  const long ldq = (long)H * kDH, ldkv = 2L * H * kDH;
  float qs[kDH];
  const float4* qr = reinterpret_cast<const float4*>(q + (b * N + n) * ldq + h * kDH);
#pragma unroll
  for (int c = 0; c < kDH / 4; ++c) {
    const float4 v = __ldg(qr + c);
    qs[4 * c] = v.x * scale; qs[4 * c + 1] = v.y * scale; qs[4 * c + 2] = v.z * scale; qs[4 * c + 3] = v.w * scale;
  }
  const float* kimg = kv + b * Nk * ldkv + h * kDH;
  float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll 1
  for (int j0 = 0; j0 < Nk; j0 += kF32Keys) {
    const int j = j0 + lane;
    float s = -INFINITY;
    if (j < Nk) {
      const float4* kr = reinterpret_cast<const float4*>(kimg + (long)j * ldkv);
      s = 0.f;
#pragma unroll
      for (int c = 0; c < kDH / 4; ++c) {
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
    o1 *= alpha;
    m = m_new;
    const int nvalid = min(kF32Keys, Nk - j0);
    const float* vr = kimg + (long)j0 * ldkv + H * kDH;
#pragma unroll 4
    for (int jj = 0; jj < nvalid; ++jj) {
      const float pj = __shfl_sync(0xffffffffu, p, jj);
      o0 = fmaf(pj, __ldg(vr + (long)jj * ldkv + lane), o0);
      o1 = fmaf(pj, __ldg(vr + (long)jj * ldkv + lane + 32), o1);
    }
  }
  float* dst = out + (b * N + n) * ldq + h * kDH;
  dst[lane] = o0 / l;
  dst[lane + 32] = o1 / l;
}

constexpr int kNormWarps = 8;

// Lane = chunk of four channels (chunk lane + 32 i, i < MAXI), one row per warp.
template <int MAXI>
__global__ void __launch_bounds__(kNormWarps * 32)
pvt_embed_norm_kernel(const float* __restrict__ tok, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ pos, const float* __restrict__ cls, float* __restrict__ out, long rows,
                      int T, int ntok, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * kNormWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nchunks = C >> 2;
  const long b = row / T;
  const int i = (int)(row - b * T);
  float4* dst = reinterpret_cast<float4*>(out + row * C);
  const float4* pr = reinterpret_cast<const float4*>(pos + (long)i * C);
  if (i < ntok) {   // the class row
    for (int ch = lane; ch < nchunks; ch += 32) {
      const float4 c = __ldg(reinterpret_cast<const float4*>(cls) + ch), p = __ldg(pr + ch);
      dst[ch] = make_float4(c.x + p.x, c.y + p.y, c.z + p.z, c.w + p.w);
    }
    return;
  }
  const float* x = tok + (b * (T - ntok) + (i - ntok)) * C;
  const float inv_c = 1.0f / (float)C;
  float4 v[MAXI];
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    const int ch = lane + 32 * k;
    v[k] = ch < nchunks ? *reinterpret_cast<const float4*>(x + ch * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXI; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
  const float mean = warp_sum(s) * inv_c;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    if (lane + 32 * k < nchunks) {
      const float a = v[k].x - mean, bb = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
      sq += (a * a + bb * bb) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) * inv_c + eps);
#pragma unroll
  for (int k = 0; k < MAXI; ++k) {
    const int ch = lane + 32 * k;
    if (ch < nchunks) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + ch);
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta) + ch);
      const float4 p = __ldg(pr + ch);
      const float y0 = (v[k].x - mean) * rstd * g.x + be.x, y1 = (v[k].y - mean) * rstd * g.y + be.y;
      const float y2 = (v[k].z - mean) * rstd * g.z + be.z, y3 = (v[k].w - mean) * rstd * g.w + be.w;
      dst[ch] = make_float4(y0 + p.x, y1 + p.y, y2 + p.z, y3 + p.w);
    }
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_pvt_sr_attention_bf16(const void* q, const void* kv, void* out, int B, int N, int Nk, int H, int dh,
                                     float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_sr_attention_bf16: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_sr_attention_bf16: head_dim must be 64 (got %d)", dh);
  TFIMM_CHECK_ARG(B <= 65535 && H <= 65535, "pvt_sr_attention_bf16: need B, H <= 65535 (B=%d H=%d)", B, H);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_sr_attention_bf16: q, kv and out must be 16-byte aligned");
  auto kernel = pvt_sr_attention_bf16_kernel;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, kSmem, attr_devs));
  const int ntiles = (N + kRows - 1) / kRows;
  const int tiles = pvt_tiles_per_cta(ntiles, (Nk + kKeys - 1) / kKeys, B, H);
  const dim3 grid((ntiles + tiles - 1) / tiles, H, B);
  kernel<<<grid, kWarps * 32, kSmem, stream>>>(reinterpret_cast<const __nv_bfloat16*>(q),
                                               reinterpret_cast<const __nv_bfloat16*>(kv),
                                               reinterpret_cast<__nv_bfloat16*>(out), N, Nk, H, tiles,
                                               scale * kLog2e);
  TFIMM_LAUNCH_OK("pvt_sr_attention_bf16_kernel");
  return kOk;
}

int tfimm_b200_pvt_sr_attention_f32(const float* q, const float* kv, float* out, int B, int N, int Nk, int H, int dh,
                                    float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && Nk > 0 && H > 0, "pvt_sr_attention_f32: bad shape B=%d N=%d Nk=%d H=%d", B, N,
                  Nk, H);
  TFIMM_CHECK_ARG(dh == kDH, "pvt_sr_attention_f32: head_dim must be 64 (got %d)", dh);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr && aligned(q, 16) && aligned(kv, 16) &&
                      aligned(out, 16),
                  "pvt_sr_attention_f32: q, kv and out must be 16-byte aligned");
  const long rows = (long)B * H * N;
  const long blocks = (rows + kF32Warps - 1) / kF32Warps;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pvt_sr_attention_f32: problem too large (%ld blocks)", blocks);
  pvt_sr_attention_f32_kernel<<<(unsigned)blocks, kF32Warps * 32, 0, stream>>>(q, kv, out, rows, N, Nk, H, scale);
  TFIMM_LAUNCH_OK("pvt_sr_attention_f32_kernel");
  return kOk;
}

int tfimm_b200_pvt_embed_norm(const float* tok, const float* gamma, const float* beta, const float* pos,
                              const float* cls, float* out, int B, int P, int ntok, int C, float eps, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && P > 0 && (ntok == 0 || ntok == 1) && C > 0 && C % 4 == 0 && C <= 1024,
                  "pvt_embed_norm: need B, P > 0, ntok 0 or 1, C %% 4 == 0 and C <= 1024 (B=%d P=%d ntok=%d C=%d)", B,
                  P, ntok, C);
  TFIMM_CHECK_ARG(tok != nullptr && gamma != nullptr && beta != nullptr && pos != nullptr && out != nullptr &&
                      aligned(tok, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(pos, 16) &&
                      aligned(out, 16),
                  "pvt_embed_norm: tok, gamma, beta, pos and out must be 16-byte aligned");
  TFIMM_CHECK_ARG(ntok == 0 || (cls != nullptr && aligned(cls, 16)),
                  "pvt_embed_norm: ntok = 1 needs a 16-byte aligned cls");
  const int T = P + ntok;
  const long rows = (long)B * T;
  const long blocks = (rows + kNormWarps - 1) / kNormWarps;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pvt_embed_norm: problem too large (%ld blocks)", blocks);
  const int maxi = (C / 4 + 31) / 32;
#define TFIMM_PEN(I)                                                                                                 \
  pvt_embed_norm_kernel<I><<<(unsigned)blocks, kNormWarps * 32, 0, stream>>>(tok, gamma, beta, pos, cls, out, rows, \
                                                                             T, ntok, C, eps)
  if (maxi <= 1) TFIMM_PEN(1);
  else if (maxi <= 2) TFIMM_PEN(2);
  else if (maxi <= 4) TFIMM_PEN(4);
  else TFIMM_PEN(8);
#undef TFIMM_PEN
  TFIMM_LAUNCH_OK("pvt_embed_norm_kernel");
  return kOk;
}

}  // extern "C"
