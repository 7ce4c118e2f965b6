// Kernels of the CaiT family (tfimm/architectures/cait.py): talking-heads self-attention and class attention.  The
// blocks' LayerNorms, GEMMs and MLPs, the patch embedding and the head run on the existing paths.
//
// Talking-heads attention (Shazeer et al. 2020) mixes the H heads' logits before the softmax and the H probability
// rows again after it:
//     S_h = q_h k_h^T,   L_g = sum_h wl[h, g] S_h + bl[g],   P_g = softmax_keys(L_g),   P'_f = sum_g P_g ww[g, f] + bw[f],
//     O_f = P'_f V_f.
// The launcher passes wl with dh^-0.5 log2 e folded in and bl with log2 e folded in, so L is in log2 units.  The
// post-mix needs every head's normalised P, so the kernels take two passes over the keys: the first finds each
// (query, g) row maximum m_g and sum l_g of 2^(L_g - m_g); the second recomputes S, mixes, normalises exactly
// (P_g = 2^(L_g - m_g) / l_g, correctly rounded), post-mixes and accumulates P' V.  Keys past N are masked on L,
// after the pre-mix (a zero K row gives L_g = bl[g], and -inf S times a weight of either sign is not -inf), and V rows
// past N are zero (P'_f = bw[f] at every key).
//
// cait_talking_heads_bf16_kernel<H, R, NW>  dh 48; one CTA holds all H heads of R query rows of one image, NW warps.
//   - Q is loaded once and held as mma.sync A fragments: warp w owns the (16-row tile, head) pairs w PPW .. w PPW + PPW - 1.
//   - Keys come in blocks of kKB = 32 for all heads: K and V one buffer each, (D + 8) bf16 per row (6H + 1 sixteen-byte
//     chunks, odd, so ldmatrix phases are conflict-free).  V(kb) is copied while S(kb) and the mix run, K(kb + 1)
//     while the mix and P V run.
//   - Each block's S of every pair goes to shared memory (fp32, rows of kKB + 8 floats), where the mixing threads read
//     all H heads of one (query, key): thread (r, j) takes query r and keys j, j + TPR, ..., the H^2-FMA mixes run in
//     fp32 on the CUDA cores with the weights read from shared memory.
//   - Pass 1 keeps per-thread (m_g, l_g) over its keys (one ex2 per key and g), merged over the TPR threads of a row
//     by shuffles and left in shared memory.  Pass 2 writes P' rounded once to bf16 into shared memory ([f][r][key],
//     80-byte rows), from which the PV warps load A fragments by ldmatrix; V by ldmatrix.trans.
//   - The output needs no final division (P was normalised); it is rounded to bf16 once, staged through shared memory
//     and stored as 16-byte chunks.
// cait_talking_heads_f32_kernel<H>  the same two passes in fp32 on the CUDA cores, any dh % 4 == 0 up to 64, 16 query
//   rows and 16-key blocks per CTA; thread (r, k) forms all H logits of its (query, key) pair itself.  exp2f and IEEE
//   division.
// cait_add_pos_kernel  the patch tokens' position embedding, added in place to the fp32 stream (the class token is
//   prepended only after the self-attention blocks, without one).
// cait_class_attn_kernel<T, DH>  out = softmax(scale q k^T) v for one query per (image, head), any number of keys:
//   each of 128 threads runs an online softmax over keys tid, tid + 128, ..., and the CTA merges the 128 partial
//   states at the end.  exp2f, one division per output.
#include "attention_mma.cuh"
#include "common.cuh"
#include "tfimm_b200_cait.h"

namespace tfimm {
namespace {

constexpr int kDH = 48;
constexpr int kKB = 32;           // keys per block (bf16 kernel)
constexpr int kSRow = kKB + 8;    // fp32 logits row: float2 stores of a quad-row tile are conflict-free
constexpr int kPRow = kKB + 8;    // bf16 P' row: 80 bytes, five 16-byte chunks

template <int H, int R, int NW>
struct THShape {
  static constexpr int D = H * kDH;
  static constexpr int kThreads = NW * 32;
  static constexpr int kPPW = (R / 16) * H / NW;   // (row tile, head) pairs per warp
  static constexpr int kTPR = kThreads / R;        // mixing threads per query row
  static constexpr int kKPT = kKB / kTPR;          // keys per mixing thread per block
  static constexpr int kRowBytes = (D + 8) * 2;
  static constexpr int kKVBytes = kKB * kRowBytes;
  static constexpr int kSBytes = H * R * kSRow * 4;
  static constexpr int kPBytes = H * R * kPRow * 2;
  static constexpr int kStatBytes = 3 * R * H * 4;            // m, l, 1 / l per (query, g)
  static constexpr int kWBytes = (2 * H * H + 2 * H) * 4;     // wl | ww | bl | bw
  static constexpr int kSmem = 2 * kKVBytes + kSBytes + kPBytes + kStatBytes + kWBytes;
  static_assert((R / 16) * H % NW == 0 && kThreads % R == 0 && kKB % kTPR == 0 && 32 % kTPR == 0, "shape");
  static_assert(R * kRowBytes <= kSBytes, "Q and the output tile are staged in the logits buffer");
  static_assert(kSmem <= 227 * 1024, "shared memory");
};

// L[g] = bl[g] + sum_h w[h, g] S[h]
template <int H>
__device__ __forceinline__ void premix(float (&L)[H], const float (&S)[H], const float* w, const float* b) {
#pragma unroll
  for (int g = 0; g < H; ++g) L[g] = b[g];
#pragma unroll
  for (int h = 0; h < H; ++h)
#pragma unroll
    for (int g = 0; g < H; ++g) L[g] = fmaf(w[h * H + g], S[h], L[g]);
}

// (m, l) <- the state of (m, l) and one more logit x (finite), one exponential: the larger maximum rescales the other
template <bool kApprox>
__device__ __forceinline__ void online_add(float& m, float& l, float x) {
  const float d = x - m;   // +inf while m = -inf
  const float e = kApprox ? ex2_approx(-fabsf(d)) : exp2f(-fabsf(d));
  if (d > 0.f) { l = fmaf(l, e, 1.f); m = x; } else { l += e; }
}
// (m, l) <- the merge of (m, l) and (mo, lo); a state with m = -inf holds nothing
template <bool kApprox>
__device__ __forceinline__ void online_merge(float& m, float& l, float mo, float lo) {
  if (mo == -INFINITY) return;
  const float d = mo - m;
  const float e = kApprox ? ex2_approx(-fabsf(d)) : exp2f(-fabsf(d));
  if (d > 0.f) { l = fmaf(l, e, lo); m = mo; } else { l = fmaf(lo, e, l); }
}

template <int H, int R, int NW>
__global__ void __launch_bounds__(NW * 32)
cait_talking_heads_bf16_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                               const float* __restrict__ wl, const float* __restrict__ bl,
                               const float* __restrict__ ww, const float* __restrict__ bw, int N) {
  using S = THShape<H, R, NW>;
  constexpr int D = S::D, RB = S::kRowBytes, CH = D / 8, PPW = S::kPPW, TPR = S::kTPR, KPT = S::kKPT;
  constexpr int NT = NW * 32;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sK = smem_u32(smem), sV = sK + S::kKVBytes;
  float* sS = reinterpret_cast<float*>(smem + 2 * S::kKVBytes);
  __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(smem + 2 * S::kKVBytes + S::kSBytes);
  float* sM = reinterpret_cast<float*>(smem + 2 * S::kKVBytes + S::kSBytes + S::kPBytes);
  float* sL = sM + R * H;
  float* sInv = sL + R * H;
  float* sWl = sInv + R * H;
  float* sWw = sWl + H * H;
  float* sBl = sWw + H * H;
  float* sBw = sBl + H;
  const uint32_t sQ = smem_u32(sS), sPa = smem_u32(sP);

  const int b = blockIdx.y, q_base = blockIdx.x * R;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long ld = 3L * D;
  const __nv_bfloat16* base = qkv + (long)b * N * ld;
  const int nblocks = (N + kKB - 1) / kKB;

  auto load_rows = [&](uint32_t dst, int row0, int nrows, int col) {
    for (int idx = tid; idx < nrows * CH; idx += NT) {
      const int r = idx / CH, c = idx - r * CH;
      const int row = row0 + r;
      const bool valid = row < N;
      cp_async_16(dst + r * RB + c * 16, base + (long)(valid ? row : 0) * ld + col + c * 8, valid);
    }
  };

  for (int i = tid; i < H * H; i += NT) { sWl[i] = wl[i]; sWw[i] = ww[i]; }
  for (int i = tid; i < H; i += NT) { sBl[i] = bl[i]; sBw[i] = bw[i]; }
  load_rows(sQ, q_base, R, 0);
  load_rows(sK, 0, kKB, D);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();

  uint32_t qf[PPW][3][4];
#pragma unroll
  for (int i = 0; i < PPW; ++i) {
    const int p = warp * PPW + i, rt = p / H, h = p % H;
#pragma unroll
    for (int ks = 0; ks < 3; ++ks)
      ldmatrix_x4(sQ + (rt * 16 + (lane & 15)) * RB + (h * 6 + ks * 2 + (lane >> 4)) * 16, qf[i][ks][0], qf[i][ks][1],
                  qf[i][ks][2], qf[i][ks][3]);
  }

  // S of this warp's pairs over the key block in sK -> sS[h][row][key]
  auto logits = [&](int nvalid) {
    const int ntiles = min(4, (nvalid + 7) >> 3);
#pragma unroll
    for (int i = 0; i < PPW; ++i) {
      const int p = warp * PPW + i, rt = p / H, h = p % H;
      float s[8][4];
      qk_bf16(s, qf[i], ntiles, lane, [&](int row, int chunk) { return sK + row * RB + (h * 6 + chunk) * 16; });
      float* dst = sS + (h * R + rt * 16 + g) * kSRow + 2 * t;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        *reinterpret_cast<float2*>(dst + nt * 8) = make_float2(s[nt][0], s[nt][1]);
        *reinterpret_cast<float2*>(dst + 8 * kSRow + nt * 8) = make_float2(s[nt][2], s[nt][3]);
      }
    }
  };
  const int mr = tid / TPR, mj = tid - mr * TPR;   // this thread's mixing row and first key
  auto mix_in = [&](float (&L)[H], int k) {
    float Sv[H];
#pragma unroll
    for (int h = 0; h < H; ++h) Sv[h] = sS[(h * R + mr) * kSRow + k];
    premix<H>(L, Sv, sWl, sBl);
  };

  // ---- pass 1: row maxima and sums of 2^L
  float m[H], l[H];
#pragma unroll
  for (int i = 0; i < H; ++i) { m[i] = -INFINITY; l[i] = 0.f; }
#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    cp_async_wait<0>();   // K(kb)
    __syncthreads();      // ... for every thread; the last block's statistics are done with sS
    const int key0 = kb * kKB, nvalid = min(kKB, N - key0);
    logits(nvalid);
    __syncthreads();
    load_rows(sK, ((kb + 1) % nblocks) * kKB, kKB, D);   // the next block, or block 0 for pass 2
    cp_async_commit();
#pragma unroll 1
    for (int i = 0; i < KPT; ++i) {
      const int k = mj + i * TPR;
      if (k >= nvalid) break;
      float L[H];
      mix_in(L, k);
#pragma unroll
      for (int c = 0; c < H; ++c) online_add<true>(m[c], l[c], L[c]);
    }
  }
#pragma unroll
  for (int off = 1; off < TPR; off <<= 1)
#pragma unroll
    for (int c = 0; c < H; ++c) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[c], off), lo = __shfl_xor_sync(0xffffffffu, l[c], off);
      online_merge<true>(m[c], l[c], mo, lo);
    }
  if (mj == 0) {
#pragma unroll
    for (int c = 0; c < H; ++c) {
      sM[mr * H + c] = m[c];
      sL[mr * H + c] = l[c];
      sInv[mr * H + c] = 1.0f / l[c];
    }
  }

  // ---- pass 2: normalised, post-mixed probabilities, O += round_bf16(P') V
  float o[PPW][6][4];
#pragma unroll
  for (int i = 0; i < PPW; ++i)
#pragma unroll
    for (int n = 0; n < 6; ++n) o[i][n][0] = o[i][n][1] = o[i][n][2] = o[i][n][3] = 0.f;
#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    cp_async_wait<0>();   // K(kb)
    __syncthreads();      // ... for every thread; P V of kb - 1 is done with sV and sP; the statistics are stored
    const int key0 = kb * kKB, nvalid = min(kKB, N - key0);
    load_rows(sV, key0, kKB, 2 * D);
    cp_async_commit();
    logits(nvalid);
    __syncthreads();
    if (kb + 1 < nblocks) load_rows(sK, key0 + kKB, kKB, D);
    cp_async_commit();
#pragma unroll 1
    for (int i = 0; i < KPT; ++i) {
      const int k = mj + i * TPR;
      float L[H];
      mix_in(L, k);
#pragma unroll
      for (int c = 0; c < H; ++c)   // L becomes P
        L[c] = k < nvalid ? div_rn_by(ex2_approx(L[c] - sM[mr * H + c]), sL[mr * H + c], sInv[mr * H + c]) : 0.f;
#pragma unroll
      for (int f = 0; f < H; ++f) {
        float acc = sBw[f];
#pragma unroll
        for (int c = 0; c < H; ++c) acc = fmaf(L[c], sWw[c * H + f], acc);
        sP[(f * R + mr) * kPRow + k] = __float2bfloat16_rn(acc);
      }
    }
    cp_async_wait<1>();   // V(kb); K(kb + 1) may still be in flight
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PPW; ++i) {
      const int p = warp * PPW + i, rt = p / H, f = p % H;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        if (kk * 16 >= nvalid) break;
        uint32_t a[4];
        ldmatrix_x4(sPa + ((f * R + rt * 16 + (lane & 15)) * kPRow + kk * 16 + (lane >> 4) * 8) * 2, a[0], a[1], a[2],
                    a[3]);
#pragma unroll
        for (int jp = 0; jp < 3; ++jp) {
          const int row = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          const int chunk = f * 6 + 2 * jp + (lane >> 4);
          uint32_t v0, v1, v2, v3;
          ldmatrix_x4_trans(sV + row * RB + chunk * 16, v0, v1, v2, v3);
          mma_bf16_16816(o[i][2 * jp], a, v0, v1);
          mma_bf16_16816(o[i][2 * jp + 1], a, v2, v3);
        }
      }
    }
  }
  cp_async_wait<0>();   // only empty groups can be pending here

  // ---- output: bf16 tile staged in the logits buffer (read last by the final mix, before the last barrier)
  uint8_t* tile = reinterpret_cast<uint8_t*>(sS);
#pragma unroll
  for (int i = 0; i < PPW; ++i) {
    const int p = warp * PPW + i, rt = p / H, f = p % H;
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      uint8_t* dst = tile + (rt * 16 + g) * RB + (f * kDH + nt * 8 + 2 * t) * 2;
      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(o[i][nt][0], o[i][nt][1]);
      *reinterpret_cast<uint32_t*>(dst + 8 * RB) = pack_bf16x2(o[i][nt][2], o[i][nt][3]);
    }
  }
  __syncthreads();
  for (int idx = tid; idx < R * CH; idx += NT) {
    const int r = idx / CH, c = idx - r * CH;
    const int row = q_base + r;
    if (row < N)
      *reinterpret_cast<uint4*>(out + ((long)b * N + row) * D + c * 8) =
          *reinterpret_cast<const uint4*>(tile + r * RB + c * 16);
  }
}

template <int H, int R, int NW>
int launch_th_bf16(const __nv_bfloat16* qkv, __nv_bfloat16* out, const float* wl, const float* bl, const float* ww,
                   const float* bw, int B, int N, cudaStream_t stream) {
  using S = THShape<H, R, NW>;
  auto kernel = cait_talking_heads_bf16_kernel<H, R, NW>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, S::kSmem, attr_devs));
  const dim3 grid((N + R - 1) / R, B);
  kernel<<<grid, NW * 32, S::kSmem, stream>>>(qkv, out, wl, bl, ww, bw, N);
  TFIMM_LAUNCH_OK("cait_talking_heads_bf16_kernel");
  return kOk;
}

// ------------------------------------------------------------------------------------------------ fp32 SIMT kernel
constexpr int kFRows = 16, kFKeys = 16, kFThreads = kFRows * kFKeys;
constexpr int kFMaxDh = 64;

struct F32Shape {
  int D, row;   // row: padded shared-memory row of Q, K and V in floats
  __host__ __device__ F32Shape(int H, int dh) : D(H * dh), row(H * dh + 4) {}
  __host__ __device__ int smem(int H) const {
    return (3 * kFRows * row + H * kFRows * (kFKeys + 1) + 2 * H * H + 2 * H) * 4 + D * 4;
  }
};

template <int H>
__global__ void __launch_bounds__(kFThreads)
cait_talking_heads_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, const float* __restrict__ wl,
                              const float* __restrict__ bl, const float* __restrict__ ww,
                              const float* __restrict__ bw, int N, int dh) {
  const F32Shape S(H, dh);
  const int D = S.D, RW = S.row, D4 = D / 4;
  extern __shared__ __align__(16) float fsm[];
  float* sQ = fsm;
  float* sK = sQ + kFRows * RW;
  float* sV = sK + kFKeys * RW;
  float* sP = sV + kFKeys * RW;                  // [f][r][key], rows of kFKeys + 1
  float* sWl = sP + H * kFRows * (kFKeys + 1);
  float* sWw = sWl + H * H;
  float* sBl = sWw + H * H;
  float* sBw = sBl + H;
  int* sF = reinterpret_cast<int*>(sBw + H);     // column -> offset of its head's P' rows

  const int b = blockIdx.y, q_base = blockIdx.x * kFRows;
  const int tid = threadIdx.x, r = tid / kFKeys, kj = tid % kFKeys;
  const long ld = 3L * D;
  const float* base = qkv + (long)b * N * ld;
  const int nblocks = (N + kFKeys - 1) / kFKeys;

  for (int i = tid; i < H * H; i += kFThreads) { sWl[i] = wl[i]; sWw[i] = ww[i]; }
  for (int i = tid; i < H; i += kFThreads) { sBl[i] = bl[i]; sBw[i] = bw[i]; }
  for (int c = tid; c < D; c += kFThreads) sF[c] = (c / dh) * kFRows * (kFKeys + 1);
  auto load_rows = [&](float* dst, int row0, int col) {
    for (int idx = tid; idx < kFRows * D4; idx += kFThreads) {
      const int rr = idx / D4, c = idx - rr * D4;
      const int row = row0 + rr;
      const bool valid = row < N;
      cp_async_16(smem_u32(dst + rr * RW + c * 4), base + (long)(valid ? row : 0) * ld + col + c * 4, valid);
    }
  };
  load_rows(sQ, q_base, 0);

  auto logits = [&](float (&L)[H]) {
    float Sv[H];
    const float* q = sQ + r * RW;
    const float* k = sK + kj * RW;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      float acc = 0.f;
      for (int d = h * dh; d < (h + 1) * dh; d += 4) {
        const float4 a = *reinterpret_cast<const float4*>(q + d), c = *reinterpret_cast<const float4*>(k + d);
        acc = fmaf(a.x, c.x, acc); acc = fmaf(a.y, c.y, acc); acc = fmaf(a.z, c.z, acc); acc = fmaf(a.w, c.w, acc);
      }
      Sv[h] = acc;
    }
    premix<H>(L, Sv, sWl, sBl);
  };

  float m[H], l[H];
#pragma unroll
  for (int i = 0; i < H; ++i) { m[i] = -INFINITY; l[i] = 0.f; }
#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    __syncthreads();   // every thread is done with the previous block's K
    load_rows(sK, kb * kFKeys, D);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if (kb * kFKeys + kj < N) {
      float L[H];
      logits(L);
#pragma unroll
      for (int c = 0; c < H; ++c) online_add<false>(m[c], l[c], L[c]);
    }
  }
#pragma unroll
  for (int off = 1; off < kFKeys; off <<= 1)
#pragma unroll
    for (int c = 0; c < H; ++c) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[c], off), lo = __shfl_xor_sync(0xffffffffu, l[c], off);
      online_merge<false>(m[c], l[c], mo, lo);
    }

  constexpr int kMaxCols = H * kFMaxDh / kFKeys;   // output columns per thread: kj, kj + 16, ...
  float o[kMaxCols];
#pragma unroll
  for (int i = 0; i < kMaxCols; ++i) o[i] = 0.f;
#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    __syncthreads();   // every thread is done with the previous block's K, V and P'
    load_rows(sK, kb * kFKeys, D);
    load_rows(sV, kb * kFKeys, 2 * D);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    const bool valid = kb * kFKeys + kj < N;
    float L[H];
    logits(L);
    float Pn[H];
#pragma unroll
    for (int c = 0; c < H; ++c) Pn[c] = valid ? exp2f(L[c] - m[c]) / l[c] : 0.f;
#pragma unroll
    for (int f = 0; f < H; ++f) {
      float acc = sBw[f];
#pragma unroll
      for (int c = 0; c < H; ++c) acc = fmaf(Pn[c], sWw[c * H + f], acc);
      sP[(f * kFRows + r) * (kFKeys + 1) + kj] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kMaxCols; ++i) {
      const int c = kj + i * kFKeys;
      if (c < D) {
        const float* p = sP + sF[c] + r * (kFKeys + 1);
        float acc = o[i];
#pragma unroll
        for (int k = 0; k < kFKeys; ++k) acc = fmaf(p[k], sV[k * RW + c], acc);
        o[i] = acc;
      }
    }
  }
  const int row = q_base + r;
  if (row < N) {
#pragma unroll
    for (int i = 0; i < kMaxCols; ++i) {
      const int c = kj + i * kFKeys;
      if (c < D) out[((long)b * N + row) * D + c] = o[i];
    }
  }
}

template <int H>
int launch_th_f32(const float* qkv, float* out, const float* wl, const float* bl, const float* ww, const float* bw,
                  int B, int N, int dh, cudaStream_t stream) {
  auto kernel = cait_talking_heads_f32_kernel<H>;
  const int smem = F32Shape(H, dh).smem(H);
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, F32Shape(H, kFMaxDh).smem(H), attr_devs));
  const dim3 grid((N + kFRows - 1) / kFRows, B);
  kernel<<<grid, kFThreads, smem, stream>>>(qkv, out, wl, bl, ww, bw, N, dh);
  TFIMM_LAUNCH_OK("cait_talking_heads_f32_kernel");
  return kOk;
}

// ------------------------------------------------------------------------------------------------ class attention
constexpr int kCThreads = 128;

__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }

template <typename T, int DH>
__global__ void __launch_bounds__(kCThreads)
cait_class_attn_kernel(const T* __restrict__ q, const T* __restrict__ kv, T* __restrict__ out, int Tk, int H,
                       float scale_log2) {
  __shared__ float sq[DH];
  __shared__ float sacc[kCThreads][DH + 1];
  __shared__ float sc[kCThreads], sred[kCThreads / 32];
  const int b = blockIdx.y, h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int D = H * DH;
  for (int d = tid; d < DH; d += kCThreads) sq[d] = to_f(q[(long)b * D + h * DH + d]);
  __syncthreads();

  float m = -INFINITY, l = 0.f, acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
  const T* base = kv + (long)b * Tk * 2 * D + h * DH;
#pragma unroll 1
  for (int j = tid; j < Tk; j += kCThreads) {
    const T* k = base + (long)j * 2 * D;
    const T* v = k + D;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DH; ++d) s = fmaf(sq[d], to_f(k[d]), s);
    s *= scale_log2;
    const float dlt = s - m;
    const float e = exp2f(-fabsf(dlt));
    if (dlt > 0.f) {   // new maximum: rescale what is there, this key weighs 1
      l = fmaf(l, e, 1.f);
      m = s;
#pragma unroll
      for (int d = 0; d < DH; ++d) acc[d] = fmaf(acc[d], e, to_f(v[d]));
    } else {
      l += e;
#pragma unroll
      for (int d = 0; d < DH; ++d) acc[d] = fmaf(e, to_f(v[d]), acc[d]);
    }
  }
  const float wm = warp_max(m);
  if (lane == 0) sred[warp] = wm;
  __syncthreads();
  float M = sred[0];
#pragma unroll
  for (int w = 1; w < kCThreads / 32; ++w) M = fmaxf(M, sred[w]);
  const float c = m == -INFINITY ? 0.f : exp2f(m - M);
  sc[tid] = c;
#pragma unroll
  for (int d = 0; d < DH; ++d) sacc[tid][d] = acc[d];
  const float ls = warp_sum(l * c);
  __syncthreads();   // sred is read by everyone before it is overwritten
  if (lane == 0) sred[warp] = ls;
  __syncthreads();
  float Lsum = 0.f;
#pragma unroll
  for (int w = 0; w < kCThreads / 32; ++w) Lsum += sred[w];
  for (int d = tid; d < DH; d += kCThreads) {
    float o = 0.f;
    for (int i = 0; i < kCThreads; ++i) o = fmaf(sc[i], sacc[i][d], o);
    st_from_float(out + (long)b * D + h * DH + d, o / Lsum);
  }
}

template <typename T>
int launch_class_attn(const T* q, const T* kv, T* out, int B, int Tk, int H, int dh, float scale,
                      cudaStream_t stream) {
  const dim3 grid(H, B);
  const float c = scale * kLog2e;
  if (dh == 32) cait_class_attn_kernel<T, 32><<<grid, kCThreads, 0, stream>>>(q, kv, out, Tk, H, c);
  else if (dh == 48) cait_class_attn_kernel<T, 48><<<grid, kCThreads, 0, stream>>>(q, kv, out, Tk, H, c);
  else cait_class_attn_kernel<T, 64><<<grid, kCThreads, 0, stream>>>(q, kv, out, Tk, H, c);
  TFIMM_LAUNCH_OK("cait_class_attn_kernel");
  return kOk;
}

// x[b, n, :] += pos[n, :] over the fp32 (B * N, D) stream, four floats per thread
__global__ void cait_add_pos_kernel(float4* __restrict__ x, const float4* __restrict__ pos, long total, int per_image) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float4 p = __ldg(pos + i % per_image);
  float4 v = x[i];
  v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
  x[i] = v;
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_cait_talking_heads_bf16(const void* qkv, void* out, const float* wl, const float* bl, const float* ww,
                                       const float* bw, int B, int N, int H, int dh, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0, "cait_talking_heads_bf16: bad shape B=%d N=%d H=%d", B, N, H);
  TFIMM_CHECK_ARG(dh == 48 && (H == 4 || H == 6 || H == 8 || H == 16),
                  "cait_talking_heads_bf16: need head_dim 48 and H in {4, 6, 8, 16} (got H=%d dh=%d)", H, dh);
  TFIMM_CHECK_ARG(B <= 65535, "cait_talking_heads_bf16: need B <= 65535 (B=%d)", B);
  TFIMM_CHECK_ARG(qkv != nullptr && out != nullptr && wl != nullptr && bl != nullptr && ww != nullptr &&
                      bw != nullptr && aligned(qkv, 16) && aligned(out, 16),
                  "cait_talking_heads_bf16: need 16-byte aligned qkv and out and all four mixing tensors");
  auto q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  auto o = reinterpret_cast<__nv_bfloat16*>(out);
  switch (H) {
    case 4: return launch_th_bf16<4, 64, 8>(q, o, wl, bl, ww, bw, B, N, stream);
    case 6: return launch_th_bf16<6, 64, 8>(q, o, wl, bl, ww, bw, B, N, stream);
    case 8: return launch_th_bf16<8, 64, 16>(q, o, wl, bl, ww, bw, B, N, stream);
    default: return launch_th_bf16<16, 32, 16>(q, o, wl, bl, ww, bw, B, N, stream);
  }
}

int tfimm_b200_cait_talking_heads_f32(const float* qkv, float* out, const float* wl, const float* bl, const float* ww,
                                      const float* bw, int B, int N, int H, int dh, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0, "cait_talking_heads_f32: bad shape B=%d N=%d H=%d", B, N, H);
  TFIMM_CHECK_ARG((H <= 4 || H == 6 || H == 8 || H == 12 || H == 16) && dh > 0 && dh <= kFMaxDh && dh % 4 == 0,
                  "cait_talking_heads_f32: need H in {1, 2, 3, 4, 6, 8, 12, 16} and head_dim a multiple of 4 up to 64 "
                  "(got H=%d dh=%d)", H, dh);
  TFIMM_CHECK_ARG(B <= 65535, "cait_talking_heads_f32: need B <= 65535 (B=%d)", B);
  TFIMM_CHECK_ARG(qkv != nullptr && out != nullptr && wl != nullptr && bl != nullptr && ww != nullptr &&
                      bw != nullptr && aligned(qkv, 16),
                  "cait_talking_heads_f32: need a 16-byte aligned qkv, out and all four mixing tensors");
  switch (H) {
#define TFIMM_CAIT_F32_CASE(h) \
  case h: return launch_th_f32<h>(qkv, out, wl, bl, ww, bw, B, N, dh, stream);
    TFIMM_CAIT_F32_CASE(1) TFIMM_CAIT_F32_CASE(2) TFIMM_CAIT_F32_CASE(3) TFIMM_CAIT_F32_CASE(4)
    TFIMM_CAIT_F32_CASE(6) TFIMM_CAIT_F32_CASE(8) TFIMM_CAIT_F32_CASE(12)
    default: return launch_th_f32<16>(qkv, out, wl, bl, ww, bw, B, N, dh, stream);
#undef TFIMM_CAIT_F32_CASE
  }
}

int tfimm_b200_cait_class_attention(const void* q, const void* kv, void* out, int dtype, int B, int T, int H, int dh,
                                    float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && T > 0 && H > 0, "cait_class_attention: bad shape B=%d T=%d H=%d", B, T, H);
  TFIMM_CHECK_ARG(dh == 32 || dh == 48 || dh == 64, "cait_class_attention: head_dim must be 32, 48 or 64 (got %d)",
                  dh);
  TFIMM_CHECK_ARG(dtype == kF32 || dtype == kBF16, "cait_class_attention: dtype must be float32 or bfloat16");
  TFIMM_CHECK_ARG(B <= 65535 && H <= 65535, "cait_class_attention: need B, H <= 65535 (B=%d H=%d)", B, H);
  TFIMM_CHECK_ARG(q != nullptr && kv != nullptr && out != nullptr, "cait_class_attention: null pointer");
  if (dtype == kBF16)
    return launch_class_attn(reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(kv),
                             reinterpret_cast<__nv_bfloat16*>(out), B, T, H, dh, scale, stream);
  return launch_class_attn(reinterpret_cast<const float*>(q), reinterpret_cast<const float*>(kv),
                           reinterpret_cast<float*>(out), B, T, H, dh, scale, stream);
}

int tfimm_b200_cait_add_pos(float* x, const float* pos, int B, int N, int D, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && D > 0 && D % 4 == 0, "cait_add_pos: need B, N > 0 and D %% 4 == 0 (B=%d N=%d D=%d)",
                  B, N, D);
  TFIMM_CHECK_ARG(x != nullptr && pos != nullptr && aligned(x, 16) && aligned(pos, 16),
                  "cait_add_pos: x and pos must be 16-byte aligned");
  const long total = (long)B * N * (D / 4);
  const long blocks = (total + 255) / 256;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "cait_add_pos: problem too large (%ld blocks)", blocks);
  cait_add_pos_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<float4*>(x),
                                                           reinterpret_cast<const float4*>(pos), total, N * (D / 4));
  TFIMM_LAUNCH_OK("cait_add_pos_kernel");
  return kOk;
}

}  // extern "C"
