// The register-level core shared by the mma.sync attention kernels.  The ViT bf16 and TF32 kernels (attention.cu), PiT
// (pit.cu) and Segment Anything's relpos attention (relpos_attention.cu) run all of it; Swin window attention
// (window_attention.cu) uses the quad reductions and the P V step.
//
// The algorithm, whose float64 statement is `_softmax_pv` in oracle/emulate_bf16.py (key_block = 64): keys are taken in
// blocks of 64 from key 0.  With logits s in log2 units, keys that do not exist at -inf, m the running row maximum and
// l the running row sum, each block does
//     m_new = max(m, max_j s_j),   alpha = 2^(m - m_new),   p_j = 2^(s_j - m_new),
//     l = alpha l + sum_j p_j,     O = alpha O + round(p) V.
// P is rounded (to bf16, or to TF32) per block, against the running maximum, and l sums the unrounded fp32 p.  At the
// end out = O / l, correctly rounded (div_rn_by).  Window attention is a single block of up to 144 keys with no running
// state, normalised the same way.
//
// Everything here works on one warp's 16-row accumulator tile of m16n8k16 / m16n8k8: thread (g, t) = (lane / 4,
// lane % 4) holds rows g and g + 8, and element e of 8-column tile nt is row g + 8 (e / 2), column 8 nt + 2 t + e % 2.
// Row reductions are over the quad of four t.
#pragma once

#include "common.cuh"

namespace tfimm {

__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// One row's sum l, from the partial sums of the four threads of its quad, and 1 / l.
struct RowNorm {
  float l, inv;
  __device__ __forceinline__ explicit RowNorm(float part) : l(quad_sum(part)), inv(1.0f / l) {}
  // x / l, correctly rounded
  __device__ __forceinline__ float operator()(float x) const { return div_rn_by(x, l, inv); }
};

// The running state of rows g and g + 8.  kEx2Ftz picks ex2.approx.ftz (PiT) over exp2f (the others); the two differ
// where the result is subnormal.
template <bool kEx2Ftz>
struct OnlineSoftmax {
  float m_run[2] = {-INFINITY, -INFINITY};   // in log2 units
  float l_run[2] = {0.f, 0.f};

  static __device__ __forceinline__ float pow2(float x) { return kEx2Ftz ? ex2_approx(x) : exp2f(x); }

  // One block of 64 keys.  s holds the logits in log2 units, with keys that do not exist already -inf; mx holds each
  // row's maximum over this thread's s (the kernels take it as they form the logits).  Every block has a key that
  // exists, so m_new is finite.  Rescales l_run and o, and leaves the unrounded P in s.
  template <int NO>
  __device__ __forceinline__ void update(float (&s)[8][4], float (&o)[NO][4], const float (&mx)[2]) {
    block<false>(s, o, mx, 0.f);
  }
  // The same with raw scores in s and mx: the logits are c s, c = scale log2 e, folded into one fma per score (PiT).
  template <int NO>
  __device__ __forceinline__ void update(float (&s)[8][4], float (&o)[NO][4], const float (&mx)[2], float c) {
    block<true>(s, o, mx, c);
  }

  // row r = 0 (g) or 1 (g + 8)
  __device__ __forceinline__ RowNorm finish(int r) const { return RowNorm(l_run[r]); }

 private:
  template <bool kRaw, int NO>
  __device__ __forceinline__ void block(float (&s)[8][4], float (&o)[NO][4], const float (&mx)[2], float c) {
    float alpha[2], neg_m[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], kRaw ? quad_max(mx[r]) * c : quad_max(mx[r]));
      alpha[r] = pow2(m_run[r] - m_new);
      m_run[r] = m_new;
      neg_m[r] = -m_new;
      l_run[r] *= alpha[r];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = pow2(kRaw ? fmaf(s[nt][e], c, neg_m[e >> 1]) : s[nt][e] + neg_m[e >> 1]);
        s[nt][e] = p;
        l_run[e >> 1] += p;
      }
    }
#pragma unroll
    for (int i = 0; i < NO; ++i) {
      o[i][0] *= alpha[0]; o[i][1] *= alpha[0];
      o[i][2] *= alpha[1]; o[i][3] *= alpha[1];
    }
  }
};

// S = Q K^T over one 64-key block of bf16 rows: s[nt] = q . k for keys 8 nt .. 8 nt + 7.  Only the 16-key chunks that
// begin in the first ntiles 8-key tiles are computed; the others stay 0.  One ldmatrix.x4 gives the k16 B fragments of
// two 8-key tiles.  kaddr(row, chunk): shared address of 16-byte chunk `chunk` of the block's key `row`.
template <int KS, class KAddr>
__device__ __forceinline__ void qk_bf16(float (&s)[8][4], const uint32_t (&qf)[KS][4], int ntiles, int lane,
                                        KAddr kaddr) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
  for (int np = 0; np < 4; ++np) {
    if (2 * np < ntiles) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const int row = np * 16 + (lane >> 4) * 8 + (lane & 7);
        const int chunk = ks * 2 + ((lane >> 3) & 1);
        uint32_t k0, k1, k2, k3;
        ldmatrix_x4(kaddr(row, chunk), k0, k1, k2, k3);
        mma_bf16_16816(s[2 * np], qf[ks], k0, k1);
        mma_bf16_16816(s[2 * np + 1], qf[ks], k2, k3);
      }
    }
  }
}

// O += round_bf16(P) V over the 16-key chunks that begin in the first ntiles 8-key tiles (P is 0 past them).  P's
// accumulator layout is the A-fragment layout, so P never leaves its thread; V comes by ldmatrix.trans, two 8-column
// tiles per x4.  vaddr(row, chunk): shared address of 16-byte chunk `chunk` of the block's value `row`.
template <int NT, int NO, class VAddr>
__device__ __forceinline__ void pv_bf16(float (&o)[NO][4], const float (&s)[NT][4], int ntiles, int lane, VAddr vaddr) {
#pragma unroll
  for (int kk = 0; kk < NT / 2; ++kk) {
    if (2 * kk < ntiles) {
      uint32_t a[4];
      a[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int jp = 0; jp < NO / 2; ++jp) {
        const int row = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int chunk = 2 * jp + (lane >> 4);
        uint32_t v0, v1, v2, v3;
        ldmatrix_x4_trans(vaddr(row, chunk), v0, v1, v2, v3);
        mma_bf16_16816(o[2 * jp], a, v0, v1);
        mma_bf16_16816(o[2 * jp + 1], a, v2, v3);
      }
    }
  }
}

}  // namespace tfimm
