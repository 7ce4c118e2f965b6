// Epilogue shared by the wgmma GEMM kernels (gemm_sm90.cu, the fc2 half of mlp_sm90.cu):
//     C = residual + gamma * act(acc + bias)            (or act(residual + ...) with act_post)
// epilogue_staged (plain GEMM) goes through a shared-memory tile with TMA in and out; epilogue_frag works on global
// memory straight from a warpgroup's accumulator fragments (wgmma.cuh).  In both, each thread owns two rows (r, r + 8) and, per
// 8-column group, two adjacent columns of each, so bias / gamma / activation run on packed fp32 pairs and the residual
// load and output store are one 4- or 8-byte access per row and group.  The residual may alias the output (in-place
// fp32 residual stream): every element is read and written by the same thread.
#pragma once
#include "common.cuh"

namespace tfimm {

struct GemmParams {
  int M, N, K;
  const float* bias;   // [N] or null
  const float* gamma;  // [N] or null
  int act;
  int has_res;
  int act_post;  // 1: activation applied after the residual add (ResNet: act(x + shortcut))
  void* c;             // output, row stride ldc elements (plain GEMM) or NHWC [B][Ho][Wo][N] (implicit convolution)
  const void* res;     // residual, same layout as c (row stride ldr), or null
  long ldc, ldr;
  // Squeeze-excite gate folded into the A operand (gemm_sm90.cu, gated instances): row m of A is multiplied by
  // a_scale[m / a_rows_per_img][k] (fp32 [a_imgs][K]) and rounded back to bf16 in shared memory, between the TMA load
  // and the MMA -- the values the separate scale_channels pass used to write to HBM.
  const float* a_scale;
  int a_rows_per_img, a_imgs;
  // Implicit convolution (gemm_sm90.cu): the A operand is not a matrix but the NHWC input itself.  A tile's 128
  // rows are a patch of cv_pb images x cv_ph rows x cv_pw columns of OUTPUT pixels; k-block kb is tap
  // (ky, kx) = kb / (C/64) and 64 input channels, fetched as ONE 4-D TMA box whose out-of-bounds elements are
  // the zero padding.  C and the residual are NHWC [cv_B][cv_Ho][cv_Wo][N].
  int conv;                  // 0: plain GEMM
  int cv_cblocks;            // C / 64
  int cv_ks, cv_stride, cv_pad;
  int cv_pb, cv_ph, cv_pw;
  int cv_tiles_x, cv_tiles_y;  // patch grid per image group (x fastest, then y, then image group)
  int cv_B, cv_Ho, cv_Wo;
  // Token mixing (gemm_sm90.cu, kModeToken) and the channel GLU (kModeGluCols).  Token mixing: the tile grid is
  // images x (M / 128) x (N / BLOCK_N); A is the transposed Dense kernel Wt[M][K] (K = tokens in), B the activation
  // X[image][K][N] read MN-major, and output row m of image b lives at b * img_c + m * ldc (residual: img_r, ldr).
  // bias is per output ROW; rows >= m_out are not stored.  glu: A rows come in groups of 16 -- 8 value rows, then
  // their 8 gate rows -- and stored row 8 (m / 16) + m % 8 is value * act(gate) (kModeGluCols: columns 2j, 2j + 1 are
  // value and gate of stored column j).  mul: elementwise multiplier in the output's element type (the gMLP gate's u
  // half), row stride ld_mul and image stride img_mul.
  int tk_imgs, m_out, glu;
  long img_c, img_r;
  const void* mul;
  long ld_mul, img_mul;
};

// Element offset of output row `r` (0..127) of tile m_blk, or -1 when the row lies outside the output.
__device__ __forceinline__ long epilogue_row_offset(const GemmParams& p, int m_blk, int r, long ld) {
  if (p.conv == 0) {
    const long m = (long)m_blk * 128 + r;
    return m < p.M ? m * ld : -1;
  }
  const int tx = m_blk % p.cv_tiles_x, tyb = m_blk / p.cv_tiles_x;
  const int ty = tyb % p.cv_tiles_y, tb = tyb / p.cv_tiles_y;
  const int per_img = p.cv_ph * p.cv_pw;
  const int b = tb * p.cv_pb + r / per_img;
  const int y = ty * p.cv_ph + (r % per_img) / p.cv_pw;
  const int x = tx * p.cv_pw + r % p.cv_pw;
  if (b >= p.cv_B || y >= p.cv_Ho || x >= p.cv_Wo) return -1;
  return (((long)b * p.cv_Ho + y) * p.cv_Wo + x) * p.N;
}

template <int NP, bool kSharedRcp = false>
__device__ __forceinline__ void apply_act_pairs(uint64_t (&v)[NP], int act) {
  static_assert(NP % 2 == 0, "activations are evaluated on groups of four elements");
  switch (act) {
    case kActGelu:
#pragma unroll
      for (int j = 0; j < NP; j += 2) {
        gelu4<kSharedRcp>(v[j], v[j + 1]);
      }
      break;
    case kActSwish:
#pragma unroll
      for (int j = 0; j < NP; j += 2) {
        swish4<kSharedRcp>(v[j], v[j + 1]);
      }
      break;
    case kActNone:
      break;
    default:
#pragma unroll
      for (int j = 0; j < NP; ++j) {
        float a, b;
        unpack2(v[j], a, b);
        v[j] = pack2(apply_act<false>(a, act), apply_act<false>(b, act));
      }
      break;
  }
}

__device__ __forceinline__ uint64_t ld_pair_or(const float* __restrict__ vec, int n, int N, float neutral) {
  if (n + 1 < N) {
    const float2 f = __ldg(reinterpret_cast<const float2*>(vec + n));
    return pack2(f.x, f.y);
  }
  return pack2(n < N ? __ldg(vec + n) : neutral, neutral);
}

__device__ __forceinline__ uint64_t ld_out_pair(const float* p, bool two) {
  if (two) {
    const float2 f = *reinterpret_cast<const float2*>(p);
    return pack2(f.x, f.y);
  }
  return pack2(*p, 0.f);
}
__device__ __forceinline__ uint64_t ld_out_pair(const __nv_bfloat16* p, bool two) {
  if (two) {
    const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p));
    return pack2(f.x, f.y);
  }
  return pack2(__bfloat162float(*p), 0.f);
}
__device__ __forceinline__ void st_out_pair(float* p, uint64_t v, bool two) {
  float a, b;
  unpack2(v, a, b);
  if (two) *reinterpret_cast<float2*>(p) = make_float2(a, b);
  else *p = a;
}
__device__ __forceinline__ void st_out_pair(__nv_bfloat16* p, uint64_t v, bool two) {
  float a, b;
  unpack2(v, a, b);
  if (two) *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b);
  else *p = __float2bfloat16_rn(a);
}

// Epilogue of one warpgroup's 64 x BN accumulator (BN / 2 fp32 per thread, wgmma.cuh layout) of tile (m_blk, n_blk);
// the warpgroup's rows start at tile row `wg_row0`.  Columns are handled 8 at a time (four values per thread: rows r and
// r + 8, columns c and c + 1), which is the granularity of the four-element activations.
// The groups go in runs of kRun: the bias, gamma and residual loads of a whole run are issued before its first store, so
// they overlap instead of each waiting behind the previous group's store (the residual may alias C, so the compiler
// cannot move a load above a store; loading ahead is legal because every element is read and written by the same
// thread).  kRun bounds the registers the loads hold: the 256-wide instances have the fewest to spare.
template <typename OutT, int BN>
__device__ __forceinline__ void epilogue_frag(const GemmParams& p, float (&acc)[BN / 2], int m_blk, int n_blk,
                                              int wg_row0) {
  constexpr int kRun = BN >= 256 ? 2 : 4;
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r = wg_row0 + wq * 16 + (lane >> 2);
  const long off_c[2] = {epilogue_row_offset(p, m_blk, r, p.ldc), epilogue_row_offset(p, m_blk, r + 8, p.ldc)};
  const long off_r[2] = {p.has_res ? epilogue_row_offset(p, m_blk, r, p.ldr) : -1,
                         p.has_res ? epilogue_row_offset(p, m_blk, r + 8, p.ldr) : -1};
  OutT* __restrict__ C = reinterpret_cast<OutT*>(p.c);
  const OutT* R = reinterpret_cast<const OutT*>(p.res);
#pragma unroll
  for (int g0 = 0; g0 < BN / 8; g0 += kRun) {
    if (n_blk * BN + g0 * 8 >= p.N) break;
    uint64_t b[kRun], s[kRun], res[kRun][2];
#pragma unroll
    for (int j = 0; j < kRun; ++j) {
      const int n = n_blk * BN + (g0 + j) * 8 + 2 * (lane & 3);
      const bool in = n < p.N, two = n + 1 < p.N;
      b[j] = p.bias != nullptr ? ld_pair_or(p.bias, n, p.N, 0.f) : 0;
      s[j] = p.gamma != nullptr ? ld_pair_or(p.gamma, n, p.N, 1.f) : 0;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        res[j][h] = p.has_res && in && off_r[h] >= 0 ? ld_out_pair(R + off_r[h] + n, two) : 0;
    }
#pragma unroll
    for (int j = 0; j < kRun; ++j) {
      const int g = g0 + j;
      const int n = n_blk * BN + g * 8 + 2 * (lane & 3);
      if (n_blk * BN + g * 8 >= p.N) break;
      const bool in = n < p.N, two = n + 1 < p.N;
      uint64_t v[2] = {pack2(acc[4 * g + 0], acc[4 * g + 1]), pack2(acc[4 * g + 2], acc[4 * g + 3])};
      if (p.bias != nullptr) {
        v[0] = add2(v[0], b[j]);
        v[1] = add2(v[1], b[j]);
      }
      if (!p.act_post) apply_act_pairs(v, p.act);
      if (p.gamma != nullptr) {
        v[0] = mul2(v[0], s[j]);
        v[1] = mul2(v[1], s[j]);
      }
      if (p.has_res) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (in && off_r[h] >= 0) v[h] = add2(v[h], res[j][h]);
      }
      if (p.act_post) apply_act_pairs(v, p.act);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (in && off_c[h] >= 0) st_out_pair(C + off_c[h] + n, v[h], two);
    }
  }
}

// ---- staged epilogue (plain GEMM, gemm_sm90.cu) ----
// The 128 x BN output tile lives in shared memory as column chunks of one 128-byte swizzle span (64 bf16 or 32 fp32
// columns); each warpgroup's 64 rows of a chunk are one 8 KB SWIZZLE_128B box, the layout TMA loads the residual into
// and stores the result from.  Box (wg, chunk) is at chunk_base + (wg * kChunks + chunk) * 8192.
template <typename OutT>
constexpr int staged_chunk_cols() { return 128 / (int)sizeof(OutT); }
constexpr int kStagedBoxBytes = 64 * 128;

// Shared-memory address of the pair (row, col), (row, col + 1) of a warpgroup's staged rows.  16-byte unit u of row r
// sits at unit u ^ (r & 7), so a warp's access for one column group (8 rows x 4 pairs) takes the fewest wavefronts
// its size allows: one for bf16 pairs (128 bytes), two for fp32 pairs (256 bytes).
template <typename OutT>
__device__ __forceinline__ uint32_t staged_addr(uint32_t s_wg, int row, int col) {
  constexpr int kCols = staged_chunk_cols<OutT>();
  const uint32_t byte = (uint32_t)(col % kCols) * (uint32_t)sizeof(OutT);
  return s_wg + (uint32_t)(col / kCols) * kStagedBoxBytes + (uint32_t)row * 128u +
         ((((byte >> 4) ^ (uint32_t)(row & 7)) << 4) | (byte & 15u));
}
__device__ __forceinline__ uint64_t ld_staged_pair(const float*, uint32_t a) {
  float x, y;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x), "=f"(y) : "r"(a) : "memory");
  return pack2(x, y);
}
__device__ __forceinline__ uint64_t ld_staged_pair(const __nv_bfloat16*, uint32_t a) {
  uint32_t u;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(a) : "memory");
  const float2 f = unpack_bf16x2(u);
  return pack2(f.x, f.y);
}
__device__ __forceinline__ void st_staged_pair(float*, uint32_t a, uint64_t v) {
  float x, y;
  unpack2(v, x, y);
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void st_staged_pair(__nv_bfloat16*, uint32_t a, uint64_t v) {
  float x, y;
  unpack2(v, x, y);
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_bf16x2(x, y)) : "memory");
}

// Tile columns kFirst .. kFirst + kSpan - 1 of one warpgroup's accumulator, through its staged boxes at s_wg (tile
// column kFirst is column 0 of the first box).  The per-element fp32 operations are those of epilogue_frag, in the
// same order.  s_bias / s_gamma hold the tile's bias and gamma values; when the tile has a residual, it has landed in
// the boxes.  Each element is read from and written back to the boxes by the same thread.
// kAct >= 0: the activation, known at compile time; kAct < 0: p.act, chosen per column group at run time.
template <typename OutT, int BN, int kFirst, int kSpan, int kAct>
__device__ __forceinline__ void staged_apply_act(const GemmParams& p, float (&acc)[BN / 2], uint32_t s_wg,
                                                 const float* s_bias, const float* s_gamma) {
  const int act = kAct >= 0 ? kAct : p.act;
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r = wq * 16 + (lane >> 2);   // warpgroup row; r + 8 has the same swizzle phase
  OutT* const tag = nullptr;
#pragma unroll
  for (int g = kFirst / 8; g < (kFirst + kSpan) / 8; ++g) {
    const int c = g * 8 + 2 * (lane & 3);
    const uint32_t a0 = staged_addr<OutT>(s_wg, r, c - kFirst), a1 = a0 + 8 * 128;
    uint64_t v[2] = {pack2(acc[4 * g + 0], acc[4 * g + 1]), pack2(acc[4 * g + 2], acc[4 * g + 3])};
    if (p.bias != nullptr) {
      const float2 b = *reinterpret_cast<const float2*>(s_bias + c);
      v[0] = add2(v[0], pack2(b.x, b.y));
      v[1] = add2(v[1], pack2(b.x, b.y));
    }
    if (!p.act_post) apply_act_pairs(v, act);
    if (p.gamma != nullptr) {
      const float2 s = *reinterpret_cast<const float2*>(s_gamma + c);
      v[0] = mul2(v[0], pack2(s.x, s.y));
      v[1] = mul2(v[1], pack2(s.x, s.y));
    }
    if (p.has_res) {
      v[0] = add2(v[0], ld_staged_pair(tag, a0));
      v[1] = add2(v[1], ld_staged_pair(tag, a1));
    }
    if (p.act_post) apply_act_pairs(v, act);
    st_staged_pair(tag, a0, v[0]);
    st_staged_pair(tag, a1, v[1]);
  }
}

// The common activations are dispatched once here rather than in every column group.  Unrolled over the groups, a
// per-group switch inlines every activation's code into each group; the epilogue's code then outgrows the instruction
// cache, and the jumps over the untaken cases make every tile's epilogue fetch it again.
template <typename OutT, int BN, int kFirst, int kSpan>
__device__ __forceinline__ void staged_apply(const GemmParams& p, float (&acc)[BN / 2], uint32_t s_wg,
                                             const float* s_bias, const float* s_gamma) {
  switch (p.act) {
    case kActNone: staged_apply_act<OutT, BN, kFirst, kSpan, kActNone>(p, acc, s_wg, s_bias, s_gamma); break;
    case kActGelu: staged_apply_act<OutT, BN, kFirst, kSpan, kActGelu>(p, acc, s_wg, s_bias, s_gamma); break;
    case kActSwish: staged_apply_act<OutT, BN, kFirst, kSpan, kActSwish>(p, acc, s_wg, s_bias, s_gamma); break;
    default: staged_apply_act<OutT, BN, kFirst, kSpan, -1>(p, acc, s_wg, s_bias, s_gamma); break;
  }
}

// Barrier over the 128 threads of consumer warpgroup wg.
__device__ __forceinline__ void warpgroup_bar_sync(int wg) {
  if (wg == 0) named_bar_sync<2>(128);
  else named_bar_sync<3>(128);
}

// One thread's TMA store of up to kChunks staged boxes of a warpgroup (rows row0 .., columns col0 ..), then the commit.
// Boxes wholly past N are not stored; the tensor map's extents clip the rest.
template <typename OutT, int kChunks>
__device__ __forceinline__ void staged_store(const GemmParams& p, const CUtensorMap* tmap_c, uint32_t s_wg, int row0,
                                             int col0) {
  constexpr int kCols = staged_chunk_cols<OutT>();
#pragma unroll
  for (int ch = 0; ch < kChunks; ++ch)
    if (col0 + ch * kCols < p.N) tma_store_2d(tmap_c, s_wg + (uint32_t)(ch * kStagedBoxBytes), col0 + ch * kCols, row0);
  tma_store_commit();
}

// Epilogue of one warpgroup (rows 64 wg .. 64 wg + 63 of tile (m_blk, n_blk)) through the staged tile s_out.  s_bias /
// s_gamma were written by the consumer threads before their mainloop; res_bar completes when the residual tile has
// landed in s_out (p.has_res).  The residual may alias C: the TMA store of the tile is issued only after its residual
// load has completed.  The output tensor map has the real extents (N, M), so the store clips the M and N tails.
template <typename OutT, int BN>
__device__ __forceinline__ void epilogue_staged(const GemmParams& p, float (&acc)[BN / 2], int m_blk, int n_blk, int wg,
                                                uint32_t s_out, const float* s_bias, const float* s_gamma,
                                                uint32_t res_bar, const CUtensorMap* tmap_c) {
  constexpr int kChunks = BN / staged_chunk_cols<OutT>();
  const uint32_t s_wg = s_out + (uint32_t)(wg * kChunks * kStagedBoxBytes);
  named_bar_sync<1>(256);   // s_bias / s_gamma were written by both consumer warpgroups
  if (p.has_res) mbar_wait(res_bar, 0);
  staged_apply<OutT, BN, 0, BN>(p, acc, s_wg, s_bias, s_gamma);
  // generic-proxy writes -> visible to the TMA engine, then one thread stores the warpgroup's rows
  fence_proxy_async_smem();
  warpgroup_bar_sync(wg);
  const int row0 = m_blk * 128 + wg * 64;
  if ((threadIdx.x & 127) == 0 && row0 < p.M) {
    staged_store<OutT, kChunks>(p, tmap_c, s_wg, row0, n_blk * BN);
    tma_store_wait_read<0>();   // the tile must not be released before the TMA engine has read it
  }
}

// Epilogue of the token-mixing GEMM (kModeToken): one warpgroup's 64 x BN accumulator of tile (img, m_blk, n_blk).
// Per element: acc + bias[row] -> act (glu: value * act(gate)) -> * gamma[col] -> * mul -> + residual -> store.
template <typename OutT, int BN>
__device__ __forceinline__ void epilogue_token(const GemmParams& p, float (&acc)[BN / 2], int img, int m_blk, int n_blk,
                                               int wg_row0) {
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int m0 = m_blk * 128 + wg_row0 + wq * 16 + (lane >> 2);   // A rows m0 and m0 + 8 (m0 % 16 < 8)
  const float b0 = p.bias != nullptr && m0 < p.M ? __ldg(p.bias + m0) : 0.f;
  const float b1 = p.bias != nullptr && m0 + 8 < p.M ? __ldg(p.bias + m0 + 8) : 0.f;
  // stored rows: (m0, m0 + 8), or the one GLU row
  const int rows[2] = {p.glu ? (m0 >> 4) * 8 + (m0 & 7) : m0, p.glu ? -1 : m0 + 8};
  OutT* __restrict__ C = reinterpret_cast<OutT*>(p.c) + (long)img * p.img_c;
  const OutT* R = reinterpret_cast<const OutT*>(p.res) + (long)img * p.img_r;
  const OutT* U = reinterpret_cast<const OutT*>(p.mul) + (long)img * p.img_mul;
#pragma unroll
  for (int g = 0; g < BN / 8; ++g) {
    const int n = n_blk * BN + g * 8 + 2 * (lane & 3);
    if (n_blk * BN + g * 8 >= p.N) break;
    const bool in = n < p.N, two = n + 1 < p.N;
    uint64_t v[2] = {pack2(acc[4 * g + 0] + b0, acc[4 * g + 1] + b0), pack2(acc[4 * g + 2] + b1, acc[4 * g + 3] + b1)};
    if (p.glu) {
      float x0, x1, g0, g1;
      unpack2(v[0], x0, x1);
      unpack2(v[1], g0, g1);
      v[0] = pack2(x0 * apply_act<false>(g0, p.act), x1 * apply_act<false>(g1, p.act));
    } else {
      apply_act_pairs(v, p.act);
    }
    if (p.gamma != nullptr) {
      const uint64_t s = ld_pair_or(p.gamma, n, p.N, 1.f);
      v[0] = mul2(v[0], s);
      v[1] = mul2(v[1], s);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rows[h];
      if (!in || row < 0 || row >= p.m_out) continue;
      if (p.mul != nullptr) v[h] = mul2(v[h], ld_out_pair(U + (long)row * p.ld_mul + n, two));
      if (p.has_res) v[h] = add2(v[h], ld_out_pair(R + (long)row * p.ldr + n, two));
      st_out_pair(C + (long)row * p.ldc + n, v[h], two);
    }
  }
}

// Epilogue of the channel GLU GEMM (kModeGluCols): accumulator columns 2j / 2j + 1 are value / gate of output column
// j, so each thread holds both halves of its pairs; stored: (value + bias) * act(gate + bias) at half width.
template <typename OutT, int BN>
__device__ __forceinline__ void epilogue_glu_cols(const GemmParams& p, float (&acc)[BN / 2], int m_blk, int n_blk,
                                                  int wg_row0) {
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r = wg_row0 + wq * 16 + (lane >> 2);
  const long off_c[2] = {epilogue_row_offset(p, m_blk, r, p.ldc), epilogue_row_offset(p, m_blk, r + 8, p.ldc)};
  OutT* __restrict__ C = reinterpret_cast<OutT*>(p.c);
#pragma unroll
  for (int g = 0; g < BN / 8; ++g) {
    const int n = n_blk * BN + g * 8 + 2 * (lane & 3);   // even: (value, gate) of output column n / 2
    if (n_blk * BN + g * 8 >= p.N) break;
    if (n >= p.N) continue;
    float bx = 0.f, bg = 0.f;
    if (p.bias != nullptr) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
      bx = b.x; bg = b.y;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (off_c[h] < 0) continue;
      const float x = acc[4 * g + 2 * h] + bx, gt = acc[4 * g + 2 * h + 1] + bg;
      const float y = x * apply_act<false>(gt, p.act);
      if constexpr (sizeof(OutT) == 2) C[off_c[h] + n / 2] = __float2bfloat16_rn(y);
      else C[off_c[h] + n / 2] = y;
    }
  }
}

}  // namespace tfimm
