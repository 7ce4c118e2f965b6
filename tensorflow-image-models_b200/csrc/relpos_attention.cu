// Multi-head self-attention with decomposed relative-position terms: the attention core of the Segment Anything image
// encoder (tfimm/architectures/segment_anything/image_encoder.py:11-73 window partition / unpartition, 121-168
// add_decomposed_rel_pos, 231-263 RelPosAttention.call):
//
//     out_i = sum_j softmax_j(scale q_i . k_j + rel_h[i, ky(j)] + rel_w[i, kx(j)]) v_j
//     rel_h[i, ky] = q_i . R_h[qy(i) - ky + S_h - 1],   rel_w[i, kx] = q_i . R_w[qx(i) - kx + S_w - 1]   (unscaled q)
//
// over the packed qkv projection (B * gh * gw, 3 * H * dh) of the real tokens, column order [q | k | v], head-major.
// One "sequence" is either the whole gh x gw grid (global blocks) or one S x S window of the grid padded up to a
// multiple of S (window blocks).  The partition is index math: sequence token (ty, tx) of window (wy, wx) is grid
// position (wy S + ty, wx S + tx).  Positions outside the grid are the zero padding of window_partition AFTER norm1, so
// the reference projects them to q = b_q, k = b_k, v = b_v (the qkv bias): they are real keys and values of every query
// of their window.  The kernels synthesise k = b_k, v = b_v for them (zero without a bias), write no output row for them,
// and the qkv GEMM never sees them.  No (N, N) score or bias tensor is materialised.
//
// bf16 path: one CTA per (128 queries, head, image x sequence), 8 warps of 16 query rows.  K / V stream through a
// double-buffered cp.async ring of 64-key blocks (a head's K / V at N = 4096 are 1 MB).  Each warp first computes
// q . R for all 2S - 1 offsets of both tables with the tensor cores (R split into bf16 hi + lo parts, so the products
// carry R to ~2^-17) and scatters them into a per-row [S_h | S_w] table in shared memory; the main loop adds the two
// gathered terms to the logits.  mma.sync m16n8k16 for every product; the online softmax is attention_mma.cuh's.
//
// fp32 path (precision="fp32", and head dims the bf16 kernel does not take): SIMT, one warp per query row.
#include "attention_mma.cuh"
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kRpWarps = 8;
constexpr int kRpRows = kRpWarps * 16;
constexpr int kRpKeys = 64;

template <int DH>
struct RpCfg {
  static constexpr int LDS = DH + 8;                  // bf16 per shared-memory row: 144 / 176 B, conflict-free ldmatrix
  static constexpr int CH = DH / 8;                   // 16-byte chunks per row
  static constexpr int KS = DH / 16;                  // k16 steps of q . k
  static constexpr int NT = DH / 8;                   // n8 tiles of the output
  static constexpr int STAGE = 2 * kRpKeys * LDS;     // K + V of one block, bf16 elements
};

// Sequence geometry.  j -> (ty, tx) = (j / sw, j % sw) by a float reciprocal: exact for sw <= 127 and j < 2^16 (the
// rounding error of (j + 0.5) / sw stays far below the 0.5 / sw distance to the next integer).
struct RpGeom {
  int gh, gw, sh, sw, nww, nseq, N;
  float inv_sw;
  __device__ __forceinline__ int ty(int j) const { return __float2int_rz((j + 0.5f) * inv_sw); }
  // grid row of sequence token j of sequence `seq`, or -1 for a padding position
  __device__ __forceinline__ int row(int seq, int j) const {
    const int y = ty(j), x = j - y * sw;
    const int gy = (seq / nww) * sh + y, gx = (seq % nww) * sw + x;
    return (gy < gh && gx < gw) ? gy * gw + gx : -1;
  }
};

// bf16 hi / lo parts of two fp32 values: x = hi + lo + O(2^-17 |x|)
__device__ __forceinline__ void split_bf16x2(float2 x, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(x.x, x.y);
  const float2 h = unpack_bf16x2(hi);
  lo = pack_bf16x2(x.x - h.x, x.y - h.y);
}

// acc(16 rows x 8 offsets) = q . R[o0 .. o0 + 7] for one n8 tile of a table with nr rows (rows >= nr are zero)
template <int DH>
__device__ __forceinline__ void q_dot_table(float (&acc)[4], const uint32_t (&qf)[DH / 16][4], const float* R, int nr,
                                            int o0, int g, int t) {
  acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
  const int o = o0 + g;
  const float* r = R + (long)min(o, nr - 1) * DH + 2 * t;
#pragma unroll
  for (int ks = 0; ks < DH / 16; ++ks) {
    float2 x0 = __ldg(reinterpret_cast<const float2*>(r + 16 * ks));
    float2 x1 = __ldg(reinterpret_cast<const float2*>(r + 16 * ks + 8));
    if (o >= nr) x0 = x1 = make_float2(0.f, 0.f);
    uint32_t h0, l0, h1, l1;
    split_bf16x2(x0, h0, l0);
    split_bf16x2(x1, h1, l1);
    mma_bf16_16816(acc, qf[ks], h0, h1);
    mma_bf16_16816(acc, qf[ks], l0, l1);
  }
}

template <int DH>
__global__ void __launch_bounds__(kRpWarps * 32, 2)
relpos_attention_bf16_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                             const __nv_bfloat16* __restrict__ pad_bias, const float* __restrict__ rel_h,
                             const float* __restrict__ rel_w, RpGeom geo, int H, float scale_log2, int rs) {
  using C = RpCfg<DH>;
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int h = blockIdx.y;
  const int b = blockIdx.z / geo.nseq, seq = blockIdx.z % geo.nseq;
  const int N = geo.N;
  const long ld = 3L * H * DH;
  const __nv_bfloat16* img = qkv + (long)b * geo.gh * geo.gw * ld + h * DH;
  const __nv_bfloat16* kpad = pad_bias != nullptr ? pad_bias + H * DH + h * DH : nullptr;
  const uint32_t sRing = smem_u32(smem);
  // per-warp region: first the 16 q rows (bf16, LDS stride), then the [S_h | S_w] rel-pos table of those rows (fp32)
  float* relbuf = reinterpret_cast<float*>(smem + 2 * C::STAGE * 2) + warp * 16 * rs;
  const uint32_t sQ = smem_u32(relbuf);
  const int q0 = blockIdx.x * kRpRows + warp * 16;   // first sequence index of this warp's rows
  const bool active = q0 < N;
  const int nblocks = (N + kRpKeys - 1) / kRpKeys;

  // ---- q rows of this warp (padding / out-of-range rows are zero and never stored)
  for (int idx = lane; idx < 16 * C::CH; idx += 32) {
    const int r = idx / C::CH, c = idx % C::CH;
    const int j = q0 + r;
    const int row = j < N ? geo.row(seq, j) : -1;
    cp_async_16(sQ + (r * C::LDS + c * 8) * 2, img + (long)max(row, 0) * ld + c * 8, row >= 0);
  }
  cp_async_commit();

  // ---- K / V block kb -> ring stage kb & 1; padding keys read the k / v bias, keys >= N are zero (masked below)
  auto load_block = [&](int kb) {
    const uint32_t sK = sRing + (kb & 1) * C::STAGE * 2;
    const uint32_t sV = sK + kRpKeys * C::LDS * 2;
    for (int idx = tid; idx < kRpKeys * C::CH; idx += kRpWarps * 32) {
      const int r = idx / C::CH, c = idx % C::CH;
      const int j = kb * kRpKeys + r;
      const int row = j < N ? geo.row(seq, j) : -2;
      const __nv_bfloat16* src = row >= 0 ? img + (long)row * ld + H * DH : kpad;
      const bool valid = row >= 0 || (row == -1 && kpad != nullptr);
      if (!valid) src = img;
      const uint32_t off = (r * C::LDS + c * 8) * 2;
      cp_async_16(sK + off, src + c * 8, valid);
      cp_async_16(sV + off, src + H * DH + c * 8, valid);
    }
    cp_async_commit();
  };
  load_block(0);
  cp_async_wait<1>();   // the q group (committed first) has landed
  __syncwarp();

  uint32_t qf[C::KS][4];
#pragma unroll
  for (int ks = 0; ks < C::KS; ++ks) {
    const int row = lane & 15, chunk = 2 * ks + (lane >> 4);
    ldmatrix_x4(sQ + (row * C::LDS + chunk * 8) * 2, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
  }
  __syncwarp();   // the q rows are in registers: the region now holds the rel-pos table

  // ---- rel-pos table of this warp's rows: relbuf[r][ky] = rel_h[r, ky], relbuf[r][S_h + kx] = rel_w[r, kx]
  if (active) {
    int qy[2], qx[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int j = min(q0 + g + 8 * hr, N - 1);
      qy[hr] = geo.ty(j);
      qx[hr] = j - qy[hr] * geo.sw;
    }
    const int nrh = 2 * geo.sh - 1, nrw = 2 * geo.sw - 1;
    for (int o0 = 0; o0 < nrh; o0 += 8) {
      float acc[4];
      q_dot_table<DH>(acc, qf, rel_h, nrh, o0, g, t);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1, ky = qy[hr] + geo.sh - 1 - (o0 + 2 * t + (e & 1));
        if (ky >= 0 && ky < geo.sh) relbuf[(g + 8 * hr) * rs + ky] = acc[e];
      }
    }
    for (int o0 = 0; o0 < nrw; o0 += 8) {
      float acc[4];
      q_dot_table<DH>(acc, qf, rel_w, nrw, o0, g, t);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1, kx = qx[hr] + geo.sw - 1 - (o0 + 2 * t + (e & 1));
        if (kx >= 0 && kx < geo.sw) relbuf[(g + 8 * hr) * rs + geo.sh + kx] = acc[e];
      }
    }
  }
  __syncwarp();

  float o[C::NT][4];
#pragma unroll
  for (int i = 0; i < C::NT; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  OnlineSoftmax<false> sm;
  const float* rel0 = relbuf + g * rs;
  const float* rel1 = relbuf + (g + 8) * rs;

#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    if (kb + 1 < nblocks) {
      load_block(kb + 1);   // its stage was released by the __syncthreads that ended block kb - 1
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      const uint32_t sK = sRing + (kb & 1) * C::STAGE * 2;
      const uint32_t sV = sK + kRpKeys * C::LDS * 2;
      const int key0 = kb * kRpKeys;
      float s[8][4];
      qk_bf16(s, qf, 8, lane, [&](int row, int chunk) { return sK + (row * C::LDS + chunk * 8) * 2; });
      // logits in log2 units: scale q.k + rel_h + rel_w; keys >= N masked; row max
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int j0 = key0 + nt * 8 + 2 * t;
        int ky = geo.ty(j0), kx = j0 - ky * geo.sw;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (c == 1 && ++kx == geo.sw) { kx = 0; ++ky; }
          const bool valid = j0 + c < N;
          const int iy = valid ? ky : 0, ix = valid ? geo.sh + kx : 0;
          const float v0 = fmaf(s[nt][c], scale_log2, (rel0[iy] + rel0[ix]) * kLog2e);
          const float v1 = fmaf(s[nt][2 + c], scale_log2, (rel1[iy] + rel1[ix]) * kLog2e);
          s[nt][c] = valid ? v0 : -INFINITY;
          s[nt][2 + c] = valid ? v1 : -INFINITY;
          mx[0] = fmaxf(mx[0], s[nt][c]);
          mx[1] = fmaxf(mx[1], s[nt][2 + c]);
        }
      }
      sm.update(s, o, mx);
      pv_bf16(o, s, 8, lane, [&](int row, int chunk) { return sV + (row * C::LDS + chunk * 8) * 2; });
    }
    __syncthreads();   // every warp is done with this stage before block kb + 2 is loaded into it
  }

  if (!active) return;
  const long ldo = (long)H * DH;
  __nv_bfloat16* dst_img = out + (long)b * geo.gh * geo.gw * ldo + h * DH + 2 * t;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const RowNorm nrm = sm.finish(hr);
    const int j = q0 + g + 8 * hr;
    const int row = j < N ? geo.row(seq, j) : -1;
    if (row >= 0) {
      __nv_bfloat16* dst = dst_img + (long)row * ldo;
#pragma unroll
      for (int nt = 0; nt < C::NT; ++nt)
        *reinterpret_cast<uint32_t*>(dst + 8 * nt) =
            pack_bf16x2(nrm(o[nt][2 * hr]), nrm(o[nt][2 * hr + 1]));
    }
  }
}

// ---- fp32 path: one warp per (image, sequence, head, real query) ----
__global__ void relpos_attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                            const float* __restrict__ pad_bias, const float* __restrict__ rel_h,
                                            const float* __restrict__ rel_w, RpGeom geo, int H, int dh, float scale,
                                            long total) {
  extern __shared__ float fsm[];
  const int warps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int N = geo.N;
  float* sc = fsm + (size_t)warp * (N + dh + geo.sh + geo.sw);
  float* qs = sc + N;
  float* rh = qs + dh;
  float* rw = rh + geo.sh;
  const long rid = (long)blockIdx.x * warps + warp;
  if (rid >= total) return;
  const int i = (int)(rid % N);
  const long rest = rid / N;
  const int h = (int)(rest % H);
  const long bs = rest / H;
  const long b = bs / geo.nseq;
  const int seq = (int)(bs % geo.nseq);
  const int qrow = geo.row(seq, i);
  if (qrow < 0) return;   // padding query: its output row does not exist
  const long ld = 3L * H * dh;
  const float* img = qkv + b * geo.gh * geo.gw * ld + (long)h * dh;
  const float* kpad = pad_bias != nullptr ? pad_bias + (long)H * dh + (long)h * dh : nullptr;
  for (int d = lane; d < dh; d += 32) qs[d] = img[(long)qrow * ld + d];
  __syncwarp();
  const int qy = geo.ty(i), qx = i - qy * geo.sw;
  for (int k = lane; k < geo.sh + geo.sw; k += 32) {
    const float* r = k < geo.sh ? rel_h + (long)(qy - k + geo.sh - 1) * dh
                                : rel_w + (long)(qx - (k - geo.sh) + geo.sw - 1) * dh;
    float acc = 0.f;
    for (int d = 0; d < dh; ++d) acc = fmaf(qs[d], r[d], acc);
    (k < geo.sh ? rh[k] : rw[k - geo.sh]) = acc;
  }
  __syncwarp();
  // key j's k row (v row = k row + H * dh), or nullptr for a zero key
  auto krow = [&](int j) -> const float* {
    const int row = geo.row(seq, j);
    return row >= 0 ? img + (long)row * ld + (long)H * dh : kpad;
  };
  float mx = -INFINITY;
  for (int j = lane; j < N; j += 32) {
    const float* kr = krow(j);
    float acc = 0.f;
    if (kr != nullptr)
      for (int d = 0; d < dh; ++d) acc = fmaf(qs[d], kr[d], acc);
    const int ky = geo.ty(j), kx = j - ky * geo.sw;
    acc = acc * scale + rh[ky] + rw[kx];
    sc[j] = acc;
    mx = fmaxf(mx, acc);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < N; j += 32) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  __syncwarp();
  float* dst = out + (b * geo.gh * geo.gw + qrow) * ((long)H * dh) + (long)h * dh;
  for (int d = lane; d < dh; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < N; ++j) {
      const float* kr = krow(j);
      if (kr != nullptr) acc = fmaf(sc[j], kr[(long)H * dh + d], acc);
    }
    dst[d] = acc * inv;
  }
}

int make_geom(RpGeom& geo, int B, int gh, int gw, int H, int dh, int window) {
  TFIMM_CHECK_ARG(B > 0 && gh > 0 && gw > 0 && H > 0 && dh > 0 && window >= 0,
                  "relpos_attention: bad shape B=%d grid=%dx%d H=%d dh=%d window=%d", B, gh, gw, H, dh, window);
  geo.gh = gh;
  geo.gw = gw;
  geo.sh = window > 0 ? window : gh;
  geo.sw = window > 0 ? window : gw;
  TFIMM_CHECK_ARG(geo.sh <= 127 && geo.sw <= 127, "relpos_attention: sequence extent %dx%d above 127", geo.sh, geo.sw);
  const int nwh = (gh + geo.sh - 1) / geo.sh;
  geo.nww = (gw + geo.sw - 1) / geo.sw;
  geo.nseq = nwh * geo.nww;
  geo.N = geo.sh * geo.sw;
  geo.inv_sw = 1.0f / geo.sw;
  TFIMM_CHECK_ARG((long)B * geo.nseq <= 65535, "relpos_attention: B x windows = %ld above 65535", (long)B * geo.nseq);
  return kOk;
}

template <int DH>
int launch_relpos_bf16(const __nv_bfloat16* qkv, __nv_bfloat16* out, const __nv_bfloat16* pad_bias,
                       const float* rel_h, const float* rel_w, int B, const RpGeom& geo, int H, float scale,
                       cudaStream_t stream) {
  using C = RpCfg<DH>;
  // per-warp row stride of the rel-pos table (fp32): holds S_h + S_w entries, and the 16 staged q rows fit in the
  // region; odd, so that the eight rows g of a fragment start in distinct banks
  const int rs = max(geo.sh + geo.sw, C::LDS / 2) | 1;
  const size_t smem = (size_t)2 * C::STAGE * 2 + (size_t)kRpWarps * 16 * rs * sizeof(float);
  if (smem > 113 * 1024) {   // S_h + S_w > 153 (dh 64) / 137 (dh 80): tfimm.backend.sam_ops checks the same bound
    set_last_error("relpos_attention: sequence extent %dx%d needs %zu B of shared memory (S_h + S_w <= 153 at head_dim "
                   "64, <= 137 at 80)", geo.sh, geo.sw, smem);
    return kUnsupported;
  }
  auto kernel = relpos_attention_bf16_kernel<DH>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, 113 * 1024, attr_devs));
  dim3 grid((geo.N + kRpRows - 1) / kRpRows, H, B * geo.nseq);
  kernel<<<grid, kRpWarps * 32, smem, stream>>>(qkv, out, pad_bias, rel_h, rel_w, geo, H, scale * kLog2e, rs);
  TFIMM_LAUNCH_OK("relpos_attention_bf16_kernel");
  return kOk;
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_relpos_attention_bf16(const void* qkv, void* out, const void* pad_bias, const float* rel_h,
                                     const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                     void* s) {
  const cudaStream_t stream = as_stream(s);
  RpGeom geo;
  if (int st = make_geom(geo, B, gh, gw, H, dh, window)) return st;
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(pad_bias) & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(rel_h) & 7u) == 0 && (reinterpret_cast<uintptr_t>(rel_w) & 7u) == 0,
                  "relpos_attention: qkv / out / pad_bias must be 16-byte and the tables 8-byte aligned");
  auto q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  auto o = reinterpret_cast<__nv_bfloat16*>(out);
  auto pb = reinterpret_cast<const __nv_bfloat16*>(pad_bias);
  if (dh == 64) return launch_relpos_bf16<64>(q, o, pb, rel_h, rel_w, B, geo, H, scale, stream);
  if (dh == 80) return launch_relpos_bf16<80>(q, o, pb, rel_h, rel_w, B, geo, H, scale, stream);
  set_last_error("relpos_attention: bf16 kernel takes head_dim 64 or 80 (got %d)", dh);
  return kUnsupported;
}

int tfimm_b200_relpos_attention_f32(const float* qkv, float* out, const float* pad_bias, const float* rel_h,
                                    const float* rel_w, int B, int gh, int gw, int H, int dh, int window, float scale,
                                    void* s) {
  const cudaStream_t stream = as_stream(s);
  RpGeom geo;
  if (int st = make_geom(geo, B, gh, gw, H, dh, window)) return st;
  const int warps = 4;
  const size_t smem = (size_t)warps * (geo.N + dh + geo.sh + geo.sw) * sizeof(float);
  if (smem > 227 * 1024) {
    set_last_error("relpos_attention_f32: sequence of %d tokens too long for the fp32 kernel", geo.N);
    return kUnsupported;
  }
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(relpos_attention_f32_kernel, 227 * 1024, attr_devs));
  const long total = (long)B * geo.nseq * H * geo.N;
  const unsigned grid = (unsigned)((total + warps - 1) / warps);
  relpos_attention_f32_kernel<<<grid, warps * 32, smem, stream>>>(qkv, out, pad_bias, rel_h, rel_w, geo, H, dh, scale,
                                                                  total);
  TFIMM_LAUNCH_OK("relpos_attention_f32_kernel");
  return kOk;
}

}  // extern "C"
