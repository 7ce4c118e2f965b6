// Depthwise convolutions and pooling (CUDA-core / HBM-bound part of the conv families).
//
//   dwconv_ln        ZeroPad(k/2) -> DepthwiseConv2D(k x k, stride 1, bias) -> LayerNorm over C,
//                    the first half of ConvNeXtBlock.call (tfimm/architectures/convnext.py:219-228,
//                    layers built at :189-198).  One warp owns a strip of TW output pixels of one row
//                    and ALL channels (LN needs every channel of a pixel); channel groups of 128 are
//                    processed with a sliding register window along x, the k*k*C fp32 taps are read
//                    through L1, and the pre-norm values are parked in shared memory for the
//                    two-pass fp32 LayerNorm.
//   dwconv_bias_act  DepthwiseConv2D(k, stride, explicit 4-sided padding) + folded-BN bias + act,
//                    with optional fused squeeze (per-image channel sums for SqueezeExcite):
//                    tfimm/architectures/efficientnet_blocks.py:312-323,393-404,241-242.
//   global_avg_pool  GlobalAveragePooling2D / reduce_mean over H,W (convnext.py:433,
//                    efficientnet.py:256, swin.py:456, layers/classifier.py:34).
#include "common.cuh"

#include <stdlib.h>

namespace tfimm {

int dwconv_bias_act_pairs(const void* x, int dtype, const float* wgt, const float* bias, void* out, float* pool_sum,
                          int B, int H, int W, int C, int ks, int stride, int pad_t, int pad_l, int Ho, int Wo,
                          int act, cudaStream_t stream);
int dwconv_bias_act_tma(const void* x, int dtype, const float* wgt, const float* bias, void* out, float* pool_sum,
                        int B, int H, int W, int C, int ks, int stride, int pad_t, int pad_l, int Ho, int Wo, int act,
                        cudaStream_t stream);
int dwconv7_ln_cluster(const void* x, int in_dtype, const float* wgt, const float* bias, const float* gamma,
                       const float* beta, void* out, int out_dtype, int B, int H, int W, int C, float eps,
                       cudaStream_t stream);

namespace {

// ----------------------------------------------------------------------------------------------
// dwconv (stride 1, "same" symmetric zero pad) + bias + LayerNorm
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld4f(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4f(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st4f(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4f(__nv_bfloat16* p, float4 v) {
  uint2 u;
  u.x = pack_bf16x2(v.x, v.y);
  u.y = pack_bf16x2(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = u;
}

template <typename InT, typename OutT, int KS, int TW, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
dwconv_ln_kernel(const InT* __restrict__ x, const float* __restrict__ wgt /*[KS*KS][C]*/,
                 const float* __restrict__ bias, const float* __restrict__ gamma,
                 const float* __restrict__ beta, OutT* __restrict__ out, int B, int H, int W, int C,
                 float eps) {
  constexpr int PAD = KS / 2;
  extern __shared__ __align__(16) float sh[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* stash = sh + (size_t)warp * TW * C;  // [TW][C] pre-norm values of this warp's strip
  const int segs = (W + TW - 1) / TW;
  // unit order (b, seg, y) with y fastest: the WARPS warps of a CTA take adjacent rows (L1 reuse)
  const long unit = (long)blockIdx.x * WARPS + warp;
  const long units = (long)B * segs * H;
  if (unit >= units) return;
  const int y = (int)(unit % H);
  const long t = unit / H;
  const int seg = (int)(t % segs);
  const int b = (int)(t / segs);
  const int x0 = seg * TW;
  const int groups = C >> 7;  // 128 channels (4 per lane) per group; C % 128 handled by tail group
  const int tail = C & 127;
  float psum[TW];
#pragma unroll
  for (int i = 0; i < TW; ++i) psum[i] = 0.f;

  const int ngroups = groups + (tail ? 1 : 0);
  for (int gidx = 0; gidx < ngroups; ++gidx) {
    const int c = gidx * 128 + lane * 4;
    const bool cvalid = c < C;  // C % 4 == 0 is required, so a lane is fully in or out
    float4 acc[TW];
    const float4 bv = cvalid ? ld4f(bias + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < TW; ++i) acc[i] = bv;
    if (cvalid) {
#pragma unroll 1
      for (int ky = 0; ky < KS; ++ky) {
        const int iy = y + ky - PAD;
        if (iy < 0 || iy >= H) continue;
        float4 wv[KS];
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) wv[kx] = ld4f(wgt + (size_t)(ky * KS + kx) * C + c);
        const InT* row = x + (((long)b * H + iy) * W) * C + c;
#pragma unroll
        for (int ix = 0; ix < TW + KS - 1; ++ix) {
          const int gx = x0 + ix - PAD;
          if (gx < 0 || gx >= W) continue;
          const float4 v = ld4f(row + (long)gx * C);
#pragma unroll
          for (int kx = 0; kx < KS; ++kx) {
            const int ox = ix - kx;  // output pixel this (input, tap) pair contributes to
            if (ox >= 0 && ox < TW) {
              acc[ox].x = fmaf(v.x, wv[kx].x, acc[ox].x);
              acc[ox].y = fmaf(v.y, wv[kx].y, acc[ox].y);
              acc[ox].z = fmaf(v.z, wv[kx].z, acc[ox].z);
              acc[ox].w = fmaf(v.w, wv[kx].w, acc[ox].w);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < TW; ++i) {
        *reinterpret_cast<float4*>(stash + (size_t)i * C + c) = acc[i];
        psum[i] += acc[i].x + acc[i].y + acc[i].z + acc[i].w;
      }
    }
  }
  __syncwarp();
  // two-pass LayerNorm per pixel over the stashed values
#pragma unroll 1
  for (int i = 0; i < TW; ++i) {
    if (x0 + i >= W) break;
    const float mean = warp_sum(psum[i]) / (float)C;
    float sq = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(stash + (size_t)i * C + c);
      const float a = v.x - mean, bq = v.y - mean, cq = v.z - mean, d = v.w - mean;
      sq += a * a + bq * bq + cq * cq + d * d;
    }
    const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
    OutT* orow = out + (((long)b * H + y) * W + (x0 + i)) * C;
    for (int c = lane * 4; c < C; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(stash + (size_t)i * C + c);
      const float4 g = ld4f(gamma + c), be = ld4f(beta + c);
      float4 o;
      o.x = (v.x - mean) * rstd * g.x + be.x;
      o.y = (v.y - mean) * rstd * g.y + be.y;
      o.z = (v.z - mean) * rstd * g.z + be.z;
      o.w = (v.w - mean) * rstd * g.w + be.w;
      st4f(orow + c, o);
    }
  }
}

// ----------------------------------------------------------------------------------------------
// generic depthwise conv + bias + activation (+ fused squeeze)
// ----------------------------------------------------------------------------------------------
// One warp: one output row x 128 channels (4 per lane, coalesced 8/16-byte accesses).  The k*k taps of the
// lane's channels live in registers for the whole row, the row is walked in strips of TW pixels with a sliding
// input window, and the squeeze sums are accumulated in registers -> ONE atomic per (lane, channel) per row.
template <typename T, int KS, int STRIDE, int TW>
__global__ void __launch_bounds__(128)
dwconv_act_kernel(const T* __restrict__ x, const float* __restrict__ wgt /*[KS*KS][C]*/,
                  const float* __restrict__ bias, T* __restrict__ out, float* __restrict__ pool_sum,
                  int B, int H, int W, int C, int Ho, int Wo, int pad_t, int pad_l, int act) {
  const int cgroups = (C + 127) >> 7;
  const long unit = (long)blockIdx.x * 4 + (threadIdx.x >> 5);
  const long units = (long)B * Ho * cgroups;
  if (unit >= units) return;
  const int lane = threadIdx.x & 31;
  const int cg = (int)(unit % cgroups);
  const long t = unit / cgroups;
  const int oy = (int)(t % Ho);
  const int b = (int)(t / Ho);
  const int c = cg * 128 + lane * 4;
  if (c >= C) return;
  constexpr int IW = (TW - 1) * STRIDE + KS;  // input columns feeding one strip
  float4 wv[KS * KS];
#pragma unroll
  for (int i = 0; i < KS * KS; ++i) wv[i] = ld4f(wgt + (size_t)i * C + c);
  const float4 bv = bias != nullptr ? ld4f(bias + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ps = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int ox0 = 0; ox0 < Wo; ox0 += TW) {
    float4 acc[TW];
#pragma unroll
    for (int i = 0; i < TW; ++i) acc[i] = bv;
#pragma unroll
    for (int ky = 0; ky < KS; ++ky) {
      const int iy = oy * STRIDE + ky - pad_t;
      if (iy < 0 || iy >= H) continue;
      const T* row = x + (((long)b * H + iy) * W) * C + c;
#pragma unroll
      for (int ix = 0; ix < IW; ++ix) {
        const int gx = ox0 * STRIDE + ix - pad_l;
        if (gx < 0 || gx >= W) continue;
        const float4 v = ld4f(row + (long)gx * C);
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          // ix = ox*STRIDE + kx
          if ((ix - kx) >= 0 && (ix - kx) % STRIDE == 0 && (ix - kx) / STRIDE < TW) {
            const int ox = (ix - kx) / STRIDE;
            const float4 w4 = wv[ky * KS + kx];
            acc[ox].x = fmaf(v.x, w4.x, acc[ox].x);
            acc[ox].y = fmaf(v.y, w4.y, acc[ox].y);
            acc[ox].z = fmaf(v.z, w4.z, acc[ox].z);
            acc[ox].w = fmaf(v.w, w4.w, acc[ox].w);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < TW; ++i) {
      if (ox0 + i < Wo) {
        float4 o;
        o.x = apply_act<true>(acc[i].x, act);
        o.y = apply_act<true>(acc[i].y, act);
        o.z = apply_act<true>(acc[i].z, act);
        o.w = apply_act<true>(acc[i].w, act);
        st4f(out + (((long)b * Ho + oy) * Wo + ox0 + i) * C + c, o);
        if (pool_sum != nullptr) {
          // sum what the next layer will actually read (bf16-rounded when T is bf16)
          if constexpr (sizeof(T) == 2) {
            const float2 r0 = unpack_bf16x2(pack_bf16x2(o.x, o.y)), r1 = unpack_bf16x2(pack_bf16x2(o.z, o.w));
            ps.x += r0.x; ps.y += r0.y; ps.z += r1.x; ps.w += r1.y;
          } else {
            ps.x += o.x; ps.y += o.y; ps.z += o.z; ps.w += o.w;
          }
        }
      }
    }
  }
  if (pool_sum != nullptr) {
    float* p = pool_sum + (long)b * C + c;
    atomicAdd(p + 0, ps.x);
    atomicAdd(p + 1, ps.y);
    atomicAdd(p + 2, ps.z);
    atomicAdd(p + 3, ps.w);
  }
}

// ----------------------------------------------------------------------------------------------
// global average pool: (B, HW, C) -> (B, C) fp32
// ----------------------------------------------------------------------------------------------
template <typename T>
__global__ void global_avg_pool_kernel(const T* __restrict__ x, float* __restrict__ out, int HW, int C) {
  // grid: (ceil(C/128), B); block 128 threads = 4 pixel-phases x 32 lanes of 4 channels
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, ph = threadIdx.x >> 5;
  const int c = blockIdx.x * 128 + lane * 4;
  __shared__ float4 red[4][32];
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const T* base = x + (long)b * HW * C + c;
    for (int p = ph; p < HW; p += 4) {
      const float4 v = ld4f(base + (long)p * C);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  red[ph][lane] = s;
  __syncthreads();
  if (ph == 0 && c < C) {
    float4 a = red[0][lane];
#pragma unroll
    for (int i = 1; i < 4; ++i) {
      a.x += red[i][lane].x; a.y += red[i][lane].y; a.z += red[i][lane].z; a.w += red[i][lane].w;
    }
    const float inv = 1.0f / (float)HW;
    *reinterpret_cast<float4*>(out + (long)b * C + c) = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
  }
}

// ----------------------------------------------------------------------------------------------
// im2col for dense k x k convolutions that are then run as tensor-core GEMMs
// ----------------------------------------------------------------------------------------------
// out[g][(b, oy, ox)][(ky, kx, c)] = x[b, oy*s + ky - pad_t, ox*s + kx - pad_l, g*cg + c] (0 outside), c < cg = C / G,
// columns padded with zeros to Kpad.  G = 1 is the plain im2col; column order == TF conv kernel (kh, kw, cin, :)
// flattened.  G > 1 lays the groups of a grouped convolution out as G separate [M][Kpad] matrices, one GEMM each.
// KS_T / C_T: compile-time kernel size and channel count for the RGB stems (7x7 and 3x3 on 3 channels), where the
// per-element (tap, channel) decomposition would otherwise be runtime integer divisions; 0 = runtime values.
// pre_mean != null (raw uint8 pixels): every in-bounds value becomes (v * pre_scale - mean[c]) * inv_std[c] -- the
// reference's create_preprocessing (tfimm/models/factory.py:153-169) -- while the zero padding stays zero, as when the
// convolution pads the preprocessed image.
template <typename InT, typename OutT, int KS_T = 0, int C_T = 0>
__global__ void im2col_kernel(const InT* __restrict__ x, OutT* __restrict__ out, int B, int H, int W, int C_rt, int G,
                              int Ho, int Wo, int ks_rt, int stride, int pad_t, int pad_l, int Kpad,
                              float pre_scale = 1.f, const float* __restrict__ pre_mean = nullptr,
                              const float* __restrict__ pre_inv_std = nullptr) {
  const int C = C_T > 0 ? C_T : C_rt;
  const int ks = KS_T > 0 ? KS_T : ks_rt;
  const int cg = C_T > 0 ? C_T : C / G;
  const int K = ks * ks * cg;
  const int chunks = Kpad >> 3;
  const long M = (long)B * Ho * Wo;
  const long total = M * chunks * G;
  const bool vec = (cg & 7) == 0;  // 8 consecutive columns stay inside one (ky, kx) pixel
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % chunks);
    const long gm = idx / chunks;
    const long m = gm % M;
    const int coff = (int)(gm / M) * cg;
    const int ox = (int)(m % Wo);
    const long t = m / Wo;
    const int oy = (int)(t % Ho);
    const long b = t / Ho;
    const int k0 = ch * 8;
    float v[8];
    if (vec) {
      const int tap = k0 / cg, c = k0 % cg;
      const int ky = tap / ks, kx = tap % ks;
      const int iy = oy * stride + ky - pad_t, ix = ox * stride + kx - pad_l;
      if (k0 < K && iy >= 0 && iy < H && ix >= 0 && ix < W) {
        ld8(x + ((b * H + iy) * W + ix) * (long)C + coff + c, v);
        if (pre_mean != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            v[j] = (v[j] * pre_scale - __ldg(pre_mean + coff + c + j)) * __ldg(pre_inv_std + coff + c + j);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = k0 + j;
        float val = 0.f;
        if (k < K) {
          const int tap = k / cg, c = k % cg;
          const int ky = tap / ks, kx = tap % ks;
          const int iy = oy * stride + ky - pad_t, ix = ox * stride + kx - pad_l;
          if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
            val = ld_as_float(x + ((b * H + iy) * W + ix) * (long)C + coff + c);
            if (pre_mean != nullptr) val = (val * pre_scale - __ldg(pre_mean + coff + c)) * __ldg(pre_inv_std + coff + c);
          }
        }
        v[j] = val;
      }
    }
    st8(out + gm * Kpad + k0, v);
  }
}

// RGB 7x7 / stride-2 stem (ResNet conv1, tfimm/architectures/resnet.py:486-494): an im2col row is seven runs of
// 21 CONTIGUOUS input values, out[m][ky*21 + j] = x[b][2 oy - pad_t + ky][(2 ox - pad_l) * 3 + j].  The generic
// kernel gathers them as 4-byte global loads per element (1.0 ms for 256 x 224 x 224 x 3: 7x its HBM time); here a
// CTA stages the 7 input rows of 32 output pixels in shared memory with coalesced loads (converted to bf16 once)
// and every thread assembles 16-byte output chunks from there.
template <typename InT>
__global__ void __launch_bounds__(256)
im2col_stem7_kernel(const InT* __restrict__ x, __nv_bfloat16* __restrict__ out, int H, int W, int Ho, int Wo,
                    int pad_t, int pad_l, int Kpad, float pre_scale = 1.f, const float* __restrict__ pre_mean = nullptr,
                    const float* __restrict__ pre_inv_std = nullptr) {
  constexpr int TW = 32;                  // output pixels per CTA
  constexpr int ROW = ((TW - 1) * 2 + 7) * 3;  // 207 input values per tap row
  __shared__ __nv_bfloat16 tile[7][ROW + 1];
  const int segs = (Wo + TW - 1) / TW;
  int t = blockIdx.x;
  const int seg = t % segs; t /= segs;
  const int oy = t % Ho;
  const int b = t / Ho;
  const int ox0 = seg * TW;
  const int e0 = (ox0 * 2 - pad_l) * 3;   // first element (within an image row of W*3 values) of the tile
  const int iy0 = oy * 2 - pad_t;
  for (int idx = threadIdx.x; idx < 7 * ROW; idx += 256) {
    const int r = idx / ROW, e = idx - r * ROW;
    const int iy = iy0 + r, ge = e0 + e;
    float v = 0.f;
    if (iy >= 0 && iy < H && ge >= 0 && ge < W * 3) {
      v = ld_as_float(x + ((long)b * H + iy) * W * 3 + ge);
      if (pre_mean != nullptr) v = (v * pre_scale - __ldg(pre_mean + ge % 3)) * __ldg(pre_inv_std + ge % 3);
    }
    tile[r][e] = __float2bfloat16_rn(v);
  }
  __syncthreads();
  const int chunks = Kpad >> 3;
  for (int task = threadIdx.x; task < TW * chunks; task += 256) {
    const int p = task / chunks, ch = task - p * chunks;
    if (ox0 + p >= Wo) continue;
    uint32_t packed[4];
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      uint16_t h[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int k = ch * 8 + j + u;
        h[u] = k < 147 ? __bfloat16_as_ushort(tile[k / 21][p * 6 + k % 21]) : (uint16_t)0;
      }
      packed[j / 2] = (uint32_t)h[0] | ((uint32_t)h[1] << 16);
    }
    const long m = ((long)b * Ho + oy) * Wo + ox0 + p;
    *reinterpret_cast<uint4*>(out + m * Kpad + ch * 8) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  }
}

// ----------------------------------------------------------------------------------------------
// squeeze-excite gate: pooled sums -> 1x1 conv (bias) -> act -> 1x1 conv (bias) -> gate act
// ----------------------------------------------------------------------------------------------
// One CTA per image.  pooled_sum[b][C] (sum over pixels), w_reduce[rd][C], w_expand[rd][C], fp32.
__global__ void se_gate_kernel(const float* __restrict__ pooled_sum, float inv_hw,
                               const float* __restrict__ w_reduce, const float* __restrict__ b_reduce,
                               const float* __restrict__ w_expand, const float* __restrict__ b_expand,
                               float* __restrict__ gate, int C, int rd, int act, int gate_act) {
  extern __shared__ float sh[];
  float* mean = sh;        // [C]
  float* hid = sh + C;     // [rd]
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mean[c] = pooled_sum[(long)b * C + c] * inv_hw;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  // Both FCs are latency-bound (weights come from L2, ~300 clk per dependent load): keep many independent loads in
  // flight -- four rows of w_reduce per warp at a time, C walked in steps of 128 -> 16 loads per lane per round.
  for (int r0 = warp; r0 < rd; r0 += 4 * warps) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float* wr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) wr[i] = w_reduce + (long)min(r0 + i * warps, rd - 1) * C;
    for (int c0 = 0; c0 < C; c0 += 128) {
      float m[4], w[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = c0 + lane + 32 * j;
        m[j] = c < C ? mean[c] : 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) w[i][j] = c < C ? __ldg(wr[i] + c) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i] = fmaf(m[j], w[i][j], acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float a = warp_sum(acc[i]);
      const int r = r0 + i * warps;
      if (lane == 0 && r < rd) hid[r] = apply_act<true>(a + b_reduce[r], act);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    // w_expand is [rd][C]: consecutive threads read consecutive channels (coalesced); 8 independent loads per round
    float a[8] = {b_expand[c], 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int r = 0;
    for (; r + 8 <= rd; r += 8) {
      float w[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) w[i] = __ldg(w_expand + (long)(r + i) * C + c);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = fmaf(hid[r + i], w[i], a[i]);
    }
    for (; r < rd; ++r) a[0] = fmaf(hid[r], __ldg(w_expand + (long)r * C + c), a[0]);
    gate[(long)b * C + c] = apply_act<true>(((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7])), gate_act);
  }
}

// x[b, p, c] *= gate[b, c]   (in place; 8 channels per thread)
template <typename T>
__global__ void scale_channels_kernel(T* __restrict__ x, const float* __restrict__ gate, long total_chunks,
                                      int HW, int C) {
  const int cpr = C >> 3;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total_chunks;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % cpr);
    const long row = idx / cpr;
    const long b = row / HW;
    float v[8], g[8];
    ld8(x + row * C + ch * 8, v);
    ld8(gate + b * C + ch * 8, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= g[j];
    st8(x + row * C + ch * 8, v);
  }
}

// ----------------------------------------------------------------------------------------------
// spatial pooling windows (ResNet stem max-pool, "avg-down" shortcuts)
// ----------------------------------------------------------------------------------------------
// mode 0: max (padding acts as -inf), mode 1: average over the in-bounds cells only (TF "same"),
// mode 2: max where out-of-bounds cells are explicit zeros (ZeroPadding2D followed by a VALID MaxPool2D).
template <typename T>
__global__ void pool2d_kernel(const T* __restrict__ x, T* __restrict__ out, int B, int H, int W, int C, int Ho,
                              int Wo, int ks, int stride, int pad_t, int pad_l, int mode) {
  const int cpr = C >> 3;
  const long total = (long)B * Ho * Wo * cpr;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % cpr);
    const long m = idx / cpr;
    const int ox = (int)(m % Wo);
    const long t = m / Wo;
    const int oy = (int)(t % Ho);
    const long b = t / Ho;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = mode == 1 ? 0.f : -INFINITY;
    int cnt = 0;
    for (int ky = 0; ky < ks; ++ky) {
      const int iy = oy * stride + ky - pad_t;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < ks; ++kx) {
        const int ix = ox * stride + kx - pad_l;
        if (ix < 0 || ix >= W) continue;
        float v[8];
        ld8(x + ((b * H + iy) * W + ix) * (long)C + ch * 8, v);
        ++cnt;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = mode == 1 ? acc[j] + v[j] : fmaxf(acc[j], v[j]);
      }
    }
    if (mode == 2 && cnt < ks * ks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], 0.f);
    }
    if (mode == 1) {
      const float inv = 1.0f / (float)max(cnt, 1);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] *= inv;
    }
    st8(out + m * C + ch * 8, acc);
  }
}

inline unsigned conv_grid_for(long total, int threads) {
  long blocks = (total + threads - 1) / threads;
  const long cap = (long)sm_count() * 16;
  return (unsigned)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace

int im2col(const void* x, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C, int groups, int ks,
           int stride, int pad_t, int pad_l, int Ho, int Wo, int Kpad, cudaStream_t stream, float pre_scale,
           const float* pre_mean, const float* pre_inv_std) {
  TFIMM_CHECK_ARG(B > 0 && ks > 0 && stride > 0 && Ho > 0 && Wo > 0, "im2col: bad geometry");
  TFIMM_CHECK_ARG(groups > 0 && C % groups == 0, "im2col: C must be divisible by groups (C=%d groups=%d)", C, groups);
  TFIMM_CHECK_ARG(Kpad % 8 == 0 && Kpad >= ks * ks * (C / groups),
                  "im2col: Kpad must be a multiple of 8 and >= k*k*C/groups");
  TFIMM_CHECK_ARG((pre_mean == nullptr) == (pre_inv_std == nullptr), "im2col: mean and inv_std come together");
  TFIMM_CHECK_ARG((in_dtype == kU8) == (pre_mean != nullptr), "im2col: uint8 input <=> fused preprocessing");
  const long total = (long)B * Ho * Wo * (Kpad / 8) * groups;
  const unsigned grid = conv_grid_for(total, 256);
  if (in_dtype == kU8) {
    // raw pixels (stems): (v * scale - mean[c]) / std[c] inside the gather
    const uint8_t* xu = reinterpret_cast<const uint8_t*>(x);
    if (C == 3 && groups == 1 && ks == 7 && stride == 2 && out_dtype == kBF16 && Kpad >= 147) {
      const long ctas = (long)B * Ho * ((Wo + 31) / 32);
      im2col_stem7_kernel<<<(unsigned)ctas, 256, 0, stream>>>(xu, reinterpret_cast<__nv_bfloat16*>(out), H, W, Ho, Wo, pad_t,
                                                           pad_l, Kpad, pre_scale, pre_mean, pre_inv_std);
    } else if (C == 3 && groups == 1 && ks == 3 && out_dtype == kBF16) {
      im2col_kernel<uint8_t, __nv_bfloat16, 3, 3><<<grid, 256, 0, stream>>>(
          xu, reinterpret_cast<__nv_bfloat16*>(out), B, H, W, C, groups, Ho, Wo, ks, stride, pad_t, pad_l, Kpad, pre_scale,
          pre_mean, pre_inv_std);
    } else if (out_dtype == kBF16) {
      im2col_kernel<uint8_t, __nv_bfloat16><<<grid, 256, 0, stream>>>(xu, reinterpret_cast<__nv_bfloat16*>(out), B, H, W, C,
                                                                     groups, Ho, Wo, ks, stride, pad_t, pad_l, Kpad,
                                                                     pre_scale, pre_mean, pre_inv_std);
    } else if (out_dtype == kF32) {
      im2col_kernel<uint8_t, float><<<grid, 256, 0, stream>>>(xu, reinterpret_cast<float*>(out), B, H, W, C, groups, Ho, Wo,
                                                             ks, stride, pad_t, pad_l, Kpad, pre_scale, pre_mean,
                                                             pre_inv_std);
    } else {
      set_last_error("im2col: unsupported output dtype %d", out_dtype);
      return kInvalidArgument;
    }
    TFIMM_LAUNCH_OK("im2col_kernel (uint8)");
    return kOk;
  }
#define TFIMM_I2C(IN, OUT)                                                                              \
  im2col_kernel<IN, OUT><<<grid, 256, 0, stream>>>(reinterpret_cast<const IN*>(x), reinterpret_cast<OUT*>(out), \
                                                  B, H, W, C, groups, Ho, Wo, ks, stride, pad_t, pad_l, Kpad)
#define TFIMM_I2C_STEM(IN, OUT, KS_T)                                                                         \
  im2col_kernel<IN, OUT, KS_T, 3><<<grid, 256, 0, stream>>>(reinterpret_cast<const IN*>(x), reinterpret_cast<OUT*>(out), \
                                                           B, H, W, C, groups, Ho, Wo, ks, stride, pad_t, pad_l, Kpad)
  if (C == 3 && groups == 1 && ks == 7 && stride == 2 && out_dtype == kBF16 && Kpad >= 147 &&
      (in_dtype == kF32 || in_dtype == kBF16)) {
    const long ctas = (long)B * Ho * ((Wo + 31) / 32);
    if (in_dtype == kF32)
      im2col_stem7_kernel<<<(unsigned)ctas, 256, 0, stream>>>(reinterpret_cast<const float*>(x),
                                                           reinterpret_cast<__nv_bfloat16*>(out), H, W, Ho, Wo, pad_t,
                                                           pad_l, Kpad);
    else
      im2col_stem7_kernel<<<(unsigned)ctas, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                           reinterpret_cast<__nv_bfloat16*>(out), H, W, Ho, Wo, pad_t,
                                                           pad_l, Kpad);
  } else if (C == 3 && groups == 1 && (ks == 7 || ks == 3) && out_dtype == kBF16 && (in_dtype == kF32 || in_dtype == kBF16)) {
    if (in_dtype == kF32) { if (ks == 7) TFIMM_I2C_STEM(float, __nv_bfloat16, 7); else TFIMM_I2C_STEM(float, __nv_bfloat16, 3); }
    else { if (ks == 7) TFIMM_I2C_STEM(__nv_bfloat16, __nv_bfloat16, 7); else TFIMM_I2C_STEM(__nv_bfloat16, __nv_bfloat16, 3); }
  } else if (in_dtype == kF32 && out_dtype == kBF16) TFIMM_I2C(float, __nv_bfloat16);
  else if (in_dtype == kBF16 && out_dtype == kBF16) TFIMM_I2C(__nv_bfloat16, __nv_bfloat16);
  else if (in_dtype == kF32 && out_dtype == kF32) TFIMM_I2C(float, float);
  else {
    set_last_error("im2col: unsupported dtype combination in=%d out=%d", in_dtype, out_dtype);
    return kInvalidArgument;
  }
#undef TFIMM_I2C
#undef TFIMM_I2C_STEM
  TFIMM_LAUNCH_OK("im2col_kernel");
  return kOk;
}

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_im2col(const void* x, int in_dtype, void* out, int out_dtype, int B, int H, int W, int C, int groups,
                      int ks, int stride, int pad_t, int pad_l, int Ho, int Wo, int Kpad, void* stream) {
  return im2col(x, in_dtype, out, out_dtype, B, H, W, C, groups, ks, stride, pad_t, pad_l, Ho, Wo, Kpad,
                as_stream(stream), 1.0f, nullptr, nullptr);
}

int tfimm_b200_im2col_u8(const void* x, void* out, int out_dtype, int B, int H, int W, int C, int ks, int stride,
                         int pad_t, int pad_l, int Ho, int Wo, int Kpad, float scale, const float* mean,
                         const float* inv_std, void* stream) {
  return im2col(x, kU8, out, out_dtype, B, H, W, C, 1, ks, stride, pad_t, pad_l, Ho, Wo, Kpad, as_stream(stream), scale,
                mean, inv_std);
}

int tfimm_b200_se_gate(const float* pooled_sum, float inv_hw, const float* w_reduce, const float* b_reduce,
                       const float* w_expand, const float* b_expand, float* gate, int B, int C, int rd, int act,
                       int gate_act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && C > 0 && rd > 0, "se_gate: bad shape");
  const size_t smem = (size_t)(C + rd) * sizeof(float);
  TFIMM_CHECK_ARG(smem <= 48 * 1024, "se_gate: C + rd too large (%d + %d)", C, rd);
  // both FCs are chains of L2 round trips whose length is C / blockDim (second FC) and rd / (4 warps) (first FC):
  // 512 threads per image for wide layers (EfficientNet-B4: 1.08 -> 0.75 ms per step; 1024 threads: 0.80)
  const int threads = C >= 512 ? 512 : 256;
  se_gate_kernel<<<B, threads, smem, stream>>>(pooled_sum, inv_hw, w_reduce, b_reduce, w_expand, b_expand, gate, C, rd,
                                               act, gate_act);
  TFIMM_LAUNCH_OK("se_gate_kernel");
  return kOk;
}

int tfimm_b200_scale_channels(void* x, int dtype, const float* gate, int B, int HW, int C, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && HW > 0 && C > 0 && C % 8 == 0, "scale_channels: need C%%8==0 (C=%d)", C);
  const long total = (long)B * HW * (C / 8);
  const unsigned grid = conv_grid_for(total, 256);
  if (dtype == kBF16)
    scale_channels_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<__nv_bfloat16*>(x), gate, total, HW, C);
  else if (dtype == kF32)
    scale_channels_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<float*>(x), gate, total, HW, C);
  else {
    set_last_error("scale_channels: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("scale_channels_kernel");
  return kOk;
}

int tfimm_b200_pool2d(const void* x, int dtype, void* out, int B, int H, int W, int C, int ks, int stride, int pad_t,
                      int pad_l, int Ho, int Wo, int mode, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && C % 8 == 0 && ks > 0 && stride > 0, "pool2d: need C%%8==0 (C=%d)", C);
  TFIMM_CHECK_ARG(mode >= 0 && mode <= 2, "pool2d: mode must be 0 (max), 1 (avg) or 2 (zero-padded max)");
  const long total = (long)B * Ho * Wo * (C / 8);
  const unsigned grid = conv_grid_for(total, 256);
  if (dtype == kBF16)
    pool2d_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(out),
                                            B, H, W, C, Ho, Wo, ks, stride, pad_t, pad_l, mode);
  else if (dtype == kF32)
    pool2d_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(x), reinterpret_cast<float*>(out), B, H, W,
                                            C, Ho, Wo, ks, stride, pad_t, pad_l, mode);
  else {
    set_last_error("pool2d: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("pool2d_kernel");
  return kOk;
}

int tfimm_b200_dwconv_ln(const void* x, int in_dtype, const float* wgt, const float* bias, const float* gamma,
                         const float* beta, void* out, int out_dtype, int B, int H, int W, int C, int ks, float eps,
                         void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "dwconv_ln: need C%%4==0 (C=%d)", C);
  TFIMM_CHECK_ARG(ks == 7, "dwconv_ln: only kernel size 7 is instantiated (got %d)", ks);
  {
    // Fast path (fp32 residual stream in, bf16 out): the thread-block-cluster kernel (dwconv_ln_cluster.cu: 64- or
    // 32-channel slabs per CTA, statistics merged through distributed shared memory).
    const int st = dwconv7_ln_cluster(x, in_dtype, wgt, bias, gamma, beta, out, out_dtype, B, H, W, C, eps, stream);
    if (st != kUnsupported) return st;
  }
  constexpr int TW = 7;
  // warps per CTA limited by the [TW][C] fp32 stash per warp
  const size_t per_warp = (size_t)TW * C * sizeof(float);
  int warps = 4;
  while (warps > 1 && per_warp * warps > 96 * 1024) warps >>= 1;
  if (per_warp * warps > 227 * 1024) {
    set_last_error("dwconv_ln: C=%d too large for the shared-memory stash", C);
    return kUnsupported;
  }
  const long units = (long)B * ((W + TW - 1) / TW) * H;
  const size_t smem = per_warp * warps;
#define TFIMM_DWLN(IN, OUT, WARPS)                                                                      \
  do {                                                                                                  \
    auto k = dwconv_ln_kernel<IN, OUT, 7, TW, WARPS>;                                                   \
    if (smem > 48 * 1024)                                                                               \
      TFIMM_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
    k<<<(unsigned)((units + WARPS - 1) / WARPS), WARPS * 32, smem, stream>>>(                           \
        reinterpret_cast<const IN*>(x), wgt, bias, gamma, beta, reinterpret_cast<OUT*>(out), B, H, W, C, eps); \
  } while (0)
#define TFIMM_DWLN_W(IN, OUT)                  \
  do {                                         \
    if (warps == 4) TFIMM_DWLN(IN, OUT, 4);    \
    else if (warps == 2) TFIMM_DWLN(IN, OUT, 2); \
    else TFIMM_DWLN(IN, OUT, 1);               \
  } while (0)
  if (in_dtype == kF32 && out_dtype == kBF16) TFIMM_DWLN_W(float, __nv_bfloat16);
  else if (in_dtype == kBF16 && out_dtype == kBF16) TFIMM_DWLN_W(__nv_bfloat16, __nv_bfloat16);
  else if (in_dtype == kF32 && out_dtype == kF32) TFIMM_DWLN_W(float, float);
  else {
    set_last_error("dwconv_ln: unsupported dtype combination in=%d out=%d", in_dtype, out_dtype);
    return kInvalidArgument;
  }
#undef TFIMM_DWLN_W
#undef TFIMM_DWLN
  TFIMM_LAUNCH_OK("dwconv_ln_kernel");
  return kOk;
}

int tfimm_b200_dwconv_bias_act(const void* x, int dtype, const float* wgt, const float* bias, void* out,
                               float* pool_sum, int B, int H, int W, int C, int ks, int stride, int pad_t, int pad_l,
                               int Ho, int Wo, int act, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "dwconv: need C%%4==0 (C=%d)", C);
  TFIMM_CHECK_ARG((ks == 3 || ks == 5 || ks == 7) && (stride == 1 || stride == 2),
                  "dwconv: kernel size 3/5/7 and stride 1/2 are instantiated (got k=%d s=%d)", ks, stride);
  TFIMM_CHECK_ARG(dtype == kBF16 || dtype == kF32, "dwconv: dtype must be bf16 or f32");
  {
    // bf16, k in {3,5}: TMA-halo shared-memory kernel (dwconv_act_tma.cu)
    {
      const int st = dwconv_bias_act_tma(x, dtype, wgt, bias, out, pool_sum, B, H, W, C, ks, stride, pad_t, pad_l, Ho,
                                         Wo, act, stream);
      if (st != kUnsupported) return st;
    }
  }
  {
    // channel-pair / register-prefetch kernel (dwconv_act.cu) for k in {3,5}, fp32 and odd shapes; the kernel
    // below is the generic fallback (k = 7).
    const int st = dwconv_bias_act_pairs(x, dtype, wgt, bias, out, pool_sum, B, H, W, C, ks, stride, pad_t, pad_l,
                                         Ho, Wo, act, stream);
    if (st != kUnsupported) return st;
  }
  constexpr int TW = 4;
  const long units = (long)B * Ho * ((C + 127) / 128);
  const unsigned grid = (unsigned)((units + 3) / 4);
#define TFIMM_DW(T, KS, ST)                                                                              \
  dwconv_act_kernel<T, KS, ST, TW><<<grid, 128, 0, stream>>>(reinterpret_cast<const T*>(x), wgt, bias,    \
                                                            reinterpret_cast<T*>(out), pool_sum, B, H, W, \
                                                            C, Ho, Wo, pad_t, pad_l, act)
#define TFIMM_DW_T(T)                             \
  do {                                            \
    if (ks == 3 && stride == 1) TFIMM_DW(T, 3, 1); \
    else if (ks == 3) TFIMM_DW(T, 3, 2);          \
    else if (ks == 5 && stride == 1) TFIMM_DW(T, 5, 1); \
    else if (ks == 5) TFIMM_DW(T, 5, 2);          \
    else if (stride == 1) TFIMM_DW(T, 7, 1);      \
    else TFIMM_DW(T, 7, 2);                       \
  } while (0)
  if (dtype == kBF16) TFIMM_DW_T(__nv_bfloat16);
  else TFIMM_DW_T(float);
#undef TFIMM_DW_T
#undef TFIMM_DW
  TFIMM_LAUNCH_OK("dwconv_act_kernel");
  return kOk;
}

int tfimm_b200_global_avg_pool(const void* x, int dtype, float* out, int B, int HW, int C, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && HW > 0 && C > 0 && C % 4 == 0, "global_avg_pool: need C%%4==0");
  dim3 grid((C + 127) / 128, B);
  if (dtype == kBF16)
    global_avg_pool_kernel<<<grid, 128, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x), out, HW, C);
  else if (dtype == kF32)
    global_avg_pool_kernel<<<grid, 128, 0, stream>>>(reinterpret_cast<const float*>(x), out, HW, C);
  else {
    set_last_error("global_avg_pool: dtype must be bf16 or f32");
    return kInvalidArgument;
  }
  TFIMM_LAUNCH_OK("global_avg_pool_kernel");
  return kOk;
}

}  // extern "C"
