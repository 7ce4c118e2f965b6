// Fused multi-head self-attention for the ViT family:
//     out[b, n, h, :] = softmax(scale * q k^T) v        (per image b, head h)
// reading q/k/v straight out of the packed qkv projection (B*N, 3*H*dh) whose
// column order is [q | k | v], each head-major -- exactly the layout produced
// by the reshape/transpose in tfimm/architectures/vit.py:149-165.  The
// (B,H,N,N) score tensor the reference materialises (vit.py:160-163) never
// leaves the SM.
//
// bf16 path: one CTA per (image, head, 224-query chunk); K and V of the head are
// staged once in XOR-swizzled shared memory with cp.async, each warp owns 16-row
// query tiles and runs the online softmax of attention_mma.cuh with mma.sync m16n8k16.
//
// tf32 path (precision="tf32"): fp32 qkv / out, mma.sync m16n8k8 TF32, K / V streamed in 64-key blocks.
//
// fp32 path (precision="fp32" parity mode, and every call with bias / mask / probs / row_map): plain SIMT, one warp
// per query row.
#include "attention_mma.cuh"
#include "common.cuh"

#include <stdlib.h>

namespace tfimm {
namespace {

constexpr int kDH = 64;

template <int NW, int TPW>
__global__ void __launch_bounds__(NW * 32, 2)
vit_attention_bf16_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                          int N, int H, float scale_log2) {
  constexpr int ROWS = NW * TPW * 16;
  extern __shared__ __align__(128) uint8_t smem[];
  const int npad = (N + 15) & ~15;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + ROWS * 128;
  const uint32_t sV = sK + npad * 128;

  const int b = blockIdx.z, h = blockIdx.y;
  const int q_base = blockIdx.x * ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long ld = 3L * H * kDH;
  const __nv_bfloat16* base = qkv + (long)b * N * ld + h * kDH;

  // ---- stage Q (this chunk), K, V (whole head) in swizzled smem ----
  for (int idx = tid; idx < ROWS * 8; idx += NW * 32) {
    const int r = idx >> 3, c = idx & 7;
    const int gr = q_base + r;
    const bool valid = gr < N;
    cp_async_16(sQ + r * 128 + ((c ^ (r & 7)) << 4), base + (long)(valid ? gr : 0) * ld + c * 8, valid);
  }
  for (int idx = tid; idx < npad * 8; idx += NW * 32) {
    const int r = idx >> 3, c = idx & 7;
    const bool valid = r < N;
    const __nv_bfloat16* src = base + (long)(valid ? r : 0) * ld + c * 8;
    const uint32_t off = r * 128 + ((c ^ (r & 7)) << 4);
    cp_async_16(sK + off, src + H * kDH, valid);
    cp_async_16(sV + off, src + 2 * H * kDH, valid);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  const int nblocks = (npad + 63) >> 6;

#pragma unroll 1
  for (int tt = 0; tt < TPW; ++tt) {
    const int tile = tt * NW + warp;      // round-robin so short sequences stay balanced
    const int q0 = tile * 16;             // row inside this CTA's chunk
    if (q_base + q0 >= N) continue;

    uint32_t qf[kDH / 16][4];
#pragma unroll
    for (int ks = 0; ks < kDH / 16; ++ks) {
      const int row = q0 + (lane & 15);
      const int chunk = ks * 2 + (lane >> 4);
      ldmatrix_x4(sQ + row * 128 + ((chunk ^ (row & 7)) << 4), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
    float o[kDH / 8][4];
#pragma unroll
    for (int i = 0; i < kDH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    OnlineSoftmax<false> sm;

#pragma unroll 1
    for (int kb = 0; kb < nblocks; ++kb) {
      const int key0 = kb * 64;
      const int ntv = min(8, (npad - key0) >> 3);  // valid 8-key tiles in this block (even)
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        if (nt < ntv) {
#pragma unroll
          for (int j = 0; j < kDH / 32; ++j) {
            const int row = key0 + nt * 8 + (lane & 7);
            const int chunk = 4 * j + (lane >> 3);
            uint32_t k0, k1, k2, k3;
            ldmatrix_x4(sK + row * 128 + ((chunk ^ (row & 7)) << 4), k0, k1, k2, k3);
            mma_bf16_16816(s[nt], qf[2 * j], k0, k1);
            mma_bf16_16816(s[nt], qf[2 * j + 1], k2, k3);
          }
        }
      }
      // scale, mask, row max
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + nt * 8 + 2 * t + (e & 1);
          const float val = (nt < ntv && key < N) ? s[nt][e] * scale_log2 : -INFINITY;
          s[nt][e] = val;
          mx[e >> 1] = fmaxf(mx[e >> 1], val);
        }
      }
      sm.update(s, o, mx);
      pv_bf16(o, s, ntv, lane, [&](int r, int chunk) {
        const int row = key0 + r;
        return sV + row * 128 + ((chunk ^ (row & 7)) << 4);
      });
    }
    // normalise (O / l correctly rounded) and write through the (now dead) Q tile in smem for coalesced stores
    const RowNorm n0 = sm.finish(0), n1 = sm.finish(1);
    __syncwarp();
    uint8_t* tile_gen = smem + q0 * 128;
#pragma unroll
    for (int nt = 0; nt < kDH / 8; ++nt) {
      const int r0 = g, r1 = g + 8;
      *reinterpret_cast<uint32_t*>(tile_gen + r0 * 128 + ((nt ^ (r0 & 7)) << 4) + t * 4) =
          pack_bf16x2(n0(o[nt][0]), n0(o[nt][1]));
      *reinterpret_cast<uint32_t*>(tile_gen + r1 * 128 + ((nt ^ (r1 & 7)) << 4) + t * 4) =
          pack_bf16x2(n1(o[nt][2]), n1(o[nt][3]));
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = lane + 32 * i;
      const int r = idx >> 3, c = idx & 7;
      const int gr = q_base + q0 + r;
      if (gr < N) {
        const uint4 val = *reinterpret_cast<const uint4*>(tile_gen + r * 128 + ((c ^ (r & 7)) << 4));
        *reinterpret_cast<uint4*>(out + ((long)b * N + gr) * ((long)H * kDH) + h * kDH + c * 8) = val;
      }
    }
  }
}

template <int NW, int TPW>
int launch_vit_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int N, int H, float scale,
                         cudaStream_t stream) {
  constexpr int ROWS = NW * TPW * 16;
  const int npad = (N + 15) & ~15;
  const size_t smem = (size_t)(ROWS + 2 * npad) * 128;
  if (smem > 227 * 1024) {
    set_last_error("attention: sequence length %d does not fit the resident-KV kernel (%zu B smem)", N, smem);
    return kUnsupported;
  }
  auto kernel = vit_attention_bf16_kernel<NW, TPW>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, 227 * 1024, attr_devs));
  dim3 grid((N + ROWS - 1) / ROWS, H, B);
  kernel<<<grid, NW * 32, smem, stream>>>(qkv, out, N, H, scale * kLog2e);
  TFIMM_LAUNCH_OK("vit_attention_bf16_kernel");
  return kOk;
}

// ---- TF32 path (precision="tf32"): fp32 qkv / out, TF32 tensor-core products ----
// One CTA per (image, head, 128-query chunk), 8 warps of 16 query rows.  fp32 K / V of a whole head do not fit shared
// memory at N = 577 (295 KB), so they stream through a double-buffered cp.async ring of 64-key blocks shared by the
// warps; each warp runs the online softmax of attention_mma.cuh with mma.sync m16n8k8 TF32.  Q, K, V are rounded to
// TF32 (cvt.rna) as their fragments are loaded; P is rounded before PV.
//
// Fragment bookkeeping: the contraction index of an m16n8k8 product is free to permute as long as A and B agree.
//   S = Q K^T: k-step ks covers dims 8 ks .. 8 ks + 7; logical k = t <-> dim 8 ks + 2t, k = t + 4 <-> dim 8 ks + 2t + 1,
//              so each thread's two A (and two B) values are adjacent in memory: one 8-byte load.
//   O = P V:   key tile nt; logical k = t <-> key 8 nt + 2t, k = t + 4 <-> key 8 nt + 2t + 1 -- exactly the two P values
//              thread t holds in the S accumulator layout (columns 2t, 2t + 1), so P never moves between threads.
// Row strides in shared memory: Q and K 72 floats (the 8-byte loads of a half-warp hit 32 distinct banks), V 68 floats
// (rows 2t and 2t + 1 of the four t's land on distinct banks for each of the eight columns g).
constexpr int kTfWarps = 8;
constexpr int kTfRows = kTfWarps * 16;
constexpr int kTfKeys = 64;
constexpr int kTfLdK = 72, kTfLdV = 68;
constexpr int kTfStageFloats = kTfKeys * (kTfLdK + kTfLdV);
constexpr size_t kTfSmemBytes = (2 * kTfStageFloats + kTfRows * kTfLdK) * sizeof(float);   // K/V ring + Q: 106 KB

__global__ void __launch_bounds__(kTfWarps * 32, 2)
vit_attention_tf32_kernel(const float* __restrict__ qkv, float* __restrict__ out, int N, int H, float scale_log2) {
  extern __shared__ __align__(16) float tsm[];
  const int b = blockIdx.z, h = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long ld = 3L * H * kDH;
  const float* base = qkv + (long)b * N * ld + h * kDH;
  const int nblocks = (N + kTfKeys - 1) / kTfKeys;

  // K / V block kb -> stage kb & 1 (16-byte chunks; keys >= N are zero-filled and masked below)
  auto load_block = [&](int kb) {
    float* sK = tsm + (kb & 1) * kTfStageFloats;
    float* sV = sK + kTfKeys * kTfLdK;
    for (int idx = tid; idx < kTfKeys * (kDH / 4); idx += kTfWarps * 32) {
      const int r = idx >> 4, c = idx & 15;
      const int key = kb * kTfKeys + r;
      const bool valid = key < N;
      const float* src = base + (long)(valid ? key : 0) * ld + c * 4;
      cp_async_16(smem_u32(sK + r * kTfLdK + c * 4), src + H * kDH, valid);
      cp_async_16(smem_u32(sV + r * kTfLdV + c * 4), src + 2 * H * kDH, valid);
    }
    cp_async_commit();
  };
  load_block(0);

  // this warp's 16 query rows, rounded once, in its own slice of shared memory (rows >= N repeat row N - 1 and are
  // never stored); the fragments are reloaded per key block rather than held in 32 registers
  const int q0 = blockIdx.x * kTfRows + warp * 16;
  const bool active = q0 < N;
  float* sQ = tsm + 2 * kTfStageFloats + warp * 16 * kTfLdK;
  for (int idx = lane; idx < 16 * (kDH / 4); idx += 32) {
    const int r = idx >> 4, c = idx & 15;
    const float4 x = __ldg(reinterpret_cast<const float4*>(base + (long)min(q0 + r, N - 1) * ld + c * 4));
    *reinterpret_cast<uint4*>(sQ + r * kTfLdK + c * 4) =
        make_uint4(tf32_rna(x.x), tf32_rna(x.y), tf32_rna(x.z), tf32_rna(x.w));
  }
  __syncwarp();
  float o[kDH / 8][4];
#pragma unroll
  for (int i = 0; i < kDH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  OnlineSoftmax<false> sm;

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
      const float* sK = tsm + (kb & 1) * kTfStageFloats;
      const float* sV = sK + kTfKeys * kTfLdK;
      const int key0 = kb * kTfKeys;
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < kDH / 8; ++ks) {
        const float2 qa = *reinterpret_cast<const float2*>(sQ + g * kTfLdK + 8 * ks + 2 * t);
        const float2 qb = *reinterpret_cast<const float2*>(sQ + (g + 8) * kTfLdK + 8 * ks + 2 * t);
        const uint32_t a[4] = {__float_as_uint(qa.x), __float_as_uint(qb.x), __float_as_uint(qa.y), __float_as_uint(qb.y)};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const float2 kv = *reinterpret_cast<const float2*>(sK + (nt * 8 + g) * kTfLdK + 8 * ks + 2 * t);
          mma_tf32_1688(s[nt], a, tf32_rna(kv.x), tf32_rna(kv.y));
        }
      }
      // scale, mask, row max (accumulator element e: row g + 8 (e / 2), key 8 nt + 2t + e % 2)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + nt * 8 + 2 * t + (e & 1);
          const float val = key < N ? s[nt][e] * scale_log2 : -INFINITY;
          s[nt][e] = val;
          mx[e >> 1] = fmaxf(mx[e >> 1], val);
        }
      }
      sm.update(s, o, mx);
      // O += P V
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const uint32_t a[4] = {tf32_rna(s[nt][0]), tf32_rna(s[nt][2]), tf32_rna(s[nt][1]), tf32_rna(s[nt][3])};
        const float* v0 = sV + (nt * 8 + 2 * t) * kTfLdV + g;
#pragma unroll
        for (int jd = 0; jd < kDH / 8; ++jd)
          mma_tf32_1688(o[jd], a, tf32_rna(v0[8 * jd]), tf32_rna(v0[kTfLdV + 8 * jd]));
      }
    }
    __syncthreads();   // every warp is done with this stage before block kb + 2 is loaded into it
  }

  if (!active) return;
  const RowNorm nrm[2] = {sm.finish(0), sm.finish(1)};
  const long ldo = (long)H * kDH;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = q0 + g + 8 * hr;
    if (row < N) {
      float* dst = out + ((long)b * N + row) * ldo + h * kDH + 2 * t;
#pragma unroll
      for (int jd = 0; jd < kDH / 8; ++jd)
        *reinterpret_cast<float2*>(dst + 8 * jd) = make_float2(nrm[hr](o[jd][2 * hr]), nrm[hr](o[jd][2 * hr + 1]));
    }
  }
}

// ---- fp32 reference-precision path: one warp per (b, h, query) ----
// Also serves Swin windows: optional additive bias[h, n, n] and mask[w % nmask, n, n]
// (tfimm/architectures/swin.py:172-194), where "b" enumerates windows.
__global__ void attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                     const float* __restrict__ bias, const float* __restrict__ mask,
                                     int nmask, long total_rows, int N, int H, int dh, float scale,
                                     float* __restrict__ probs, const int* __restrict__ row_map,
                                     int nw_img) {
  extern __shared__ float sh[];
  const int warps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sc = sh + (size_t)warp * (N + dh);
  float* qs = sc + N;
  const long rid = (long)blockIdx.x * warps + warp;
  if (rid >= total_rows) return;
  const int n = (int)(rid % N);
  const long bh = rid / N;
  const int h = (int)(bh % H);
  const long b = bh / H;
  const long ld = 3L * H * dh;
  // Token (b, j) lives in row b*N + j, or -- for Swin windows -- wherever the roll + window-partition
  // permutation put it: image (b / nw_img), token row_map[(b % nw_img) * N + j] (swin.py:299-303).
  const long row_base = row_map != nullptr ? (b / nw_img) * ((long)nw_img * N) : b * N;
  const int* rmap = row_map != nullptr ? row_map + (b % nw_img) * (long)N : nullptr;
  auto grow = [&](int j) -> long { return row_base + (rmap != nullptr ? rmap[j] : j); };
  const float* base = qkv + (long)h * dh;
  for (int d = lane; d < dh; d += 32) qs[d] = base[grow(n) * ld + d] * scale;
  __syncwarp();
  float mx = -INFINITY;
  for (int j = lane; j < N; j += 32) {
    const float* kr = base + grow(j) * ld + (long)H * dh;
    float acc = 0.f;
    for (int d = 0; d < dh; ++d) acc = fmaf(qs[d], kr[d], acc);
    if (bias != nullptr) acc += bias[((long)h * N + n) * N + j];
    if (mask != nullptr) acc += mask[((b % nmask) * N + n) * (long)N + j];
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
  if (probs != nullptr)
    for (int j = lane; j < N; j += 32) probs[((bh * N) + n) * (long)N + j] = sc[j] * inv;
  for (int d = lane; d < dh; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < N; ++j) acc = fmaf(sc[j], base[grow(j) * ld + 2L * H * dh + d], acc);
    out[grow(n) * ((long)H * dh) + (long)h * dh + d] = acc * inv;
  }
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_attention_bf16(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention: bad shape B=%d N=%d H=%d", B, N, H);
  if (dh != kDH) {
    set_last_error("attention: bf16 kernel supports head_dim 64 only (got %d)", dh);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0,
                  "attention: pointers must be 16-byte aligned");
  auto q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  auto o = reinterpret_cast<__nv_bfloat16*>(out);
  // resident K/V + one query tile per CTA must fit 227 KB: 224-row tiles up to N = 784, 128-row tiles up to N = 832
  // (vit_base_patch8_224 has N = 785); longer sequences are kUnsupported (the host falls back to the fp32 kernel)
  if (N <= 128 || N > 784) return launch_vit_attention<4, 2>(q, o, B, N, H, scale, stream);
  return launch_vit_attention<7, 2>(q, o, B, N, H, scale, stream);
}

int tfimm_b200_attention_tf32(const float* qkv, float* out, int B, int N, int H, int dh, float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention_tf32: bad shape B=%d N=%d H=%d", B, N, H);
  if (dh != kDH) {
    set_last_error("attention_tf32: head_dim 64 only (got %d)", dh);
    return kUnsupported;
  }
  TFIMM_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0,
                  "attention_tf32: pointers must be 16-byte aligned");
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(vit_attention_tf32_kernel, (int)kTfSmemBytes, attr_devs));
  dim3 grid((N + kTfRows - 1) / kTfRows, H, B);
  vit_attention_tf32_kernel<<<grid, kTfWarps * 32, kTfSmemBytes, stream>>>(qkv, out, N, H,
                                                                           scale * kLog2e);
  TFIMM_LAUNCH_OK("vit_attention_tf32_kernel");
  return kOk;
}

int tfimm_b200_attention_f32(const float* qkv, float* out, const float* bias, const float* mask, int nmask, long B,
                             int N, int H, int dh, float scale, float* probs, const int* row_map, int nw_img, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(row_map == nullptr || (nw_img > 0 && B % nw_img == 0), "attention_f32: bad window map");
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0 && dh > 0, "attention_f32: bad shape");
  const int warps = 4;
  const long total = B * H * N;
  const size_t smem = (size_t)warps * (N + dh) * sizeof(float);
  if (smem > 48 * 1024) {
    set_last_error("attention_f32: sequence too long for the fp32 parity kernel (N=%d)", N);
    return kUnsupported;
  }
  const unsigned grid = (unsigned)((total + warps - 1) / warps);
  attention_f32_kernel<<<grid, warps * 32, smem, stream>>>(qkv, out, bias, mask, nmask > 0 ? nmask : 1, total,
                                                          N, H, dh, scale, probs, row_map, nw_img > 0 ? nw_img : 1);
  TFIMM_LAUNCH_OK("attention_f32_kernel");
  return kOk;
}

}  // extern "C"
