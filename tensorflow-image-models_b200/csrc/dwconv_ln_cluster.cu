// ConvNeXt block head on sm_90a:  ZeroPadding2D(3) -> DepthwiseConv2D(7x7, bias) -> LayerNorm over C
// (tfimm/architectures/convnext.py:189-198, 219-223), channel-slab / thread-block-cluster formulation.
//
// A depthwise 7x7 is 49 MACs per element: FP32-FMA bound on the CUDA cores (not HBM bound) *if* the taps and
// the input halo come from on-chip memory and the instruction stream is mostly FMAs.  LayerNorm needs every
// channel of a pixel.  Both are reconciled by splitting the channels of one 14x7 pixel tile over the CTAs of a
// thread-block cluster; clusters are persistent and walk over the tiles of the batch:
//
//   CTA (cluster rank r) owns channels [r*CS, (r+1)*CS) (CS = 64 or 32) of the current 14(rows) x 7(cols) tile
//     A. ONE 4-D TMA box copy (C, W, H, B) brings the 20x13xCS fp32 input halo into shared memory; the
//        zero padding of the convolution is the TMA out-of-bounds fill (negative / past-the-edge coordinates),
//        so there is no index arithmetic or predicate in the load path at all
//     B. a thread keeps the 49 taps of ONE channel pair in registers (packed fp32x2, loaded once per kernel)
//        and computes a 2-row x 7-column output block: every 8-byte shared-memory load (one halo pixel, two
//        channels, already fp32x2) feeds up to 14 fp32 pair FMAs; 686 per 104 loads.  Results (+bias) go to an
//        fp32 stash [98][CS] in shared memory, so the LayerNorm sees exact fp32 convolution outputs
//        -> the halo buffer is free again: the TMA copy of the cluster's NEXT tile is issued here
//     C. LayerNorm statistics: per-pixel (sum, centred second moment) of the slab, exchanged between the CTAs
//        of the cluster through distributed shared memory and merged with the parallel-variance formula
//     D. normalise the own slab and write bf16 rows (16 B per lane)
// The tile loop is software-pipelined: the cluster barrier is split (arrive after C of tile i, wait after the
// FMA phase B of tile i+1), so the DSMEM exchange latency hides behind FMA work; stash and partial statistics
// are double-buffered for that.  224 threads per CTA; shared memory ~119 KB for CS = 64 (one CTA per SM) and ~60 KB
// for CS = 32 (two CTAs per SM, so one CTA's FMA phase also overlaps the other's statistics / store phases).
#include "common.cuh"

#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace tfimm {
namespace {

constexpr int kTH = 14;              // output tile rows (7 row pairs)
constexpr int kTW = 7;               // output tile columns
constexpr int kHH = kTH + 6;         // 20 halo rows
constexpr int kHW = kTW + 6;         // 13 halo columns
constexpr int kPix = kTH * kTW;      // 98
constexpr int kWarps = kTH / 2;      // one warp per output row pair
constexpr int kThreads = kWarps * 32;

template <int CS>
struct DwCfg {
  static constexpr int kPairs = CS / 2;                  // channel pairs per slab (<= 32: one lane each)
  static constexpr int kOct = CS / 8;                    // 8-channel groups per pixel row
  static constexpr int kPixPerWarp = 32 / kOct;          // pixels per warp step in phases C/D
  static constexpr int kHaloBytes = kHH * kHW * CS * 4;  // fp32
  static constexpr int kStashBytes = kPix * CS * 4;      // fp32, per buffer (two buffers)
  static constexpr int kStatBytes = kPix * 4 * 6;        // 2 x (part_sum, part_m2), mean, rstd
  static constexpr int kSmemBytes = kHaloBytes + 2 * kStashBytes + kStatBytes + 16;
};

template <int CS>
__global__ void __launch_bounds__(kThreads, CS == 32 ? 2 : 1)   // CS = 64: the fp32 stash allows one CTA per SM
dwconv7_ln_cluster_kernel(const __grid_constant__ CUtensorMap tmap_x, const float* __restrict__ wgt /*[49][C]*/,
                          const float* __restrict__ bias, const float* __restrict__ gamma,
                          const float* __restrict__ beta, __nv_bfloat16* __restrict__ out, int H, int W, int C,
                          int tiles_x, int tiles_per_img, int n_tiles, int cluster_size, float eps) {
  using Cfg = DwCfg<CS>;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint64_t* halo = reinterpret_cast<const uint64_t*>(smem);                 // [20*13][CS/2] fp32x2
  float* stash_base = reinterpret_cast<float*>(smem + Cfg::kHaloBytes);          // 2 x [98][CS] fp32
  float* part_base = reinterpret_cast<float*>(smem + Cfg::kHaloBytes + 2 * Cfg::kStashBytes);  // 2 x (sum, m2)[98]
  float* s_mean = part_base + 4 * kPix;
  float* s_rstd = s_mean + kPix;
  const uint32_t bar = smem_u32(s_rstd + kPix);
  const uint32_t halo_addr = smem_u32(smem);

  cg::cluster_group cluster = cg::this_cluster();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int crank = (int)cluster.block_rank();
  const int cluster_id = blockIdx.x / cluster_size, n_clusters = gridDim.x / cluster_size;
  const int c_base = crank * CS;

  if (tid == 0) {
    prefetch_tmap(&tmap_x);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto issue_halo = [&](int tile) {
    const int b = tile / tiles_per_img, t = tile % tiles_per_img;
    mbar_expect_tx(bar, Cfg::kHaloBytes);
    tma_load_4d(halo_addr, &tmap_x, bar, c_base, (t % tiles_x) * kTW - 3, (t / tiles_x) * kTH - 3, b);
  };
  int tile = cluster_id;
  if (tid == 0 && tile < n_tiles) issue_halo(tile);

  // taps of this lane's channel pair: registers for the whole kernel
  const bool pair_on = lane < Cfg::kPairs;
  const int c0 = c_base + 2 * (pair_on ? lane : 0);
  uint64_t w[49];
#pragma unroll
  for (int t = 0; t < 49; ++t) w[t] = pack2(__ldg(wgt + (size_t)t * C + c0), __ldg(wgt + (size_t)t * C + c0 + 1));
  const uint64_t bv = pack2(__ldg(bias + c0), __ldg(bias + c0 + 1));

  const int q = lane / Cfg::kOct, o = lane % Cfg::kOct;  // phases C/D: pixel slot / channel octet of this lane
  const float inv_c = 1.0f / (float)C;

  auto load8 = [&](const float* stash, int p, float (&v)[8]) { ld8(stash + (size_t)p * CS + o * 8, v); };
  auto oct_sum = [&](float s) {
#pragma unroll
    for (int off = 1; off < Cfg::kOct; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    return s;
  };

  // ---- C. slab statistics per pixel: sum and second moment about the slab mean ----
  auto slab_stats = [&](int t, int buf) {
    const int t_in_img = t % tiles_per_img;
    const int ty0 = (t_in_img / tiles_x) * kTH, tx0 = (t_in_img % tiles_x) * kTW;
    const float* stash = stash_base + (size_t)buf * kPix * CS;
    float* part_sum = part_base + buf * 2 * kPix;
    float* part_m2 = part_sum + kPix;
    for (int p0 = warp * Cfg::kPixPerWarp; p0 < kPix; p0 += kWarps * Cfg::kPixPerWarp) {
      const int p = p0 + q;
      const bool ok = p < kPix && (ty0 + p / kTW) < H && (tx0 + p % kTW) < W;
      float v[8];
      if (ok) load8(stash, p, v);
      else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
      const float s = oct_sum(((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7])));
      const float m = s * (1.0f / CS);
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) d += (v[j] - m) * (v[j] - m);
      d = oct_sum(d);
      if (o == 0 && p < kPix) {
        part_sum[p] = s;
        part_m2[p] = ok ? d : 0.f;
      }
    }
  };

  // ---- merge the slabs of the cluster, then D. normalise the own slab and write ----
  auto finish_tile = [&](int t, int buf) {
    const int b = t / tiles_per_img, t_in_img = t % tiles_per_img;
    const int ty0 = (t_in_img / tiles_x) * kTH, tx0 = (t_in_img % tiles_x) * kTW;
    const float* stash = stash_base + (size_t)buf * kPix * CS;
    float* part_sum = part_base + buf * 2 * kPix;
    float* part_m2 = part_sum + kPix;
    // Chan et al.: M2 = sum_r [ M2_r + CS * (mean_r - mean)^2 ]
    for (int p = tid; p < kPix; p += kThreads) {
      float s = 0.f;
      for (int r = 0; r < cluster_size; ++r) s += cluster.map_shared_rank(part_sum, r)[p];
      const float mean = s * inv_c;
      float m2 = 0.f;
      for (int r = 0; r < cluster_size; ++r) {
        const float dm = cluster.map_shared_rank(part_sum, r)[p] * (1.0f / CS) - mean;
        m2 += cluster.map_shared_rank(part_m2, r)[p] + (float)CS * dm * dm;
      }
      s_mean[p] = mean;
      s_rstd[p] = rsqrtf(m2 * inv_c + eps);
    }
    __syncthreads();
    float g[8], be[8];
    *reinterpret_cast<float4*>(&g[0]) = __ldg(reinterpret_cast<const float4*>(gamma + c_base + o * 8));
    *reinterpret_cast<float4*>(&g[4]) = __ldg(reinterpret_cast<const float4*>(gamma + c_base + o * 8 + 4));
    *reinterpret_cast<float4*>(&be[0]) = __ldg(reinterpret_cast<const float4*>(beta + c_base + o * 8));
    *reinterpret_cast<float4*>(&be[4]) = __ldg(reinterpret_cast<const float4*>(beta + c_base + o * 8 + 4));
    for (int p0 = warp * Cfg::kPixPerWarp; p0 < kPix; p0 += kWarps * Cfg::kPixPerWarp) {
      const int p = p0 + q;
      if (!(p < kPix && (ty0 + p / kTW) < H && (tx0 + p % kTW) < W)) continue;
      const float rs = s_rstd[p], mrs = -s_mean[p] * rs;
      float v[8];
      load8(stash, p, v);
      float y[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = fmaf(fmaf(v[j], rs, mrs), g[j], be[j]);
      uint4 u;
      u.x = pack_bf16x2(y[0], y[1]);
      u.y = pack_bf16x2(y[2], y[3]);
      u.z = pack_bf16x2(y[4], y[5]);
      u.w = pack_bf16x2(y[6], y[7]);
      __nv_bfloat16* orow = out + (((long)b * H + ty0 + p / kTW) * W + tx0 + p % kTW) * C + c_base + o * 8;
      *reinterpret_cast<uint4*>(orow) = u;
    }
  };

  int it = 0, prev_tile = -1;
  for (; tile < n_tiles; tile += n_clusters, ++it) {
    const int buf = it & 1;
    const int ty0 = ((tile % tiles_per_img) / tiles_x) * kTH;
    mbar_wait(bar, (uint32_t)(it & 1));
    // every thread is past D of tile it-1 (same stash parity as it+1) and C of tile it-2 before B writes
    __syncthreads();

    // ---- B. depthwise 7x7: warp = output row pair, lane = channel pair ----
    const int oy0 = 2 * warp;
    if (pair_on && ty0 + oy0 < H) {
      uint64_t acc0[7], acc1[7];
#pragma unroll
      for (int i = 0; i < 7; ++i) acc0[i] = acc1[i] = bv;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint64_t* row = halo + (size_t)((oy0 + r) * kHW) * Cfg::kPairs + lane;
#pragma unroll
        for (int ix = 0; ix < kHW; ++ix) {
          const uint64_t v = row[(size_t)ix * Cfg::kPairs];
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) {
            const int ox = ix - kx;
            if (ox >= 0 && ox < 7) {
              if (r <= 6) acc0[ox] = fma2(v, w[r * 7 + kx], acc0[ox]);
              if (r >= 1) acc1[ox] = fma2(v, w[(r - 1) * 7 + kx], acc1[ox]);
            }
          }
        }
      }
      float2* st0 =
          reinterpret_cast<float2*>(stash_base + (size_t)buf * kPix * CS) + (size_t)(oy0 * kTW) * Cfg::kPairs + lane;
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        float a0, a1;
        unpack2(acc0[i], a0, a1);
        st0[(size_t)i * Cfg::kPairs] = make_float2(a0, a1);
        unpack2(acc1[i], a0, a1);
        st0[(size_t)(kTW + i) * Cfg::kPairs] = make_float2(a0, a1);
      }
    }
    __syncthreads();
    // halo buffer is free: fetch the next tile of this cluster while the statistics / store phases run
    if (tid == 0 && tile + n_clusters < n_tiles) issue_halo(tile + n_clusters);

    if (prev_tile >= 0) {
      cluster_wait_acquire();  // partial statistics of the previous tile are visible cluster-wide
      finish_tile(prev_tile, buf ^ 1);
    }
    slab_stats(tile, buf);
    cluster_arrive_release();
    prev_tile = tile;
  }
  if (prev_tile >= 0) {
    cluster_wait_acquire();
    finish_tile(prev_tile, (it - 1) & 1);
  }
  // a CTA must not exit while peers may still read its partial statistics through DSMEM
  cluster.sync();
}

template <int CS>
int launch_cluster(const void* x, const float* wgt, const float* bias, const float* gamma, const float* beta,
                   void* out, int B, int H, int W, int C, float eps, cudaStream_t stream) {
  using Cfg = DwCfg<CS>;
  auto kernel = dwconv7_ln_cluster_kernel<CS>;
  const int cl = C / CS;
  static std::atomic<unsigned long long> attr_devs{0};
  static int max_clusters[17] = {0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, Cfg::kSmemBytes, attr_devs, /*nonportable_cluster=*/true));
  const int tiles_x = (W + kTW - 1) / kTW, tiles_y = (H + kTH - 1) / kTH;
  const long n_tiles = (long)B * tiles_x * tiles_y;

  CUtensorMap tmap;
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
  const uint32_t box[4] = {(uint32_t)CS, (uint32_t)kHW, (uint32_t)kHH, 1u};
  int rc = make_tmap(&tmap, x, kF32, 4, dims, strides, box, "dwconv7_ln input", /*swizzle_128b=*/false);
  if (rc != kOk) return rc;

  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cl;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (max_clusters[cl] == 0) {
    cfg.gridDim = dim3((unsigned)(cl * 64));
    int n = 0;
    TFIMM_CUDA_OK(cudaOccupancyMaxActiveClusters(&n, kernel, &cfg));
    if (n <= 0) return kUnsupported;  // this cluster size cannot be co-scheduled on the device
    max_clusters[cl] = n;
  }
  const long n_clusters = n_tiles < max_clusters[cl] ? n_tiles : max_clusters[cl];
  cfg.gridDim = dim3((unsigned)(n_clusters * cl));
  TFIMM_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, tmap, wgt, bias, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out),
                                   H, W, C, tiles_x, tiles_x * tiles_y, (int)n_tiles, cl, eps));
  return kOk;
}

}  // namespace

// Returns kUnsupported (without setting an error) when the shape does not fit the cluster formulation, so the
// caller can use the generic kernel.
int dwconv7_ln_cluster(const void* x, int in_dtype, const float* wgt, const float* bias, const float* gamma,
                       const float* beta, void* out, int out_dtype, int B, int H, int W, int C, float eps,
                       cudaStream_t stream) {
  if (out_dtype != kBF16 || in_dtype != kF32) return kUnsupported;
  if ((long)B * H * W * C >= (1L << 40) || (reinterpret_cast<uintptr_t>(x) & 15u) != 0) return kUnsupported;
  if (C % 64 == 0 && C / 64 <= 16) return launch_cluster<64>(x, wgt, bias, gamma, beta, out, B, H, W, C, eps, stream);
  if (C % 32 == 0 && C / 32 <= 16) return launch_cluster<32>(x, wgt, bias, gamma, beta, out, B, H, W, C, eps, stream);
  return kUnsupported;
}

}  // namespace tfimm
