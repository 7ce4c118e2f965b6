// Kernels of the PiT family (tfimm/architectures/pit.py): self-attention at head dims 32, 48 and 64 for any sequence
// length, and the spatial half of the pooling layer between stages.  The blocks' LayerNorms and GEMMs, the stem and the
// token Dense run on the existing paths.
//
// pit_attention_bf16_kernel<DH>  out = softmax(scale q k^T) v for one (image, head, 64-query tile) per CTA.
//   - 4 warps, 16 query rows each.  Q is loaded once by cp.async and held as mma.sync A fragments (DH / 16 k16 steps).
//   - K and V stream through a ring of kStages stages of 64 keys each, filled by cp.async and shared by the four
//     warps, so shared memory does not grow with T.  Keys past T are zero-filled by the copy and masked to -inf in the
//     scores, so they add nothing to the row sums and zero V rows to the output.
//   - Shared-memory rows are DH + 8 bf16 long: DH / 8 + 1 sixteen-byte chunks, an odd number, so the eight row
//     addresses of every ldmatrix phase fall on eight different 16-byte bank groups at DH 32, 48 and 64.
//   - S = Q K^T, the online softmax and O += P V are attention_mma.cuh's, on mma.sync m16n8k16.  The row maximum is
//     taken on the raw scores, and each score costs one fma (scale log2 e folded in) and one ex2.approx.ftz.  DH 48 is
//     three k16 steps for S and six n8 tiles for O.
//   - The normalised tile is staged through the warp's own (dead) Q rows in shared memory and stored as 16-byte
//     chunks; rows past T are not stored.
// pit_pool_kernel  the 3 x 3 / 2, groups = C, 2C-filter convolution with zero padding 1, plus bias, fp32 on the CUDA
//   cores.  A thread owns four input channels (one float4) and so the eight output channels 8 c4 .. 8 c4 + 7 that read
//   them (output o reads input o / 2); it keeps those 72 weights and 8 biases in registers and walks kPoolPix
//   consecutive output pixels.  Consecutive threads take consecutive c4 of one pixel, so loads and stores are
//   coalesced.  The grid rows are read from and written to the token streams in place: no reshape, pad or concat.
//   When asked, the same launch copies the token rows of x to bf16 (the operand of the token Dense in bf16 models).
#include "attention_mma.cuh"
#include "common.cuh"
#include "tfimm_b200_pit.h"

namespace tfimm {
namespace {

constexpr int kWarps = 4;
constexpr int kRows = kWarps * 16;  // queries per CTA
constexpr int kKeys = 64;           // keys per ring stage
constexpr int kStages = 3;

template <int DH>
struct AttnShape {
  static constexpr int kChunks = DH / 8;              // 16-byte chunks of a row of q, k or v
  static constexpr int kRowBytes = (DH + 8) * 2;      // padded shared-memory row
  static constexpr int kStageBytes = 2 * kKeys * kRowBytes;
  static constexpr int kSmem = kRows * kRowBytes + kStages * kStageBytes;
};

template <int DH>
__global__ void __launch_bounds__(kWarps * 32)
pit_attention_bf16_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int H,
                          float scale_log2) {
  using S = AttnShape<DH>;
  constexpr int RB = S::kRowBytes, CH = S::kChunks;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sRing = sQ + kRows * RB;

  const int b = blockIdx.z, h = blockIdx.y;
  const int q_base = blockIdx.x * kRows;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const long ld = 3L * H * DH;
  const __nv_bfloat16* base = qkv + (long)b * T * ld + h * DH;
  const int nblocks = (T + kKeys - 1) / kKeys;

  // one commit group per call, empty past the last block, so that wait_group counts stay uniform
  auto load_block = [&](int kb) {
    if (kb < nblocks) {
      const uint32_t sK = sRing + (kb % kStages) * S::kStageBytes;
      const uint32_t sV = sK + kKeys * RB;
      for (int idx = tid; idx < kKeys * CH; idx += kWarps * 32) {
        const int r = idx / CH, c = idx - r * CH;
        const int key = kb * kKeys + r;
        const bool valid = key < T;
        const __nv_bfloat16* src = base + (long)(valid ? key : 0) * ld + c * 8;
        cp_async_16(sK + r * RB + c * 16, src + H * DH, valid);
        cp_async_16(sV + r * RB + c * 16, src + 2 * H * DH, valid);
      }
    }
    cp_async_commit();
  };

  for (int idx = tid; idx < kRows * CH; idx += kWarps * 32) {
    const int r = idx / CH, c = idx - r * CH;
    const int row = q_base + r;
    const bool valid = row < T;
    cp_async_16(sQ + r * RB + c * 16, base + (long)(valid ? row : 0) * ld + c * 8, valid);
  }
#pragma unroll
  for (int kb = 0; kb < kStages - 1; ++kb) load_block(kb);   // Q travels in block 0's group
  cp_async_wait<kStages - 2>();
  __syncthreads();

  const int q0 = warp * 16;
  const bool active = q_base + q0 < T;
  uint32_t qf[DH / 16][4];
#pragma unroll
  for (int ks = 0; ks < DH / 16; ++ks) {
    const int row = q0 + (lane & 15);
    const int chunk = ks * 2 + (lane >> 4);
    ldmatrix_x4(sQ + row * RB + chunk * 16, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
  }
  float o[DH / 8][4];
#pragma unroll
  for (int i = 0; i < DH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  OnlineSoftmax<true> sm;

#pragma unroll 1
  for (int kb = 0; kb < nblocks; ++kb) {
    cp_async_wait<kStages - 2>();   // this thread's copies of block kb have landed
    __syncthreads();                // everyone's have, and every warp is done with block kb - 1's stage
    load_block(kb + kStages - 1);   // into that stage
    if (!active) continue;
    const uint32_t sK = sRing + (kb % kStages) * S::kStageBytes;
    const uint32_t sV = sK + kKeys * RB;
    const int key0 = kb * kKeys;
    const int nvalid = min(kKeys, T - key0);
    const int ntiles = (nvalid + 7) >> 3;   // 8-key tiles holding a key < T

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
  cp_async_wait<0>();   // only empty groups can be pending here
  if (!active) return;

  const RowNorm n0 = sm.finish(0), n1 = sm.finish(1);
  uint8_t* tile = smem + q0 * RB;   // this warp's Q rows: read only by this warp, before the key loop
#pragma unroll
  for (int nt = 0; nt < DH / 8; ++nt) {
    *reinterpret_cast<uint32_t*>(tile + g * RB + nt * 16 + t * 4) =
        pack_bf16x2(n0(o[nt][0]), n0(o[nt][1]));
    *reinterpret_cast<uint32_t*>(tile + (g + 8) * RB + nt * 16 + t * 4) =
        pack_bf16x2(n1(o[nt][2]), n1(o[nt][3]));
  }
  __syncwarp();
  const long ldo = (long)H * DH;
  for (int idx = lane; idx < 16 * CH; idx += 32) {
    const int r = idx / CH, c = idx - r * CH;
    const int row = q_base + q0 + r;
    if (row < T)
      *reinterpret_cast<uint4*>(out + ((long)b * T + row) * ldo + h * DH + c * 8) =
          *reinterpret_cast<const uint4*>(tile + r * RB + c * 16);
  }
}

template <int DH>
int launch_pit_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int H, float scale,
                         cudaStream_t stream) {
  auto kernel = pit_attention_bf16_kernel<DH>;
  static std::atomic<unsigned long long> attr_devs{0};
  TFIMM_CUDA_OK(set_max_dynamic_smem(kernel, AttnShape<DH>::kSmem, attr_devs));
  const dim3 grid((T + kRows - 1) / kRows, H, B);
  kernel<<<grid, kWarps * 32, AttnShape<DH>::kSmem, stream>>>(qkv, out, T, H, scale * kLog2e);
  TFIMM_LAUNCH_OK("pit_attention_bf16_kernel");
  return kOk;
}

constexpr int kPoolThreads = 256;
constexpr int kPoolPix = 4;   // output pixels per thread

__global__ void __launch_bounds__(kPoolThreads)
pit_pool_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ out, __nv_bfloat16* __restrict__ tokens, int B, int nb, int H, int W, int C,
                int Ho, int Wo) {
  const int C4 = C / 4;
  const long T = nb + (long)H * W, To = nb + (long)Ho * Wo;
  const long i = (long)blockIdx.x * kPoolThreads + threadIdx.x;
  if (tokens != nullptr && i < (long)B * nb * C4) {
    const long row = i / C4;   // (b, j) = (row / nb, row % nb)
    const int c4 = (int)(i - row * C4);
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + ((row / nb) * T + row % nb) * C) + c4);
    uint2 packed;
    packed.x = pack_bf16x2(v.x, v.y);
    packed.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(tokens + row * C + 4 * c4) = packed;
  }
  const long npix = (long)B * Ho * Wo;
  const long groups = (npix + kPoolPix - 1) / kPoolPix;
  if (i >= groups * C4) return;
  const int c4 = (int)(i % C4);
  const long pg = i / C4;

  float wk[9][8], bs[8];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const float4 lo = __ldg(reinterpret_cast<const float4*>(w + (long)k * 2 * C) + 2 * c4);
    const float4 hi = __ldg(reinterpret_cast<const float4*>(w + (long)k * 2 * C) + 2 * c4 + 1);
    wk[k][0] = lo.x; wk[k][1] = lo.y; wk[k][2] = lo.z; wk[k][3] = lo.w;
    wk[k][4] = hi.x; wk[k][5] = hi.y; wk[k][6] = hi.z; wk[k][7] = hi.w;
  }
  {
    const float4 lo = __ldg(reinterpret_cast<const float4*>(bias) + 2 * c4);
    const float4 hi = __ldg(reinterpret_cast<const float4*>(bias) + 2 * c4 + 1);
    bs[0] = lo.x; bs[1] = lo.y; bs[2] = lo.z; bs[3] = lo.w;
    bs[4] = hi.x; bs[5] = hi.y; bs[6] = hi.z; bs[7] = hi.w;
  }
  const long HWo = (long)Ho * Wo;
#pragma unroll 1
  for (int j = 0; j < kPoolPix; ++j) {
    const long p = pg * kPoolPix + j;
    if (p >= npix) break;
    const long b = p / HWo;
    const int r = (int)(p - b * HWo);
    const int oy = r / Wo, ox = r - oy * Wo;
    float acc[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) acc[m] = bs[m];
    const float* img = x + (b * T + nb) * C + 4 * c4;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy - 1 + ky;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * ox - 1 + kx;
        if (ix < 0 || ix >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(img + ((long)iy * W + ix) * C));
        const int k = ky * 3 + kx;
        acc[0] = fmaf(wk[k][0], v.x, acc[0]); acc[1] = fmaf(wk[k][1], v.x, acc[1]);
        acc[2] = fmaf(wk[k][2], v.y, acc[2]); acc[3] = fmaf(wk[k][3], v.y, acc[3]);
        acc[4] = fmaf(wk[k][4], v.z, acc[4]); acc[5] = fmaf(wk[k][5], v.z, acc[5]);
        acc[6] = fmaf(wk[k][6], v.w, acc[6]); acc[7] = fmaf(wk[k][7], v.w, acc[7]);
      }
    }
    float4* dst = reinterpret_cast<float4*>(out + (b * To + nb + r) * 2L * C) + 2 * c4;
    dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_pit_attention_bf16(const void* qkv, void* out, int B, int T, int H, int dh, float scale, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && T > 0 && H > 0, "pit_attention_bf16: bad shape B=%d T=%d H=%d", B, T, H);
  TFIMM_CHECK_ARG(dh == 32 || dh == 48 || dh == 64, "pit_attention_bf16: head_dim must be 32, 48 or 64 (got %d)", dh);
  TFIMM_CHECK_ARG(B <= 65535 && H <= 65535, "pit_attention_bf16: need B, H <= 65535 (B=%d H=%d)", B, H);
  TFIMM_CHECK_ARG(qkv != nullptr && out != nullptr && aligned(qkv, 16) && aligned(out, 16),
                  "pit_attention_bf16: qkv and out must be 16-byte aligned");
  auto q = reinterpret_cast<const __nv_bfloat16*>(qkv);
  auto o = reinterpret_cast<__nv_bfloat16*>(out);
  if (dh == 32) return launch_pit_attention<32>(q, o, B, T, H, scale, stream);
  if (dh == 48) return launch_pit_attention<48>(q, o, B, T, H, scale, stream);
  return launch_pit_attention<64>(q, o, B, T, H, scale, stream);
}

int tfimm_b200_pit_pool(const float* x, const float* w, const float* bias, float* out, void* tokens_bf16, int B,
                        int nb_tokens, int H, int W, int C, void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && nb_tokens >= 0,
                  "pit_pool: need B, H, W > 0, C %% 4 == 0 and nb_tokens >= 0 (B=%d H=%d W=%d C=%d nb_tokens=%d)", B,
                  H, W, C, nb_tokens);
  TFIMM_CHECK_ARG(x != nullptr && w != nullptr && bias != nullptr && out != nullptr && aligned(x, 16) &&
                      aligned(w, 16) && aligned(bias, 16) && aligned(out, 16) && aligned(tokens_bf16, 8),
                  "pit_pool: need 16-byte aligned x, w, bias, out and an 8-byte aligned tokens_bf16");
  TFIMM_CHECK_ARG(tokens_bf16 == nullptr || nb_tokens > 0, "pit_pool: tokens_bf16 given without token rows");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long C4 = C / 4;
  const long groups = ((long)B * Ho * Wo + kPoolPix - 1) / kPoolPix;
  const long threads = max(groups, tokens_bf16 != nullptr ? (long)B * nb_tokens : 0L) * C4;
  const long blocks = (threads + kPoolThreads - 1) / kPoolThreads;
  TFIMM_CHECK_ARG(blocks <= 0x7fffffffL, "pit_pool: problem too large (%ld blocks)", blocks);
  pit_pool_kernel<<<(unsigned)blocks, kPoolThreads, 0, stream>>>(x, w, bias, out,
                                                                 reinterpret_cast<__nv_bfloat16*>(tokens_bf16), B,
                                                                 nb_tokens, H, W, C, Ho, Wo);
  TFIMM_LAUNCH_OK("pit_pool_kernel");
  return kOk;
}

}  // extern "C"
