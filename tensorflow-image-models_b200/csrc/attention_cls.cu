// Attention for the first `nq` query tokens only (class / distillation tokens), all keys.
//
// ViT.forward_features returns token 0 (or tokens 0..1 for the distilled DeiTs) of the LAST block's output
// (tfimm/architectures/vit.py:452-464): in that block only the class-token rows of softmax(QK^T)V, proj, norm2 and
// the MLP influence the logits (keys and values still come from every token).  This kernel is the attention core
// of that pruned last block: one warp per (image, head, query token), fp32 math, bf16 in / out.
//   scores: lanes own keys j = lane, lane + 32, ... (64-dim dot products against q kept in shared memory)
//   softmax: warp-wide max / sum in fp32
//   output: lanes own two of the 64 head dimensions; p_j is broadcast by shuffle, V rows are read coalesced
#include "common.cuh"

namespace tfimm {
namespace {

constexpr int kDh = 64;
constexpr int kMaxKeysPerLane = 16;  // N <= 512

__global__ void __launch_bounds__(128)
attention_cls_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int B, int N, int H, int nq,
                     float scale) {
  __shared__ float q_sh[4][kDh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long unit = (long)blockIdx.x * 4 + warp;
  const long units = (long)B * H * nq;
  if (unit >= units) return;
  const int qi = (int)(unit % nq);
  const int h = (int)((unit / nq) % H);
  const int b = (int)(unit / ((long)nq * H));
  const int D = H * kDh;
  const __nv_bfloat16* base = qkv + (long)b * N * 3 * D;
  {
    const float2 q2 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(base + (long)qi * 3 * D + h * kDh + 2 * lane));
    q_sh[warp][2 * lane] = q2.x * scale;
    q_sh[warp][2 * lane + 1] = q2.y * scale;
  }
  __syncwarp();
  float s[kMaxKeysPerLane];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < kMaxKeysPerLane; ++i) {
    const int j = lane + 32 * i;
    s[i] = -INFINITY;
    if (j < N) {
      const __nv_bfloat16* k = base + (long)j * 3 * D + D + h * kDh;
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < kDh; d += 8) {
        float v[8];
        ld8(k + d, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc = fmaf(v[e], q_sh[warp][d + e], acc);
      }
      s[i] = acc;
      mx = fmaxf(mx, acc);
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxKeysPerLane; ++i) {
    const float p = (lane + 32 * i < N) ? __expf(s[i] - mx) : 0.f;
    s[i] = p;
    sum += p;
  }
  const float inv = 1.0f / warp_sum(sum);
  float o0 = 0.f, o1 = 0.f;
  const __nv_bfloat16* vbase = base + 2 * D + h * kDh + 2 * lane;
#pragma unroll
  for (int i = 0; i < kMaxKeysPerLane; ++i) {
    if (32 * i >= N) break;
    const int cnt = min(32, N - 32 * i);
    for (int l = 0; l < cnt; ++l) {
      const float p = __shfl_sync(0xffffffffu, s[i], l);
      const float2 v2 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vbase + (long)(32 * i + l) * 3 * D));
      o0 = fmaf(p, v2.x, o0);
      o1 = fmaf(p, v2.y, o1);
    }
  }
  *reinterpret_cast<uint32_t*>(out + ((long)b * nq + qi) * D + h * kDh + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
}

}  // namespace

}  // namespace tfimm

using namespace tfimm;

extern "C" {

int tfimm_b200_attention_cls_bf16(const void* qkv, void* out, int B, int N, int H, int dh, int nq, float scale,
                                  void* s) {
  const cudaStream_t stream = as_stream(s);
  TFIMM_CHECK_ARG(B > 0 && N > 0 && H > 0 && nq > 0 && nq <= N, "attention_cls: bad shape");
  TFIMM_CHECK_ARG(dh == kDh, "attention_cls: head_dim must be 64 (got %d)", dh);
  TFIMM_CHECK_ARG(N <= 32 * kMaxKeysPerLane, "attention_cls: at most %d tokens (got %d)", 32 * kMaxKeysPerLane, N);
  const long units = (long)B * H * nq;
  attention_cls_kernel<<<(unsigned)((units + 3) / 4), 128, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(out), B, N, H, nq, scale);
  TFIMM_LAUNCH_OK("attention_cls_kernel");
  return kOk;
}

}  // extern "C"
