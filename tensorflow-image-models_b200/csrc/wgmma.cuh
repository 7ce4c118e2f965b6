// wgmma.mma_async m64nNk16, bf16 inputs, fp32 accumulators in registers (sm_90a), one specialisation per tile width N.
//   wgmma_ss: A and B from shared memory (descriptors, gmma_desc_k_sw128 in common.cuh); TB = 1 reads B MN-major
//             (imm-trans-b, descriptor gmma_desc_mn_sw128): the token-mixing GEMM's activation operand
//   wgmma_rs: A from registers (four bf16x2 per thread, the m64k16 A-fragment layout), B from shared memory
// accumulate == 0 overwrites d.  Accumulator element i of thread t (lane l of warp w of the warpgroup) is row
// 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
// Inline PTX cannot generate operand lists, so they are spelled out.
#pragma once
#include <stdint.h>

namespace tfimm {

#define TFIMM_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                    "+f"(d[i + 6]), "+f"(d[i + 7])

template <int N, int TB = 0>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate);
template <int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate);

template <int TB>
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %34, 0; wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, %35;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24)
               : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %66, 0; wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, %67;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56)
               : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %130, 0; wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
               "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,"
               "%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,"
               "%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, %131;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56), TFIMM_F8(64), TFIMM_F8(72), TFIMM_F8(80), TFIMM_F8(88),
                 TFIMM_F8(96), TFIMM_F8(104), TFIMM_F8(112), TFIMM_F8(120)
               : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TB));
}
template <int N, int TB>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  static_assert(N == 64 || N == 128 || N == 256, "wgmma_ss: tile width 64, 128 or 256");
  if constexpr (N == 64) wgmma_ss_n64<TB>(d, a_desc, b_desc, accumulate);
  else if constexpr (N == 128) wgmma_ss_n128<TB>(d, a_desc, b_desc, accumulate);
  else wgmma_ss_n256<TB>(d, a_desc, b_desc, accumulate);
}
template <>
__device__ __forceinline__ void wgmma_rs<96>(float (&d)[48], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %53, 0; wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47}, {%48,%49,%50,%51}, %52, p, 1, 1, 0;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %69, 0; wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 0;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_rs<192>(float (&d)[96], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %101, 0; wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
               "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, {%96,%97,%98,%99}, %100, p, 1, 1, 0;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56), TFIMM_F8(64), TFIMM_F8(72), TFIMM_F8(80), TFIMM_F8(88)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_rs<256>(float (&d)[128], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %133, 0; wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
               "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,"
               "%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,"
               "%120,%121,%122,%123,%124,%125,%126,%127}, {%128,%129,%130,%131}, %132, p, 1, 1, 0;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56), TFIMM_F8(64), TFIMM_F8(72), TFIMM_F8(80), TFIMM_F8(88),
                 TFIMM_F8(96), TFIMM_F8(104), TFIMM_F8(112), TFIMM_F8(120)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

// TF32 form (precision="tf32"): wgmma m64nNk8.f32.tf32.tf32, both operands K-major from shared memory (TF32 takes no
// transpose immediates).  A k8 step is 32 bytes of a 128-byte swizzle span, like the bf16 k16 step: the descriptors
// advance identically.
template <int N>
__device__ __forceinline__ void wgmma_ss_tf32(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate);

template <>
__device__ __forceinline__ void wgmma_ss_tf32<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc,
                                                  uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %34, 0; wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24)
               : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_ss_tf32<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc,
                                                   uint32_t accumulate) {
  asm volatile("{.reg .pred p; setp.ne.b32 p, %66, 0; wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
               "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,"
               "%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
               "%60,%61,%62,%63}, %64, %65, p, 1, 1;}"
               : TFIMM_F8(0), TFIMM_F8(8), TFIMM_F8(16), TFIMM_F8(24), TFIMM_F8(32), TFIMM_F8(40),
                 TFIMM_F8(48), TFIMM_F8(56)
               : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

#undef TFIMM_F8

}  // namespace tfimm
