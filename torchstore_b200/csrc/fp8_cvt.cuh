// fp8 <-> f32 conversions with torch's .to() semantics, shared by the copy kernel (copy_rects.cu), the
// scaled quantisers (block_fp8.cu, scaled_fp8.cu) and the dequantiser (dequant_fp8.cu).
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

namespace tsb {

// The narrowing cvt exists only in .satfinite form: values past the largest finite one and +-Inf
// saturate to it, and every NaN becomes one canonical NaN.  torch's .to() instead rounds to nearest
// even all the way: e4m3fn has no Inf, so whatever rounds past 448 (|x| > 464), +-Inf and NaN become
// 0x7F|sign; e5m2 overflows to +-Inf (0x7C|sign) from |x| >= 61440 on, and a NaN keeps its sign
// (0x7F|sign).  fp8_fix replaces the cvt's byte for exactly those inputs; below the thresholds the
// cvt already rounds like torch (subnormals included).  An f16 source is widened with cvt.f32.f16 like
// torch's CUDA .to() does, which makes every NaN positive: a negative f16 NaN gives 0x7F, as in torch.
template <bool kE4M3>
__device__ __forceinline__ uint32_t fp8_fix(uint32_t cvt_byte, uint32_t f32_bits) {
  const uint32_t a = f32_bits & 0x7fffffffu;
  const uint32_t sign = (f32_bits >> 24) & 0x80u;
  if (kE4M3) return a > 0x43e80000u /* 464.0f */ ? (0x7fu | sign) : cvt_byte;
  return a >= 0x47700000u /* 61440.0f */ ? ((a > 0x7f800000u ? 0x7fu : 0x7cu) | sign) : cvt_byte;
}
// two f32 bit patterns -> two fp8 bytes (lo in bits 0..7, hi in bits 8..15)
template <bool kE4M3>
__device__ __forceinline__ uint32_t f32x2_to_fp8x2(uint32_t lo, uint32_t hi) {
  unsigned short r;
  if (kE4M3)
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__uint_as_float(hi)), "f"(__uint_as_float(lo)));
  else
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__uint_as_float(hi)), "f"(__uint_as_float(lo)));
  return fp8_fix<kE4M3>(r & 0xffu, lo) | (fp8_fix<kE4M3>(static_cast<uint32_t>(r) >> 8, hi) << 8);
}

// two fp8 bytes (bits 0..15) -> f16x2 (exact: every fp8 value is an f16 value)
template <bool kE4M3>
__device__ __forceinline__ uint32_t fp8x2_to_f16x2(uint32_t two) {
  uint32_t r;
  const unsigned short b = static_cast<unsigned short>(two);
  if (kE4M3) asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(b));
  else asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(r) : "h"(b));
  return r;
}

// f32 -> bf16 bits, round to nearest even (the fused cast's narrowing, NaN bytes included)
__device__ __forceinline__ uint32_t float_to_bf16_bits(float f) {
  __nv_bfloat16 h = __float2bfloat16_rn(f);
  return *reinterpret_cast<unsigned short*>(&h);
}

}  // namespace tsb
