// The scalar conversions of the fused casts, all bit-exact with torch's .to() (round to nearest even; the fp8
// rules are fp8_cvt.cuh's), shared by the copy kernel (copy_rects.cu) and the transposing mover
// (transpose_rects.cu): convert<S, D>(v) for every pair tsb_cast_supported accepts.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "fp8_cvt.cuh"

namespace tsb {

template <typename S, typename D>
__device__ __forceinline__ D convert(S v);
template <> __device__ __forceinline__ __nv_bfloat16 convert<float, __nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half convert<float, __half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ float convert<__nv_bfloat16, float>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float convert<__half, float>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ __half convert<__nv_bfloat16, __half>(__nv_bfloat16 v) { return __float2half_rn(__bfloat162float(v)); }
template <> __device__ __forceinline__ __nv_bfloat16 convert<__half, __nv_bfloat16>(__half v) { return __float2bfloat16_rn(__half2float(v)); }
template <> __device__ __forceinline__ float convert<double, float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double convert<float, double>(float v) { return static_cast<double>(v); }

// ---- fp8 (float8_e4m3fn, float8_e5m2) ------------------------------------------------------------
// Storage tags of the fp8 side of a scalar cast (the vector movers handle raw bytes).
struct F8E4M3 { unsigned char x; };
struct F8E5M2 { unsigned char x; };

// The e4m3fn / e5m2 narrowing (f32x2_to_fp8x2, fp8_fix), the fp8 widening (fp8x2_to_f16x2) and the
// f32 -> bf16 narrowing (float_to_bf16_bits) live in fp8_cvt.cuh.
__device__ __forceinline__ float f16_bits_to_float(uint32_t bits16) {
  unsigned short b = static_cast<unsigned short>(bits16);
  return __half2float(*reinterpret_cast<__half*>(&b));
}

template <> __device__ __forceinline__ F8E4M3 convert<float, F8E4M3>(float v) { return F8E4M3{static_cast<unsigned char>(f32x2_to_fp8x2<true>(__float_as_uint(v), 0u))}; }
template <> __device__ __forceinline__ F8E5M2 convert<float, F8E5M2>(float v) { return F8E5M2{static_cast<unsigned char>(f32x2_to_fp8x2<false>(__float_as_uint(v), 0u))}; }
template <> __device__ __forceinline__ F8E4M3 convert<__nv_bfloat16, F8E4M3>(__nv_bfloat16 v) { return convert<float, F8E4M3>(__bfloat162float(v)); }
template <> __device__ __forceinline__ F8E5M2 convert<__nv_bfloat16, F8E5M2>(__nv_bfloat16 v) { return convert<float, F8E5M2>(__bfloat162float(v)); }
template <> __device__ __forceinline__ F8E4M3 convert<__half, F8E4M3>(__half v) { return convert<float, F8E4M3>(__half2float(v)); }
template <> __device__ __forceinline__ F8E5M2 convert<__half, F8E5M2>(__half v) { return convert<float, F8E5M2>(__half2float(v)); }
template <> __device__ __forceinline__ float convert<F8E4M3, float>(F8E4M3 v) { return f16_bits_to_float(fp8x2_to_f16x2<true>(v.x)); }
template <> __device__ __forceinline__ float convert<F8E5M2, float>(F8E5M2 v) { return f16_bits_to_float(fp8x2_to_f16x2<false>(v.x)); }
template <> __device__ __forceinline__ __half convert<F8E4M3, __half>(F8E4M3 v) { return __float2half_rn(convert<F8E4M3, float>(v)); }
template <> __device__ __forceinline__ __half convert<F8E5M2, __half>(F8E5M2 v) { return __float2half_rn(convert<F8E5M2, float>(v)); }
template <> __device__ __forceinline__ __nv_bfloat16 convert<F8E4M3, __nv_bfloat16>(F8E4M3 v) { return __float2bfloat16_rn(convert<F8E4M3, float>(v)); }
template <> __device__ __forceinline__ __nv_bfloat16 convert<F8E5M2, __nv_bfloat16>(F8E5M2 v) { return __float2bfloat16_rn(convert<F8E5M2, float>(v)); }

}  // namespace tsb
