// Device helpers of the scaled fp8 kernels (block_fp8.cu, scaled_fp8.cu, dequant_fp8.cu, requant_fp8.cu,
// source_quant.cu): exact widening of bf16/f16/f32 source bits to f32, |x| as an ordered integer, the folding
// 16-byte loads, the CTA max, and the 16-element narrowing x * scale -> e4m3fn (or int8) with its stores.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

#include "fp8_cvt.cuh"
#include "tsb_internal.h"

namespace tsb {

// 16-byte loads (16-element chunks) in flight per thread.  4 at 6 CTAs per SM (block_fp8_kernel: 40 registers,
// a bf16 stage is 32 KiB) measured faster on H100 than 8 at 4 CTAs per SM (64 registers), see DESIGN.md section 6.
constexpr int kUnroll = 4;

// The CTA's max of every thread's `m` (s_red: one word per warp), handed to thread0(max) in thread 0.
template <class F>
__device__ __forceinline__ void cta_max(uint32_t m, uint32_t* s_red, F&& thread0) {
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31u) == 0) s_red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t a = s_red[0];
#pragma unroll
    for (uint32_t w = 1; w < kQuantThreads / 32; ++w) a = max(a, s_red[w]);
    thread0(a);
  }
}

// The two passes over a plan's tiles (scaled_fp8.cu, requant_fp8.cu): clear the n_groups amax words on the
// stream, then the amax kernel and the quantise kernel, one CTA per tile.  `name` prefixes the error messages.
template <class Tile>
int launch_two_pass(void (*amax_kernel)(const Tile*, uint32_t*), void (*quant_kernel)(const Tile*, const uint32_t*),
                    const char* name, const Tile* tiles, uint32_t n_tiles, uint32_t* amax, uint32_t n_groups,
                    cudaStream_t stream) {
  const std::string what(name);
  const cudaError_t e = cudaMemsetAsync(amax, 0, 4ull * n_groups, stream);
  if (e != cudaSuccess) return cuda_fail(e, (what + " amax clear").c_str());
  amax_kernel<<<n_tiles, kQuantThreads, 0, stream>>>(tiles, amax);
  if (int st = launched((what + "_amax_kernel launch").c_str())) return st;
  quant_kernel<<<n_tiles, kQuantThreads, 0, stream>>>(tiles, amax);
  return launched((what + "_quant_kernel launch").c_str());
}

__device__ __forceinline__ uint4 ldg16(const char* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ float f16_bits_to_f32(uint32_t bits16) {
  const unsigned short b = static_cast<unsigned short>(bits16);
  return __half2float(*reinterpret_cast<const __half*>(&b));
}

// Source dtypes: element size and the exact widening of one element's bits to f32 bits.
template <uint32_t DT> struct Src;
template <> struct Src<TSB_F32> {
  static constexpr uint32_t kBytes = 4;
  static __device__ __forceinline__ uint32_t f32(uint32_t bits) { return bits; }
};
template <> struct Src<TSB_BF16> {
  static constexpr uint32_t kBytes = 2;
  static __device__ __forceinline__ uint32_t f32(uint32_t bits) { return bits << 16; }
};
template <> struct Src<TSB_F16> {
  static constexpr uint32_t kBytes = 2;
  static __device__ __forceinline__ uint32_t f32(uint32_t bits) { return __float_as_uint(f16_bits_to_f32(bits)); }
};

// A scaled e4m3fn source (requant_fp8.cu): two fp8 bytes (bits 0..15) -> the f32 bits of f32(q) * scale for
// each, the value a dequantising pull into f32 writes (exact widening, one correctly rounded multiply, no
// flush to zero).
__device__ __forceinline__ void scaled_e4m3x2(uint32_t two, float scale, uint32_t* lo, uint32_t* hi) {
  const uint32_t h2 = fp8x2_to_f16x2<true>(two);
  *lo = __float_as_uint(__fmul_rn(f16_bits_to_f32(h2 & 0xffffu), scale));
  *hi = __float_as_uint(__fmul_rn(f16_bits_to_f32(h2 >> 16), scale));
}

// |x| as an integer: finite < Inf < NaN
__device__ __forceinline__ uint32_t abs_bits(uint32_t f32_bits) { return f32_bits & 0x7fffffffu; }

// fold the elements of one 32-bit source word into a running max of abs_bits
template <uint32_t DT>
__device__ __forceinline__ uint32_t fold_word(uint32_t m, uint32_t w) {
  if (Src<DT>::kBytes == 4) return max(m, abs_bits(w));
  return max(m, max(abs_bits(Src<DT>::f32(w & 0xffffu)), abs_bits(Src<DT>::f32(w >> 16))));
}

// fold one 16-byte load
template <uint32_t DT>
__device__ __forceinline__ uint32_t fold16(uint32_t m, const uint4& v) {
  return fold_word<DT>(fold_word<DT>(fold_word<DT>(fold_word<DT>(m, v.x), v.y), v.z), v.w);
}

// f32 bits of element j of a chunk starting at `s` (any memory the thread may dereference)
template <uint32_t DT>
__device__ __forceinline__ uint32_t elem(const unsigned char* s, uint32_t j) {
  if (Src<DT>::kBytes == 4) return *reinterpret_cast<const uint32_t*>(s + 4 * j);
  return Src<DT>::f32(*reinterpret_cast<const unsigned short*>(s + 2 * j));
}

// the f32 bits of the 16 source words `w` (16 elements, 2 or 4 bytes each) in element order
template <uint32_t DT>
__device__ __forceinline__ void widen16(const uint4* w4, uint32_t f[16]) {
  constexpr uint32_t es = Src<DT>::kBytes;
#pragma unroll
  for (uint32_t i = 0; i < es; ++i) {
    const uint4 w = w4[i];
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {
      if constexpr (es == 4) {
        f[4 * i + k] = words[k];
      } else {
        f[8 * i + 2 * k] = Src<DT>::f32(words[k] & 0xffffu);
        f[8 * i + 2 * k + 1] = Src<DT>::f32(words[k] >> 16);
      }
    }
  }
}

// 16 elements from shared memory: `s` is 16-byte aligned when nvalid == 16; elements past nvalid are 0
template <uint32_t DT>
__device__ __forceinline__ void load16_shared(const unsigned char* s, uint32_t nvalid, uint32_t f[16]) {
  if (nvalid == 16) {
    widen16<DT>(reinterpret_cast<const uint4*>(s), f);
  } else {
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j) f[j] = j < nvalid ? elem<DT>(s, j) : 0u;
  }
}

// x * scale (correctly rounded) -> e4m3fn with torch's .to() rounding, 4 bytes per word
__device__ __forceinline__ void narrow16(const uint32_t f[16], float scale, uint32_t o[4]) {
#pragma unroll
  for (uint32_t q = 0; q < 4; ++q) {
    uint32_t x[4];
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) x[j] = __float_as_uint(__fmul_rn(__uint_as_float(f[4 * q + j]), scale));
    o[q] = f32x2_to_fp8x2<true>(x[0], x[1]) | (f32x2_to_fp8x2<true>(x[2], x[3]) << 16);
  }
}

// x * scale (correctly rounded) -> int8: round to nearest even, saturated to [-128, 127], NaN -> 0, 4 bytes per
// word.  `scale` is I8Out's: a NaN product arises exactly in the groups whose scale is not positive (a NaN group's
// scale is NaN; an Inf group's is 0, and Inf * 0 is NaN while its finite elements give +-0), so the NaN rule is
// applied per group here, not left to what the cvt does with NaN.  In a finite group scale is positive and finite
// and |x * scale| stays below 128.
__device__ __forceinline__ void narrow16_i8(const uint32_t f[16], float scale, uint32_t o[4]) {
  const bool finite_group = scale > 0.0f;
#pragma unroll
  for (uint32_t q = 0; q < 4; ++q) {
    int32_t i[4];
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) i[j] = __float2int_rn(__fmul_rn(__uint_as_float(f[4 * q + j]), scale));
    // saturate pairs to s8 and pack: bytes 2, 3 first, then 0, 1 below them
    uint32_t hi;
    asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, 0;" : "=r"(hi) : "r"(i[3]), "r"(i[2]));
    uint32_t w;
    asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(i[1]), "r"(i[0]), "r"(hi));
    o[q] = finite_group ? w : 0u;
  }
}

// the first nvalid of 16 fp8 bytes to global memory: one STG.128 when whole and aligned, else bytes
__device__ __forceinline__ void store16(char* d, uint32_t nvalid, const uint32_t o[4]) {
  if (nvalid == 16 && (reinterpret_cast<uintptr_t>(d) & 15u) == 0) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
  } else {
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j)
      if (j < nvalid) d[j] = static_cast<char>((o[j >> 2] >> (8 * (j & 3))) & 0xffu);
  }
}

// amax bits -> (scale, scale_inv) of a format whose largest magnitude is qmax (448 for e4m3fn, 127 for int8):
// amax_c = max(amax, 1e-4f), scale = qmax / amax_c, scale_inv = amax_c / qmax, both correctly rounded; a NaN amax
// gives NaN for both
__device__ __forceinline__ void scales_of_amax(uint32_t a, float* scale, float* scale_inv, float qmax = 448.0f) {
  if (a > 0x7f800000u) {
    *scale = __uint_as_float(0x7fffffffu);
    *scale_inv = *scale;
  } else {
    const float amax_c = fmaxf(__uint_as_float(a), 1e-4f);
    *scale = __fdiv_rn(qmax, amax_c);
    *scale_inv = __fdiv_rn(amax_c, qmax);
  }
}

// The UE8M0 variant (TSB_QUANT_UE8M0): scale_inv is t = amax_c / 448 (correctly rounded) when t is a power of two
// (or Inf), else the next power of two up, found on t's bits; scale = 1 / scale_inv is exact (0 for Inf).  t is
// always a normal float here (2.2e-7 <= t <= FLT_MAX / 448), so the exponent step has no subnormal or overflow
// case.  A NaN amax gives NaN for both.
__device__ __forceinline__ void ue8m0_scales_of_amax(uint32_t a, float* scale, float* scale_inv) {
  if (a > 0x7f800000u) {
    *scale = __uint_as_float(0x7fffffffu);
    *scale_inv = *scale;
  } else {
    const uint32_t t = __float_as_uint(__fdiv_rn(fmaxf(__uint_as_float(a), 1e-4f), 448.0f));
    *scale_inv = __uint_as_float((t & 0x007fffffu) ? (t & 0x7f800000u) + 0x00800000u : t);
    *scale = __fdiv_rn(1.0f, *scale_inv);
  }
}

// A group's (scale, scale_inv) from its amax bits, by the plan's scale format
template <bool kUe8m0>
__device__ __forceinline__ void group_scales(uint32_t a, float* scale, float* scale_inv) {
  if constexpr (kUe8m0)
    ue8m0_scales_of_amax(a, scale, scale_inv);
  else
    scales_of_amax(a, scale, scale_inv);
}

// The destination formats of the quantising pulls (block_fp8.cu, scaled_fp8.cu): a group's (scale, scale_inv)
// from its amax bits, and the 16-element narrowing.  Their kernels are templates on one of these.
template <bool kUe8m0>
struct E4m3Out {  // float8_e4m3fn (TSB_F8E4M3), float32 or power-of-two scales
  static __device__ __forceinline__ void scales(uint32_t a, float* scale, float* scale_inv) {
    group_scales<kUe8m0>(a, scale, scale_inv);
  }
  static __device__ __forceinline__ void narrow(const uint32_t f[16], float scale, uint32_t o[4]) { narrow16(f, scale, o); }
};
struct I8Out {  // int8 (TSB_I8), symmetric, scale step 127
  static __device__ __forceinline__ void scales(uint32_t a, float* scale, float* scale_inv) {
    scales_of_amax(a, scale, scale_inv, 127.0f);
  }
  static __device__ __forceinline__ void narrow(const uint32_t f[16], float scale, uint32_t o[4]) { narrow16_i8(f, scale, o); }
};

}  // namespace tsb
