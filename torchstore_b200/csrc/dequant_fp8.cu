// Dequantising pulls (sm_90a, H100): gather block-, channel- or tensor-scaled float8_e4m3fn or int8 source
// rectangles into f32 / bf16 / f16 destinations, y = to_dst(f32(q) * scale), the torch rendering
// (q.float() * s_expanded).to(dst) of DeepSeek's weight_dequant.  One plan reads one source format; its
// launch picks the kernel instantiation (E4m3In / I8In), the tables are the same for both.
//
// Host side: the plan compiler maps every rect's *source* onto its source shard's [batch, rows, cols]
// grid (rect_source_boxes, block_fp8.cu), cuts the boxes at the scale groups (128x128 blocks anchored at
// the global origin through the shard's (row0, col0) phase; per channel and per tensor no cut is needed:
// a tile carries the scale of its first row and the step to the next row's) and splits them into tiles of
// at most kDqTileElems elements and kDqTileRows rows, so that a big shard spreads over every SM.
// Device side: one 256-thread CTA per tile, streaming, no reduction and no shared-memory staging of data.
// Each thread takes 16 fp8 (or int8) elements per step, kUnroll steps in flight: one 16-byte load when the tile is
// aligned, widening (exact), one f32 multiply per element (__fmul_rn: round to nearest even, no flush to
// zero), the fused cast's narrowing, then 32 B (bf16/f16) or 64 B (f32) of 16-byte stores.  A channel
// tile's scales are staged in shared memory once per row; block and tensor tiles load their one scale.
// Ragged or misaligned chunks take a scalar path.

#include <algorithm>
#include <cstring>

#include "fp8_quant.cuh"
#include "tsb_internal.h"

namespace tsb {

int dq_source_geoms(const tsb_dq_source_t* sources, uint64_t n_sources, std::vector<TargetGeom>* out) {
  constexpr GridRules kSourceRules{"source", "NULL src or scale", "src", "scale",
                                   (1u << TSB_SCALE_PER_BLOCK) | (1u << TSB_SCALE_PER_CHANNEL) | (1u << TSB_SCALE_PER_TENSOR), 1ull << 31};
  std::vector<TargetGeom>& geom = *out;
  geom.resize(n_sources);
  for (uint64_t s = 0; s < n_sources; ++s) {
    const tsb_dq_source_t& S = sources[s];
    int st = check_grid(kSourceRules, s, {S.src, S.scale, S.batch, S.rows, S.cols, S.row0, S.col0, 1, S.granularity, S.pad, !S.src || !S.scale});
    if (st) return st;
    geom[s] = {S.src, S.batch, S.rows, S.cols};
  }
  return TSB_OK;
}

namespace {

int dequant_fp8_compile(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                        uint64_t n_sources, DqTables* out) {
  if ((n && !rects) || (n_sources && !sources)) return fail(TSB_ERR_INVALID, "dequant_fp8: NULL rects or sources");
  std::vector<TargetGeom> geom;
  int st = dq_source_geoms(sources, n_sources, &geom);
  if (st) return st;
  std::vector<TargetBox> boxes;
  for (uint64_t i = 0; i < n; ++i) {
    if ((st = rect_source_boxes(rects[i], i, geom.data(), n_sources, &boxes))) return st;
  }
  for (const TargetBox& x : boxes) {
    const tsb_dq_source_t& S = sources[x.target];
    const uint32_t es = quant_src_bytes(x.dtype);
    const bool block = S.granularity == TSB_SCALE_PER_BLOCK;
    const uint64_t g = block ? kBqBlock : ~0ull;  // group edge in both dims (block), else no cut
    // block grid of the shard's scale tensor: blocks anchored at the global origin
    const uint64_t br0 = S.row0 / kBqBlock, bc0 = S.col0 / kBqBlock;
    const uint64_t nbr = (S.row0 + S.rows + kBqBlock - 1) / kBqBlock - br0, nbc = (S.col0 + S.cols + kBqBlock - 1) / kBqBlock - bc0;
    // box row y reads source row x.r0 + rs * y (rs 2: a rotary head half); a block cut falls where that row
    // crosses a block edge
    const uint64_t rs = x.rstep;
    for (uint64_t y0 = 0; y0 < x.er;) {
      const uint64_t sy = x.r0 + rs * y0;
      const uint64_t y1 = block ? std::min(x.er, y0 + (((S.row0 + sy) / g + 1) * g - S.row0 - sy + rs - 1) / rs) : x.er;
      for (uint64_t c0 = x.c0; c0 < x.c0 + x.ec;) {
        const uint64_t c1 = block ? std::min(x.c0 + x.ec, ((S.col0 + c0) / g + 1) * g - S.col0) : x.c0 + x.ec;
        uint64_t scale;
        if (block)
          scale = S.scale + 4 * ((x.b * nbr + (S.row0 + sy) / kBqBlock - br0) * nbc + (S.col0 + c0) / kBqBlock - bc0);
        else if (S.granularity == TSB_SCALE_PER_CHANNEL)
          scale = S.scale + 4 * (x.b * S.rows + sy);
        else
          scale = S.scale + 4 * x.b;
        const uint16_t step = S.granularity == TSB_SCALE_PER_CHANNEL ? static_cast<uint16_t>(4 * rs) : 0;
        const uint64_t h = y1 - y0, w = c1 - c0;
        const uint64_t tr = std::min<uint64_t>(kDqTileRows, std::max<uint64_t>(1, kDqTileElems / w));
        const uint64_t tc = std::min<uint64_t>(w, kDqTileElems);
        for (uint64_t r = 0; r < h; r += tr) {
          for (uint64_t c = 0; c < w; c += tc) {
            DqTile t;
            memset(&t, 0, sizeof(t));
            t.rows = static_cast<uint32_t>(std::min(tr, h - r));
            t.cols = static_cast<uint32_t>(std::min(tc, w - c));
            t.src = S.src + (x.b * S.rows + sy + rs * r) * S.cols + c0 + c;
            t.src_stride = static_cast<int64_t>(rs * S.cols);
            t.dst = x.src + (y0 + r) * x.row_stride + (c0 + c - x.c0) * es;
            t.dst_stride = x.row_stride;
            t.scale = scale + step * r;
            t.scale_step = step;
            t.dst_dtype = static_cast<uint8_t>(x.dtype);
            t.vec = aligned16(t.src, t.src_stride, t.rows) && aligned16(t.dst, t.dst_stride, t.rows) ? 1 : 0;
            out->tiles.push_back(t);
            const uint64_t elems = static_cast<uint64_t>(t.rows) * t.cols;
            out->read(elems, x.src_device, device);
            out->payload_bytes += elems * es;
          }
        }
        c0 = c1;
      }
      y0 = y1;
    }
    if (out->tiles.size() >= (1ull << 31)) return fail(TSB_ERR_UNSUPPORTED, "dequant_fp8: more than 2^31 tiles");
  }
  return TSB_OK;
}

// f32 -> destination bits: the fused cast's narrowing (copy_rects.cu), identity for f32
template <uint32_t DT> __device__ __forceinline__ uint32_t narrow_bits(float y);
template <> __device__ __forceinline__ uint32_t narrow_bits<TSB_F32>(float y) { return __float_as_uint(y); }
template <> __device__ __forceinline__ uint32_t narrow_bits<TSB_BF16>(float y) { return float_to_bf16_bits(y); }
template <> __device__ __forceinline__ uint32_t narrow_bits<TSB_F16>(float y) { return __half_as_ushort(__float2half_rn(y)); }

// The source formats: the exact widening to f32 of one byte (widen1), and of the two bytes in bits 0..15 (pair,
// then lo and hi of its result)
struct E4m3In {  // float8_e4m3fn (TSB_F8E4M3): through f16, NaN stays NaN
  static __device__ __forceinline__ uint32_t pair(uint32_t two) { return fp8x2_to_f16x2<true>(two); }
  static __device__ __forceinline__ float lo(uint32_t p) { return f16_bits_to_f32(p & 0xffffu); }
  static __device__ __forceinline__ float hi(uint32_t p) { return f16_bits_to_f32(p >> 16); }
  static __device__ __forceinline__ float widen1(uint32_t byte) { return lo(pair(byte)); }
};
struct I8In {  // int8 (TSB_I8): (float)(int8_t)b
  static __device__ __forceinline__ uint32_t pair(uint32_t two) { return two; }
  static __device__ __forceinline__ float lo(uint32_t p) { return static_cast<float>(static_cast<int8_t>(p & 0xffu)); }
  static __device__ __forceinline__ float hi(uint32_t p) { return static_cast<float>(static_cast<int8_t>((p >> 8) & 0xffu)); }
  static __device__ __forceinline__ float widen1(uint32_t byte) { return lo(byte); }
};

template <uint32_t DT, class In>
__device__ __forceinline__ void dequant_tile(const DqTile& t, const float* s_scale, float scale0) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const char* src = reinterpret_cast<const char*>(t.src);
  char* dst = reinterpret_cast<char*>(t.dst);
  const uint32_t cpr = (t.cols + 15u) / 16u;
  const uint32_t total = t.rows * cpr;
  for (uint32_t base = threadIdx.x; base < total; base += kQuantThreads * kUnroll) {
    uint4 v[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t idx = base + k * kQuantThreads;
      if (idx < total) {
        const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
        if (t.vec && c + 16u <= t.cols) v[k] = ldg16(src + static_cast<int64_t>(r) * t.src_stride + c);
      }
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t idx = base + k * kQuantThreads;
      if (idx >= total) continue;
      const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
      const float scale = t.scale_step ? s_scale[r] : scale0;
      char* d = dst + static_cast<int64_t>(r) * t.dst_stride + static_cast<uint64_t>(c) * es;
      if (t.vec && c + 16u <= t.cols) {
        const uint32_t words[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
        uint32_t o[4 * es];
#pragma unroll
        for (uint32_t j = 0; j < 8; ++j) {  // element pairs (2j, 2j+1)
          const uint32_t h2 = In::pair(words[j >> 1] >> (16 * (j & 1)));
          const uint32_t lo = narrow_bits<DT>(__fmul_rn(In::lo(h2), scale));
          const uint32_t hi = narrow_bits<DT>(__fmul_rn(In::hi(h2), scale));
          if constexpr (es == 4) {
            o[2 * j] = lo;
            o[2 * j + 1] = hi;
          } else {
            o[j] = lo | (hi << 16);
          }
        }
#pragma unroll
        for (uint32_t i = 0; i < es; ++i)
          asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(d + 16 * i), "r"(o[4 * i]), "r"(o[4 * i + 1]),
                       "r"(o[4 * i + 2]), "r"(o[4 * i + 3]) : "memory");
      } else {
        const unsigned char* s = reinterpret_cast<const unsigned char*>(src + static_cast<int64_t>(r) * t.src_stride + c);
        const uint32_t nvalid = min(16u, t.cols - c);
        for (uint32_t j = 0; j < nvalid; ++j) {
          const uint32_t y = narrow_bits<DT>(__fmul_rn(In::widen1(__ldg(s + j)), scale));
          if constexpr (es == 4)
            *reinterpret_cast<uint32_t*>(d + 4 * j) = y;
          else
            *reinterpret_cast<unsigned short*>(d + 2 * j) = static_cast<unsigned short>(y);
        }
      }
    }
  }
}

// In: the source format, E4m3In or I8In (one per plan).  kStepped: channel tiles may read every other source row
// (a rotary head half), so a row's scale is scale_step bytes after the previous one; otherwise 4 bytes.
template <class In, bool kStepped = false>
__global__ void __launch_bounds__(kQuantThreads) dequant_fp8_kernel(const DqTile* __restrict__ tiles) {
  __shared__ float s_scale[kDqTileRows];
  const DqTile t = tiles[blockIdx.x];
  const float* scales = reinterpret_cast<const float*>(t.scale);
  float scale0 = 0.0f;
  if (t.scale_step) {  // per channel: one scale per row, fetched once
    for (uint32_t r = threadIdx.x; r < t.rows; r += kQuantThreads)
      s_scale[r] = __ldg(kStepped ? scales + r * (t.scale_step / 4u) : scales + r);
    __syncthreads();
  } else {
    scale0 = __ldg(scales);
  }
  switch (t.dst_dtype) {
    case TSB_BF16: dequant_tile<TSB_BF16, In>(t, s_scale, scale0); break;
    case TSB_F16: dequant_tile<TSB_F16, In>(t, s_scale, scale0); break;
    default: dequant_tile<TSB_F32, In>(t, s_scale, scale0); break;
  }
}

// Whether the rects of a dequantising pull (each already checked by rect_source_boxes) read int8 (TSB_I8) rather
// than float8_e4m3fn: TSB_ERR_INVALID when they mix the two.
int dq_src_int8(const tsb_rect_t* rects, uint64_t n, bool* int8) {
  *int8 = n && rects[0].src_dtype == TSB_I8;
  for (uint64_t i = 1; i < n; ++i)
    if ((rects[i].src_dtype == TSB_I8) != *int8)
      return fail(TSB_ERR_INVALID, "rect " + std::to_string(i) + ": the rects of one plan read one source dtype, "
                                   "float8_e4m3fn or int8");
  return TSB_OK;
}

// d = DqTile table, one CTA per tile
int dequant_fp8_plan(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources, uint64_t n_sources,
                     QuantPlan* q) {
  DqTables tb;
  int st = dequant_fp8_compile(device, rects, n, sources, n_sources, &tb);
  if (st || (st = dq_src_int8(rects, n, &q->int8))) return st;
  q->add(tb.tiles);
  q->seal(0);
  const uint32_t n_tiles = static_cast<uint32_t>(tb.tiles.size());
  q->describe(n, n_tiles, kDqTileElems, tb);
  // plans with rotary channel tiles (scale step 8) take the stepped instantiations, every other plan the plain ones
  const bool stepped = std::any_of(tb.tiles.begin(), tb.tiles.end(), [](const DqTile& t) { return t.scale_step > 4; });
  const auto kernel = stepped ? (q->int8 ? dequant_fp8_kernel<I8In, true> : dequant_fp8_kernel<E4m3In, true>)
                              : (q->int8 ? dequant_fp8_kernel<I8In> : dequant_fp8_kernel<E4m3In>);
  q->launch = [n_tiles, kernel](char* d, cudaStream_t s) {
    kernel<<<n_tiles, kQuantThreads, 0, s>>>(reinterpret_cast<const DqTile*>(d));
    return launched("dequant_fp8_kernel launch");
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_dequant_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                           uint64_t n_sources, uint32_t flags, tsb_plan_t* out) {
  return quant_plan_create("tsb_dequant_fp8_plan_create", device, flags, 0, out,
                           [&](QuantPlan* q) { return dequant_fp8_plan(device, rects, n, sources, n_sources, q); });
}

extern "C" int tsb_dequant_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                            uint64_t n_sources, uint32_t flags, void* out_tiles, uint64_t tile_cap,
                                            uint64_t* out_n_tiles) {
  return quant_compile_host("tsb_dequant_fp8_compile_host", flags, 0,
                            [&](QuantPlan* q) { return dequant_fp8_plan(device, rects, n, sources, n_sources, q); },
                            {{out_tiles, tile_cap, out_n_tiles, "out_tiles"}}, nullptr);
}
