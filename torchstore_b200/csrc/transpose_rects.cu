// Transposing pulls (sm_90a, H100): move rects whose destination is contiguous along its last dim and whose
// source is contiguous along the destination's dim -2, i.e. dst[..., i, j] = to_dst(src[..., j, i]) for an
// input-major trainer weight read into an output-major generator parameter (PackedPart(transpose=True)).
// The copy kernel would move such a rect one element per access on the source side; this one reads and writes
// whole 16-byte sectors on both sides.
//
// Host side: every rect is cut into square tiles of T x T elements (T = 64 for 1- and 2-byte sources, 32 for 4-
// and 8-byte ones) of each 2-D slice of its outer dims; one 48-byte record per tile (the table grows with rects
// and tiles, not with elements), grouped by dtype pair.
// Device side: one persistent launch per dtype pair, SMs x resident CTAs, each CTA striding over the tiles.  A
// tile is read with 16-byte loads along the source's contiguous dim into a shared-memory tile whose row pitch is
// one bank (two for 8-byte elements) more than the tile's bytes, so the transposed reads of the write phase hit at
// most 2 ways per bank; it is written back with 16-byte stores along the destination's contiguous dim, the fused
// cast (cast_cvt.cuh, bit-exact with torch's .to()) applied at the store.  Edge tiles, and rows that are not
// 16-byte aligned on either side, take per-element accesses in the same kernel.

#include <algorithm>
#include <cstring>
#include <memory>
#include <type_traits>

#include "cast_cvt.cuh"
#include "tsb_internal.h"

namespace tsb {

namespace {

constexpr uint32_t kTrThreads = 256;

// One T x T (or edge) tile of a transposed rect.  Element (i, j), i < rows, j < cols, moves from
// src + i * sizeof(src elem) + j * src_stride to dst + i * dst_stride + j * sizeof(dst elem).
struct alignas(8) TrTile {
  uint64_t src;          // source element of destination (0, 0)
  uint64_t dst;          // destination element (0, 0)
  int64_t src_stride;    // bytes between source rows (consecutive destination columns)
  int64_t dst_stride;    // bytes between destination rows
  uint32_t rows, cols;   // destination extent: rows run along the source's contiguous dim
  uint8_t src_dtype, dst_dtype;
  uint8_t vec;           // bit 0: 16-byte source loads, bit 1: 16-byte destination stores
  uint8_t pad0_;
  uint32_t pad1_;
};
static_assert(sizeof(TrTile) == 48, "TrTile is part of tsb_transpose_compile_host's output");

uint32_t tr_bytes(uint32_t dt) {
  switch (dt) {
    case TSB_U8: case TSB_F8E4M3: case TSB_F8E5M2: return 1;
    case TSB_U16: case TSB_F16: case TSB_BF16: return 2;
    case TSB_U32: case TSB_F32: return 4;
    case TSB_U64: case TSB_F64: return 8;
    default: return 0;
  }
}
__host__ __device__ constexpr uint32_t tile_edge(uint32_t src_bytes) { return src_bytes <= 2 ? 64 : 32; }

template <uint32_t DT> struct Ty;
template <> struct Ty<TSB_U8> { using T = uint8_t; };
template <> struct Ty<TSB_U16> { using T = uint16_t; };
template <> struct Ty<TSB_U32> { using T = uint32_t; };
template <> struct Ty<TSB_U64> { using T = uint64_t; };
template <> struct Ty<TSB_F16> { using T = __half; };
template <> struct Ty<TSB_BF16> { using T = __nv_bfloat16; };
template <> struct Ty<TSB_F32> { using T = float; };
template <> struct Ty<TSB_F64> { using T = double; };
template <> struct Ty<TSB_F8E4M3> { using T = F8E4M3; };
template <> struct Ty<TSB_F8E5M2> { using T = F8E5M2; };

template <uint32_t B> struct Raw;
template <> struct Raw<1> { using T = uint8_t; };
template <> struct Raw<2> { using T = uint16_t; };
template <> struct Raw<4> { using T = uint32_t; };
template <> struct Raw<8> { using T = unsigned long long; };

template <class S, class D>
__device__ __forceinline__ D cvt(S v) {
  if constexpr (std::is_same_v<S, D>) return v;
  else return convert<S, D>(v);
}

__device__ __forceinline__ uint4 ldg16(const char* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void stg16(char* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

template <class S, class D>
__global__ void __launch_bounds__(kTrThreads) transpose_kernel(const TrTile* __restrict__ tiles, uint32_t n_tiles) {
  constexpr uint32_t sb = sizeof(S), db = sizeof(D);
  using RS = typename Raw<sb>::T;
  constexpr uint32_t T = tile_edge(sb);
  constexpr uint32_t P = T * sb + (sb < 4 ? 4 : sb);  // shared row pitch (bytes): one source row per destination column
  constexpr uint32_t SE = 16 / sb;                    // elements per 16-byte source chunk
  constexpr uint32_t SC = T / SE;                     // chunks per source row of a full tile
  constexpr uint32_t DE = 16 / db;                    // elements per 16-byte destination chunk
  constexpr uint32_t DC = T / DE;                     // chunks per destination row of a full tile
  constexpr uint32_t kLoads = (T * SC + kTrThreads - 1) / kTrThreads;
  constexpr uint32_t kStores = (T * DC + kTrThreads - 1) / kTrThreads;
  __shared__ __align__(16) unsigned char s[T * P];
  for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const TrTile tile = tiles[t];
    const char* src = reinterpret_cast<const char*>(tile.src);
    char* dst = reinterpret_cast<char*>(tile.dst);
    const bool vs = tile.vec & 1u, vd = tile.vec & 2u;
    // load: source row j (destination column j), chunk c along i (destination rows)
    uint4 v[kLoads];
#pragma unroll
    for (uint32_t k = 0; k < kLoads; ++k) {
      const uint32_t idx = threadIdx.x + k * kTrThreads;
      const uint32_t j = idx / SC, i0 = (idx % SC) * SE;
      if (idx < T * SC && j < tile.cols && vs && i0 + SE <= tile.rows) v[k] = ldg16(src + static_cast<int64_t>(j) * tile.src_stride + i0 * sb);
    }
#pragma unroll
    for (uint32_t k = 0; k < kLoads; ++k) {
      const uint32_t idx = threadIdx.x + k * kTrThreads;
      const uint32_t j = idx / SC, i0 = (idx % SC) * SE;
      if (idx >= T * SC || j >= tile.cols || i0 >= tile.rows) continue;
      unsigned char* d = s + j * P + i0 * sb;
      if (vs && i0 + SE <= tile.rows) {
        uint32_t* w = reinterpret_cast<uint32_t*>(d);
        w[0] = v[k].x;
        w[1] = v[k].y;
        w[2] = v[k].z;
        w[3] = v[k].w;
      } else {
        const RS* p = reinterpret_cast<const RS*>(src + static_cast<int64_t>(j) * tile.src_stride + i0 * sb);
        for (uint32_t e = 0; e < SE && i0 + e < tile.rows; ++e) reinterpret_cast<RS*>(d)[e] = __ldg(p + e);
      }
    }
    __syncthreads();
    // store: destination row i, chunk c along j
#pragma unroll
    for (uint32_t k = 0; k < kStores; ++k) {
      const uint32_t idx = threadIdx.x + k * kTrThreads;
      const uint32_t i = idx / DC, j0 = (idx % DC) * DE;
      if (idx >= T * DC || i >= tile.rows || j0 >= tile.cols) continue;
      union {
        uint4 u;
        typename Raw<db>::T r[DE];
      } o;
#pragma unroll
      for (uint32_t e = 0; e < DE; ++e) {
        const D y = cvt<S, D>(*reinterpret_cast<const S*>(s + (j0 + e) * P + i * sb));
        o.r[e] = *reinterpret_cast<const typename Raw<db>::T*>(&y);
      }
      char* d = dst + static_cast<int64_t>(i) * tile.dst_stride + j0 * db;
      if (vd && j0 + DE <= tile.cols) {
        stg16(d, o.u);
      } else {
#pragma unroll
        for (uint32_t e = 0; e < DE; ++e)
          if (j0 + e < tile.cols) reinterpret_cast<typename Raw<db>::T*>(d)[e] = o.r[e];
      }
    }
    __syncthreads();
  }
}

using TrKernel = void (*)(const TrTile*, uint32_t);

template <uint32_t SD, uint32_t DD>
TrKernel k() { return transpose_kernel<typename Ty<SD>::T, typename Ty<DD>::T>; }

// The kernel of a dtype pair: same-dtype moves by element size, and every fused cast of tsb_cast_supported.
TrKernel kernel_for(uint32_t s, uint32_t d) {
  if (s == d) {
    switch (tr_bytes(s)) {
      case 1: return k<TSB_U8, TSB_U8>();
      case 2: return k<TSB_U16, TSB_U16>();
      case 4: return k<TSB_U32, TSB_U32>();
      case 8: return k<TSB_U64, TSB_U64>();
      default: return nullptr;
    }
  }
#define TSB_TR(a, b) \
  if (s == a && d == b) return k<a, b>();
  TSB_TR(TSB_F32, TSB_BF16) TSB_TR(TSB_F32, TSB_F16) TSB_TR(TSB_BF16, TSB_F32) TSB_TR(TSB_F16, TSB_F32)
  TSB_TR(TSB_BF16, TSB_F16) TSB_TR(TSB_F16, TSB_BF16) TSB_TR(TSB_F64, TSB_F32) TSB_TR(TSB_F32, TSB_F64)
  TSB_TR(TSB_F32, TSB_F8E4M3) TSB_TR(TSB_F32, TSB_F8E5M2) TSB_TR(TSB_BF16, TSB_F8E4M3) TSB_TR(TSB_BF16, TSB_F8E5M2)
  TSB_TR(TSB_F16, TSB_F8E4M3) TSB_TR(TSB_F16, TSB_F8E5M2) TSB_TR(TSB_F8E4M3, TSB_F32) TSB_TR(TSB_F8E5M2, TSB_F32)
  TSB_TR(TSB_F8E4M3, TSB_BF16) TSB_TR(TSB_F8E5M2, TSB_BF16) TSB_TR(TSB_F8E4M3, TSB_F16) TSB_TR(TSB_F8E5M2, TSB_F16)
#undef TSB_TR
  return nullptr;
}

int transpose_compile(int device, const tsb_rect_t* rects, uint64_t n, std::vector<TrTile>* tiles, PlanBytes* bytes) {
  if (n && !rects) return fail(TSB_ERR_INVALID, "transpose: NULL rects");
  for (uint64_t i = 0; i < n; ++i) {
    const tsb_rect_t& r = rects[i];
    const std::string what = "rect " + std::to_string(i);
    if (r.ndim < 2 || r.ndim > TSB_MAX_DIMS)
      return fail(TSB_ERR_INVALID, what + ": a transposed rect has 2 to TSB_MAX_DIMS dims, not " + std::to_string(r.ndim));
    const uint32_t sb = tr_bytes(r.src_dtype), db = tr_bytes(r.dst_dtype);
    if (!sb || !db)
      return fail(TSB_ERR_INVALID, what + ": unknown dtype " + std::to_string(sb ? r.dst_dtype : r.src_dtype));
    if (!kernel_for(r.src_dtype, r.dst_dtype))
      return fail(TSB_ERR_UNSUPPORTED, what + ": no transposing kernel for dtype " + std::to_string(r.src_dtype) +
                                           " -> " + std::to_string(r.dst_dtype) + " (tsb_cast_supported pairs and same-dtype moves only)");
    if (!r.src || !r.dst) return fail(TSB_ERR_INVALID, what + ": NULL src or dst");
    const uint32_t nd = r.ndim;
    uint64_t outer = 1;
    bool empty = false;
    for (uint32_t d = 0; d < nd; ++d) {
      if (r.extent[d] < 0) return fail(TSB_ERR_INVALID, what + ": negative extent");
      if (r.extent[d] == 0) empty = true;
      if (r.src_stride[d] % sb || r.dst_stride[d] % db)
        return fail(TSB_ERR_INVALID, what + ": strides must be whole elements");
      if (d + 2 < nd) outer *= static_cast<uint64_t>(r.extent[d]);
    }
    if (r.src % sb || r.dst % db) return fail(TSB_ERR_INVALID, what + ": src and dst must be element-aligned");
    if (empty) continue;
    const uint64_t A = r.extent[nd - 2], B = r.extent[nd - 1];
    if (B > 1 && r.dst_stride[nd - 1] != db)
      return fail(TSB_ERR_INVALID, what + ": not a transposed rect: its destination is not contiguous along its last dim");
    if (A > 1 && r.src_stride[nd - 2] != sb)
      return fail(TSB_ERR_INVALID, what + ": not a transposed rect: its source is not contiguous along the destination's "
                                          "dim -2");
    if (A > 0xffffffffull || B > 0xffffffffull) return fail(TSB_ERR_UNSUPPORTED, what + ": extent of 2^32 or more");
    const uint32_t T = tile_edge(sb);
    for (uint64_t o = 0; o < outer; ++o) {
      int64_t so = 0, dof = 0;
      for (uint64_t rem = o, d = nd - 2; d-- > 0;) {  // outer index, innermost outer dim fastest
        const uint64_t e = static_cast<uint64_t>(r.extent[d]), x = rem % e;
        rem /= e;
        so += static_cast<int64_t>(x) * r.src_stride[d];
        dof += static_cast<int64_t>(x) * r.dst_stride[d];
      }
      for (uint64_t a = 0; a < A; a += T) {
        for (uint64_t b = 0; b < B; b += T) {
          TrTile t;
          memset(&t, 0, sizeof(t));
          t.src = r.src + so + a * sb + b * r.src_stride[nd - 1];
          t.dst = r.dst + dof + a * r.dst_stride[nd - 2] + b * db;
          t.src_stride = r.src_stride[nd - 1];
          t.dst_stride = r.dst_stride[nd - 2];
          t.rows = static_cast<uint32_t>(std::min<uint64_t>(T, A - a));
          t.cols = static_cast<uint32_t>(std::min<uint64_t>(T, B - b));
          t.src_dtype = static_cast<uint8_t>(r.src_dtype);
          t.dst_dtype = static_cast<uint8_t>(r.dst_dtype);
          t.vec = (aligned16(t.src, t.src_stride, t.cols) ? 1 : 0) | (aligned16(t.dst, t.dst_stride, t.rows) ? 2 : 0);
          tiles->push_back(t);
        }
      }
    }
    const uint64_t elems = outer * A * B;
    bytes->read(elems * sb, r.src_device, device);
    bytes->payload_bytes += elems * db;
    if (tiles->size() >= (1ull << 31)) return fail(TSB_ERR_UNSUPPORTED, "transpose: more than 2^31 tiles");
  }
  // one launch per dtype pair: group the tiles by pair, keeping rect order inside a group
  std::stable_sort(tiles->begin(), tiles->end(), [](const TrTile& x, const TrTile& y) {
    return x.src_dtype != y.src_dtype ? x.src_dtype < y.src_dtype : x.dst_dtype < y.dst_dtype;
  });
  return TSB_OK;
}

// d = TrTile table; one persistent launch per dtype pair
int transpose_plan(int device, const tsb_rect_t* rects, uint64_t n, QuantPlan* q) {
  std::vector<TrTile> tiles;
  PlanBytes bytes;
  if (int st = transpose_compile(device, rects, n, &tiles, &bytes)) return st;
  q->add(tiles);
  q->seal(0);
  struct Group {
    TrKernel kernel;
    uint32_t first, count, grid;
  };
  auto groups = std::make_shared<std::vector<Group>>();
  for (uint32_t i = 0; i < tiles.size();) {
    uint32_t e = i;
    while (e < tiles.size() && tiles[e].src_dtype == tiles[i].src_dtype && tiles[e].dst_dtype == tiles[i].dst_dtype) ++e;
    groups->push_back({kernel_for(tiles[i].src_dtype, tiles[i].dst_dtype), i, e - i, 0});
    i = e;
  }
  const uint32_t n_tiles = static_cast<uint32_t>(tiles.size());
  q->describe(n, n_tiles, tile_edge(2) * tile_edge(2), bytes);
  q->launch = [device, groups](char* d, cudaStream_t s) -> int {
    for (Group& g : *groups) {
      if (!g.grid) {  // SMs x resident CTAs, found at the first launch (compile_host makes no CUDA call)
        int sm = 0, per_sm = 0;
        if (int st = device_sm_count(device, &sm)) return st;
        TSB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, g.kernel, kTrThreads, 0));
        g.grid = std::max<uint32_t>(1, std::min<uint32_t>(g.count, static_cast<uint32_t>(sm) * std::max(1, per_sm)));
      }
      g.kernel<<<g.grid, kTrThreads, 0, s>>>(reinterpret_cast<const TrTile*>(d) + g.first, g.count);
      if (int st = launched("transpose_kernel launch")) return st;
    }
    return TSB_OK;
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_transpose_plan_create(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, tsb_plan_t* out) {
  return quant_plan_create("tsb_transpose_plan_create", device, flags, 0, out,
                           [&](QuantPlan* q) { return transpose_plan(device, rects, n, q); });
}

extern "C" int tsb_transpose_compile_host(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, void* out_tiles,
                                          uint64_t tile_cap, uint64_t* out_n_tiles) {
  return quant_compile_host("tsb_transpose_compile_host", flags, 0,
                            [&](QuantPlan* q) { return transpose_plan(device, rects, n, q); },
                            {{out_tiles, tile_cap, out_n_tiles, "out_tiles"}}, nullptr);
}
