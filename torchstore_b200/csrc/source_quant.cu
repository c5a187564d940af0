// Source-side quantisation (sm_90a, H100): a publisher's refresh of block-, channel- or tensor-scaled
// float8_e4m3fn (or int8) staging from its live bf16/f16/f32 shards, the producer half of the scaled weight sync.
//
// Groups are shard-local and anchored at the global origin, the layout a scaled source handle describes
// (tsb_dq_source_t): a block-scaled shard at global offset (row0, col0) has one group per global 128x128 block
// it touches, cut to the shard, so an FSDP shard starting mid-block gets partial first and last block rows.
// Per group the formula of the quantising pulls applies, from the same device helpers (fp8_quant.cuh): the staging
// format (E4m3Out / I8Out) picks the unit kernel (source_quant_kernel / source_int8_kernel) and the two-pass kernels.
//
// Host side: every target is cut into work in group order, with trivial addressing (a shard is one
// contiguous tensor; there are no pieces):
//   blocks, and per-channel rows of at most kSqStageBytes source bytes -> units (one CTA each)
//   per-tensor matrices and longer per-channel rows                   -> two-pass tiles of at most kSqTileElems
// Device side:
//   source_quant_kernel<DT>  one 256-thread CTA per unit, one launch per source dtype (units are grouped by dtype,
//                            so an f32 unit's register budget never lowers the occupancy of bf16 units).  Each
//                            thread issues every 16-byte load of its (at most 4) 16-element chunks up front into
//                            registers, folds |x| into its group's amax (warp redux + one shared atomicMax per warp
//                            and group), and after the scales are known narrows the same registers and stores.  Each
//                            source byte is read once; with 4 resident CTAs per SM (bf16/f16) one CTA's loads are in
//                            flight while the others quantise and store.  Units whose rows are not 16-byte aligned
//                            load element by element into the same registers.
//   two-pass tiles           scaled_fp8.cu's amax and quantise kernels (the tile format is SqTile); the amax words
//                            are cleared on the launch stream before pass 1, so a replayed plan starts from zero.

#include <algorithm>
#include <array>
#include <cstring>

#include "fp8_quant.cuh"
#include "tsb_internal.h"

namespace tsb {

namespace {

struct Compiler {
  SrcQTables* out;

  void unit(const tsb_source_quant_target_t& T, uint32_t es, uint64_t src_elem, uint64_t scale_inv, uint64_t rows,
            uint64_t cols, bool per_row) {
    SrcQUnit u;
    memset(&u, 0, sizeof(u));
    u.src = T.src + src_elem * es;
    u.dst = T.dst + src_elem;
    u.scale_inv = scale_inv;
    u.src_pitch = static_cast<uint32_t>(T.cols * es);
    u.dst_pitch = static_cast<uint32_t>(T.cols);
    u.rows = static_cast<uint32_t>(rows);
    u.cols = static_cast<uint32_t>(cols);
    u.per_row = per_row ? 1u : 0u;
    u.src_dtype = static_cast<uint16_t>(T.src_dtype);
    u.vec = vec_ok(u.src, u.src_pitch, rows, cols, es) ? 1 : 0;
    out->unit_bytes = std::max<uint32_t>(out->unit_bytes, static_cast<uint32_t>(rows * cols * es));
    out->units.push_back(u);
    out->src_bytes += rows * cols * es;
  }

  // `n` contiguous elements from element `first` as one two-pass group; its first tile writes `scale_inv`
  void group(const tsb_source_quant_target_t& T, uint32_t es, uint64_t first, uint64_t n, uint64_t scale_inv) {
    const uint32_t g = out->n_groups++;
    for (uint64_t c = 0; c < n; c += kSqTileElems) {
      SqTile t;
      memset(&t, 0, sizeof(t));
      const uint64_t cols = std::min<uint64_t>(kSqTileElems, n - c);
      t.src = T.src + (first + c) * es;
      t.dst = T.dst + first + c;
      t.scale = c == 0 ? scale_inv : 0;
      t.dst_pitch = static_cast<uint32_t>(cols);
      t.rows = 1;
      t.cols = static_cast<uint32_t>(cols);
      t.group = g;
      t.src_dtype = T.src_dtype;
      t.vec = vec_ok(t.src, 0, 1, cols, es) ? 1u : 0u;
      out->tiles.push_back(t);
      out->src_bytes += cols * es;
    }
  }

  void target(const tsb_source_quant_target_t& T) {
    const uint32_t es = quant_src_bytes(T.src_dtype);
    if (T.granularity == TSB_SCALE_PER_BLOCK) {
      const uint64_t br0 = T.row0 / kBqBlock, br1 = (T.row0 + T.rows + kBqBlock - 1) / kBqBlock;
      const uint64_t bc0 = T.col0 / kBqBlock, bc1 = (T.col0 + T.cols + kBqBlock - 1) / kBqBlock;
      for (uint64_t b = 0; b < T.batch; ++b) {
        for (uint64_t i = br0; i < br1; ++i) {
          const uint64_t r0 = std::max(i * kBqBlock, T.row0) - T.row0, r1 = std::min((i + 1) * kBqBlock, T.row0 + T.rows) - T.row0;
          for (uint64_t j = bc0; j < bc1; ++j) {
            const uint64_t c0 = std::max(j * kBqBlock, T.col0) - T.col0, c1 = std::min((j + 1) * kBqBlock, T.col0 + T.cols) - T.col0;
            const uint64_t s = ((b * (br1 - br0) + i - br0) * (bc1 - bc0) + j - bc0);
            unit(T, es, (b * T.rows + r0) * T.cols + c0, T.scale_inv + 4 * s, r1 - r0, c1 - c0, false);
          }
        }
      }
    } else if (T.granularity == TSB_SCALE_PER_CHANNEL) {
      const uint64_t all = T.batch * T.rows;  // per channel, the matrices of a stack are consecutive rows
      const uint32_t spitch = round16(T.cols * es);
      const uint64_t cpr = (T.cols + 15) / 16;  // 16-element chunks per row
      if (spitch > kSqStageBytes || cpr > kSrcQChunks * kQuantThreads) {
        for (uint64_t r = 0; r < all; ++r) group(T, es, r * T.cols, T.cols, T.scale_inv + 4 * r);
        return;
      }
      const uint64_t per_band =
          std::min<uint64_t>(std::min<uint64_t>(kSqBandRows, kSqStageBytes / spitch), kSrcQChunks * kQuantThreads / cpr);
      for (uint64_t r = 0; r < all; r += per_band)
        unit(T, es, r * T.cols, T.scale_inv + 4 * r, std::min(per_band, all - r), T.cols, true);
    } else {
      for (uint64_t b = 0; b < T.batch; ++b) group(T, es, b * T.rows * T.cols, T.rows * T.cols, T.scale_inv + 4 * b);
    }
  }
};

constexpr GridRules kTargetRules{"target", "NULL src, dst or scale_inv", "src", "scale_inv",
                                 (1u << TSB_SCALE_PER_BLOCK) | (1u << TSB_SCALE_PER_CHANNEL) | (1u << TSB_SCALE_PER_TENSOR), 1ull << 30};

int source_quant_compile(const tsb_source_quant_target_t* targets, uint64_t n, SrcQTables* out) {
  if (n && !targets) return fail(TSB_ERR_INVALID, "source_quant: NULL targets");
  Compiler cc{out};
  for (uint64_t t = 0; t < n; ++t) {
    const tsb_source_quant_target_t& T = targets[t];
    const uint32_t es = quant_src_bytes(T.src_dtype);
    if (!es)
      return fail(TSB_ERR_INVALID, "target " + std::to_string(t) + ": src_dtype must be TSB_F32, TSB_BF16 or TSB_F16, not " +
                                       std::to_string(T.src_dtype));
    int st = check_grid(kTargetRules, t, {T.src, T.scale_inv, T.batch, T.rows, T.cols, T.row0, T.col0, es, T.granularity, 0,
                                          !T.src || !T.dst || !T.scale_inv});
    if (st) return st;
    uint64_t groups = T.batch;
    if (T.granularity == TSB_SCALE_PER_CHANNEL) groups *= T.rows;
    if (T.granularity == TSB_SCALE_PER_BLOCK)
      groups *= ((T.row0 + T.rows + kBqBlock - 1) / kBqBlock - T.row0 / kBqBlock) *
                ((T.col0 + T.cols + kBqBlock - 1) / kBqBlock - T.col0 / kBqBlock);
    out->payload_bytes += T.batch * T.rows * T.cols + 4 * groups;
    cc.target(T);
    if (out->units.size() >= (1ull << 31) || out->tiles.size() >= (1ull << 31) || out->n_groups >= (1u << 31))
      return fail(TSB_ERR_UNSUPPORTED, "source_quant: more than 2^31 units, tiles or groups");
  }
  // one launch per source dtype: bf16, f16, f32
  const auto rank = [](const SrcQUnit& u) { return u.src_dtype == TSB_BF16 ? 0 : u.src_dtype == TSB_F16 ? 1 : 2; };
  std::stable_sort(out->units.begin(), out->units.end(), [&](const SrcQUnit& a, const SrcQUnit& b) { return rank(a) < rank(b); });
  for (const SrcQUnit& u : out->units) ++out->n_units[rank(u)];
  return TSB_OK;
}

// Load the first `nvalid` elements of a 16-element chunk at `s` into `d` (its source words; the rest 0).
template <uint32_t DT>
__device__ __forceinline__ void load_chunk(const char* s, uint32_t nvalid, bool vec, uint32_t d[4 * Src<DT>::kBytes]) {
  constexpr uint32_t es = Src<DT>::kBytes;
#pragma unroll
  for (uint32_t i = 0; i < 4 * es; ++i) d[i] = 0;
  if (vec) {  // nvalid * es is a multiple of 16 here
#pragma unroll
    for (uint32_t i = 0; i < es; ++i) {
      if (16 * i < nvalid * es) {
        const uint4 v = ldg16(s + 16 * i);
        d[4 * i] = v.x;
        d[4 * i + 1] = v.y;
        d[4 * i + 2] = v.z;
        d[4 * i + 3] = v.w;
      }
    }
  } else {
#pragma unroll
    for (uint32_t k = 0; k < 16; ++k) {
      if (k < nvalid) {
        if (es == 4)
          d[k] = __ldg(reinterpret_cast<const uint32_t*>(s) + k);
        else
          d[k / 2] |= static_cast<uint32_t>(__ldg(reinterpret_cast<const unsigned short*>(s) + k)) << (16 * (k & 1));
      }
    }
  }
}

// the f32 bits of a chunk's 16 elements from its source words
template <uint32_t DT>
__device__ __forceinline__ void widen_chunk(const uint32_t d[4 * Src<DT>::kBytes], uint32_t f[16]) {
#pragma unroll
  for (uint32_t k = 0; k < 16; ++k) {
    if constexpr (Src<DT>::kBytes == 4)
      f[k] = d[k];
    else
      f[k] = Src<DT>::f32((d[k / 2] >> (16 * (k & 1))) & 0xffffu);
  }
}

// The CTA's unit in staging format Out (fp8_quant.cuh), the body of the unit kernels below
template <uint32_t DT, class Out>
__device__ __forceinline__ void quantise_unit(const SrcQUnit* __restrict__ units, uint32_t* s_amax, float* s_scale) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const SrcQUnit u = units[blockIdx.x];
  const char* src = reinterpret_cast<const char*>(u.src);
  const uint32_t cpr = (u.cols + 15u) / 16u, total = u.rows * cpr;
  const uint32_t ng = u.per_row ? u.rows : 1u;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  for (uint32_t g = threadIdx.x; g < ng; g += kQuantThreads) s_amax[g] = 0;
  // every load of this thread's chunks first: chunk j is idx = threadIdx.x + j * kQuantThreads
  uint32_t d[kSrcQChunks][4 * es];
#pragma unroll
  for (uint32_t j = 0; j < kSrcQChunks; ++j) {
    const uint32_t idx = threadIdx.x + j * kQuantThreads;
    const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
    if (idx < total) {
      load_chunk<DT>(src + static_cast<uint64_t>(r) * u.src_pitch + c * es, min(16u, u.cols - c), u.vec, d[j]);
    } else {
#pragma unroll
      for (uint32_t i = 0; i < 4 * es; ++i) d[j][i] = 0;  // folded as zeros by the warp's other lanes
    }
  }
  __syncthreads();  // the zeroed amax words are visible (the loads stay in flight)
  uint32_t mine = 0;
#pragma unroll
  for (uint32_t j = 0; j < kSrcQChunks; ++j) {
    const uint32_t base = warp * 32 + j * kQuantThreads;  // warp-uniform
    if (base >= total) break;
    const uint32_t idx = base + lane;
    uint32_t f[16], m = 0;
    widen_chunk<DT>(d[j], f);
#pragma unroll
    for (uint32_t k = 0; k < 16; ++k) m = max(m, abs_bits(f[k]));  // zero words past the chunk's end or the unit's
    if (u.per_row) {
      const uint32_t rf = base / cpr, rl = (min(base + 32u, total) - 1u) / cpr;
      if (rf == rl) {
        m = __reduce_max_sync(0xffffffffu, m);
        if (lane == 0) atomicMax(s_amax + rf, m);
      } else if (idx < total) {
        atomicMax(s_amax + idx / cpr, m);
      }
    } else {
      mine = max(mine, m);
    }
  }
  if (!u.per_row) {
    mine = __reduce_max_sync(0xffffffffu, mine);
    if (lane == 0) atomicMax(s_amax, mine);
  }
  __syncthreads();
  for (uint32_t g = threadIdx.x; g < ng; g += kQuantThreads) {
    float scale, scale_inv;
    Out::scales(s_amax[g], &scale, &scale_inv);
    s_scale[g] = scale;
    reinterpret_cast<float*>(u.scale_inv)[g] = scale_inv;
  }
  __syncthreads();
#pragma unroll
  for (uint32_t j = 0; j < kSrcQChunks; ++j) {
    const uint32_t idx = threadIdx.x + j * kQuantThreads;
    if (idx < total) {
      const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
      uint32_t f[16], o[4];
      widen_chunk<DT>(d[j], f);
      Out::narrow(f, s_scale[u.per_row ? r : 0u], o);
      store16(reinterpret_cast<char*>(u.dst) + static_cast<uint64_t>(r) * u.dst_pitch + c, min(16u, u.cols - c), o);
    }
  }
}

// float8_e4m3fn staging; kUe8m0: power-of-two scales (TSB_QUANT_UE8M0)
template <uint32_t DT, bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads) source_quant_kernel(const SrcQUnit* __restrict__ units) {
  __shared__ uint32_t s_amax[kSqBandRows];
  __shared__ float s_scale[kSqBandRows];
  quantise_unit<DT, E4m3Out<kUe8m0>>(units, s_amax, s_scale);
}

// int8 staging (TSB_I8).  Capped at the registers of its float8_e4m3fn twin: left alone, the int8 narrowing takes
// 64 on 2-byte sources against the twin's 62, with no spill either way.
template <uint32_t DT>
__global__ void __maxnreg__(Src<DT>::kBytes == 4 ? 95 : 62) source_int8_kernel(const SrcQUnit* __restrict__ units) {
  __shared__ uint32_t s_amax[kSqBandRows];
  __shared__ float s_scale[kSqBandRows];
  quantise_unit<DT, I8Out>(units, s_amax, s_scale);
}

// The staging format of `dst_dtype` in q->int8: TSB_ERR_INVALID unless TSB_F8E4M3 or TSB_I8, and for TSB_I8 with
// TSB_QUANT_UE8M0 (q->ue8m0)
int source_quant_dst(uint32_t dst_dtype, QuantPlan* q) {
  if (dst_dtype != TSB_F8E4M3 && dst_dtype != TSB_I8)
    return fail(TSB_ERR_INVALID, "source_quant: dst_dtype must be TSB_F8E4M3 or TSB_I8, not " + std::to_string(dst_dtype));
  q->int8 = dst_dtype == TSB_I8;
  if (q->int8 && q->ue8m0) return fail(TSB_ERR_INVALID, "source_quant: int8 staging takes float32 scales: TSB_QUANT_UE8M0 is refused");
  return TSB_OK;
}

// d = {SrcQUnit table | SqTile table | amax words}: one launch per source dtype over its units, one CTA each, then
// scaled_fp8.cu's two passes over the tiles.  The tables do not depend on dst_dtype.
int source_quant_plan(const tsb_source_quant_target_t* targets, uint64_t n, uint32_t dst_dtype, QuantPlan* q) {
  SrcQTables tb;
  int st = source_quant_dst(dst_dtype, q);
  if (st || (st = source_quant_compile(targets, n, &tb))) return st;
  q->add(tb.units);
  const size_t tiles = q->add(tb.tiles), amax = q->seal(tb.n_groups);
  q->describe(n, static_cast<uint32_t>(tb.units.size() + tb.tiles.size()), tb.unit_bytes, tb);
  const SqLaunch two_pass{nullptr, nullptr, nullptr, nullptr, 0, static_cast<uint32_t>(tb.tiles.size()), tb.n_groups, 0, q->ue8m0,
                          q->int8};
  // the unit kernels by rank (bf16, f16, f32) and staging format
  using Kernel = void (*)(const SrcQUnit*);
  const std::array<Kernel, 3> kernels =
      q->int8    ? std::array<Kernel, 3>{source_int8_kernel<TSB_BF16>, source_int8_kernel<TSB_F16>, source_int8_kernel<TSB_F32>}
      : q->ue8m0 ? std::array<Kernel, 3>{source_quant_kernel<TSB_BF16, true>, source_quant_kernel<TSB_F16, true>,
                                         source_quant_kernel<TSB_F32, true>}
                 : std::array<Kernel, 3>{source_quant_kernel<TSB_BF16, false>, source_quant_kernel<TSB_F16, false>,
                                         source_quant_kernel<TSB_F32, false>};
  q->launch = [two_pass, tiles, amax, kernels, int8 = q->int8, n_units = std::array<uint32_t, 3>{tb.n_units[0], tb.n_units[1], tb.n_units[2]}](char* d, cudaStream_t s) -> int {
    const SrcQUnit* units = reinterpret_cast<const SrcQUnit*>(d);
    for (int k = 0; k < 3; ++k) {
      const uint32_t n = n_units[k];
      if (!n) continue;
      kernels[k]<<<n, kQuantThreads, 0, s>>>(units);
      if (int st = launched(int8 ? "source_int8_kernel launch" : "source_quant_kernel launch")) return st;
      units += n;
    }
    if (!two_pass.n_tiles) return TSB_OK;
    SqLaunch l = two_pass;
    l.tiles = reinterpret_cast<const SqTile*>(d + tiles);
    l.amax = reinterpret_cast<uint32_t*>(d + amax);
    return launch_scaled_fp8(l, s);
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_source_quant_plan_create_as(int device, const tsb_source_quant_target_t* targets, uint64_t n,
                                               uint32_t dst_dtype, uint32_t flags, tsb_plan_t* out) {
  return quant_plan_create("tsb_source_quant_plan_create", device, flags, TSB_QUANT_UE8M0, out,
                           [&](QuantPlan* q) { return source_quant_plan(targets, n, dst_dtype, q); });
}

extern "C" int tsb_source_quant_compile_host_as(int device, const tsb_source_quant_target_t* targets, uint64_t n,
                                                uint32_t dst_dtype, uint32_t flags, void* out_units, uint64_t unit_cap,
                                                uint64_t* out_n_units, void* out_tiles, uint64_t tile_cap,
                                                uint64_t* out_n_tiles, uint64_t* out_n_groups) {
  (void)device;
  return quant_compile_host("tsb_source_quant_compile_host", flags, TSB_QUANT_UE8M0,
                            [&](QuantPlan* q) { return source_quant_plan(targets, n, dst_dtype, q); },
                            {{out_units, unit_cap, out_n_units, "out_units"}, {out_tiles, tile_cap, out_n_tiles, "out_tiles"}},
                            out_n_groups);
}

extern "C" int tsb_source_quant_plan_create(int device, const tsb_source_quant_target_t* targets, uint64_t n, uint32_t flags,
                                            tsb_plan_t* out) {
  return tsb_source_quant_plan_create_as(device, targets, n, TSB_F8E4M3, flags, out);
}

extern "C" int tsb_source_quant_compile_host(int device, const tsb_source_quant_target_t* targets, uint64_t n, uint32_t flags,
                                             void* out_units, uint64_t unit_cap, uint64_t* out_n_units, void* out_tiles,
                                             uint64_t tile_cap, uint64_t* out_n_tiles, uint64_t* out_n_groups) {
  return tsb_source_quant_compile_host_as(device, targets, n, TSB_F8E4M3, flags, out_units, unit_cap, out_n_units, out_tiles,
                                          tile_cap, out_n_tiles, out_n_groups);
}
