// copy_rects: the reshard kernel of libtstore_b200 (sm_90a, H100).
//
// One persistent launch moves every rectangle of a compiled plan: local-shard slice -> (peer or
// local) gather into the destination shard, with the optional dtype cast fused into the store.
// It replaces, in the reference,
//   * asyncio.gather(rdma_buffer.read_into(...))          direct_weight_sync.py:338-340
//   * dest[dest_slices].copy_(recv[src_slices])            direct_weight_sync.py:343-350
//   * client_tensor.copy_(shm_tensor) / shm.copy_(tensor)  transport/shared_memory.py:374,475
//   * local.to(transfer_dtype) / staging.copy_(src)        direct_weight_sync.py:133,167-168
//
// Work decomposition (built on the host by plan.cu):
//   rect  -> rows x units   (unit = 16 B for byte moves, 8 elements for vector casts)
//   tile  = <= tile_units units: either a segment of one wide row or a group of whole narrow rows
//   tiles are listed in an order that round-robins over source GPUs (NVSwitch port fairness)
//   CTA b processes tiles b, b+grid, b+2*grid, ...; the next tile's rect header is staged into
//   shared memory with cp.async while the current tile is being moved, so the index math never
//   waits on HBM.
// Data path of the 8 copy warps: LDG.128 (non-coherent, no L1 allocate), UNROLL independent loads
// in flight per thread, then coalesced STG.128.
// Data path of the link warp (9th warp, only launched when the plan has NVLink sources): a ring of
// TMA bulk copies, peer global -> shared (cp.async.bulk + mbarrier complete_tx) -> local global
// (cp.async.bulk.global.shared), rows issued in parallel by the 32 lanes.  The 1-2 us NVLink round
// trip is covered by bytes parked in shared memory instead of registers of stalled copy warps, so
// the local HBM copies of the same launch run at full rate beside the link traffic.

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <atomic>

#include "tsb_internal.h"

namespace tsb {

namespace {

constexpr int kThreads = kCopyThreads;

__device__ __forceinline__ uint4 ldg16(const char* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void stg16(char* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

// ---- movers: how one unit travels from src to dst ---------------------------------------------
template <int U>
struct MoveB16T {
  static constexpr int kUnroll = U;
  using Reg = uint4;
  static __device__ __forceinline__ Reg ld(const char* p) { return ldg16(p); }
  static __device__ __forceinline__ void st(char* p, const Reg& v) { stg16(p, v); }
};
using MoveB16 = MoveB16T<4>;
template <typename T>
struct MoveSmall {
  static constexpr int kUnroll = 4;
  using Reg = T;
  static __device__ __forceinline__ Reg ld(const char* p) { return __ldg(reinterpret_cast<const T*>(p)); }
  static __device__ __forceinline__ void st(char* p, const Reg& v) { *reinterpret_cast<T*>(p) = v; }
};

// scalar conversions, all round-to-nearest-even like torch's .to()
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

template <typename S, typename D>
struct CastScalar {
  static constexpr int kUnroll = 4;
  using Reg = S;
  static __device__ __forceinline__ Reg ld(const char* p) { return *reinterpret_cast<const S*>(p); }
  static __device__ __forceinline__ void st(char* p, const Reg& v) { *reinterpret_cast<D*>(p) = convert<S, D>(v); }
};

// 8 elements per unit; 4-byte -> 2-byte (32 B in, 16 B out)
template <typename D>
struct CastNarrowV8 {
  static constexpr int kUnroll = 2;
  struct Reg { uint4 a, b; };
  static __device__ __forceinline__ Reg ld(const char* p) { return Reg{ldg16(p), ldg16(p + 16)}; }
  static __device__ __forceinline__ uint32_t pack(uint32_t lo, uint32_t hi) {
    D l = convert<float, D>(__uint_as_float(lo));
    D h = convert<float, D>(__uint_as_float(hi));
    return static_cast<uint32_t>(*reinterpret_cast<unsigned short*>(&l)) |
           (static_cast<uint32_t>(*reinterpret_cast<unsigned short*>(&h)) << 16);
  }
  static __device__ __forceinline__ void st(char* p, const Reg& v) {
    uint4 o;
    o.x = pack(v.a.x, v.a.y);
    o.y = pack(v.a.z, v.a.w);
    o.z = pack(v.b.x, v.b.y);
    o.w = pack(v.b.z, v.b.w);
    stg16(p, o);
  }
};
// 8 elements per unit; 2-byte -> 4-byte (16 B in, 32 B out)
template <typename S>
struct CastWidenV8 {
  static constexpr int kUnroll = 4;
  using Reg = uint4;
  static __device__ __forceinline__ Reg ld(const char* p) { return ldg16(p); }
  static __device__ __forceinline__ uint32_t up(uint32_t bits16) {
    unsigned short b = static_cast<unsigned short>(bits16);
    S s = *reinterpret_cast<S*>(&b);
    return __float_as_uint(convert<S, float>(s));
  }
  static __device__ __forceinline__ void st(char* p, const Reg& v) {
    uint4 lo, hi;
    lo.x = up(v.x & 0xffffu); lo.y = up(v.x >> 16); lo.z = up(v.y & 0xffffu); lo.w = up(v.y >> 16);
    hi.x = up(v.z & 0xffffu); hi.y = up(v.z >> 16); hi.z = up(v.w & 0xffffu); hi.w = up(v.w >> 16);
    stg16(p, lo);
    stg16(p + 16, hi);
  }
};
// 8 elements per unit; 2-byte -> 2-byte (bf16 <-> f16)
template <typename S, typename D>
struct CastHalfV8 {
  static constexpr int kUnroll = 4;
  using Reg = uint4;
  static __device__ __forceinline__ Reg ld(const char* p) { return ldg16(p); }
  static __device__ __forceinline__ uint32_t cv(uint32_t w) {
    unsigned short b0 = static_cast<unsigned short>(w & 0xffffu), b1 = static_cast<unsigned short>(w >> 16);
    D d0 = convert<S, D>(*reinterpret_cast<S*>(&b0));
    D d1 = convert<S, D>(*reinterpret_cast<S*>(&b1));
    return static_cast<uint32_t>(*reinterpret_cast<unsigned short*>(&d0)) |
           (static_cast<uint32_t>(*reinterpret_cast<unsigned short*>(&d1)) << 16);
  }
  static __device__ __forceinline__ void st(char* p, const Reg& v) {
    uint4 o{cv(v.x), cv(v.y), cv(v.z), cv(v.w)};
    stg16(p, o);
  }
};

// ---- index math --------------------------------------------------------------------------------
__device__ __forceinline__ void row_offsets(const DevRect& r, uint32_t row, int64_t& so, int64_t& dof) {
  const uint32_t n = r.n_outer;
  if (n <= 1) {  // n == 0: rows == 1, row == 0
    so = n ? static_cast<int64_t>(row) * r.src_stride[0] : 0;
    dof = n ? static_cast<int64_t>(row) * r.dst_stride[0] : 0;
    return;
  }
  so = 0;
  dof = 0;
  for (int d = static_cast<int>(n) - 1; d >= 1; --d) {
    const uint32_t e = r.ext[d];
    const uint32_t q = row / e;
    const uint32_t rem = row - q * e;
    so += static_cast<int64_t>(rem) * r.src_stride[d];
    dof += static_cast<int64_t>(rem) * r.dst_stride[d];
    row = q;
  }
  so += static_cast<int64_t>(row) * r.src_stride[0];
  dof += static_cast<int64_t>(row) * r.dst_stride[0];
}

// A segment of a single (wide) row: pure streaming copy, no per-unit index math.
template <typename M>
__device__ __forceinline__ void move_wide(const DevRect& r, uint32_t tile_in_rect, uint32_t tile_units) {
  constexpr int U = M::kUnroll;
  const uint32_t sub = r.src_unit_bytes, dub = r.dst_unit_bytes;
  const uint32_t row = tile_in_rect / r.split;
  const uint32_t seg = tile_in_rect - row * r.split;
  const uint32_t ustart = seg * tile_units;
  const uint32_t ucount = min(tile_units, r.units_per_row - ustart);
  int64_t so, dof;
  row_offsets(r, row, so, dof);
  const char* __restrict__ src = reinterpret_cast<const char*>(r.src) + so + static_cast<int64_t>(ustart) * sub;
  char* __restrict__ dst = reinterpret_cast<char*>(r.dst) + dof + static_cast<int64_t>(ustart) * dub;
  for (uint32_t i = threadIdx.x; i < ucount; i += kThreads * U) {
    typename M::Reg v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const uint32_t idx = i + k * kThreads;
      if (idx < ucount) v[k] = M::ld(src + static_cast<size_t>(idx) * sub);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const uint32_t idx = i + k * kThreads;
      if (idx < ucount) M::st(dst + static_cast<size_t>(idx) * dub, v[k]);
    }
  }
}

// A group of whole narrow rows of a 2-D rect (one outer dim): unit index -> (row, col) with a
// multiply-high instead of a divide.  This is the FSDP->TP hot case (1 KiB .. 28 KiB rows).
template <typename M>
__device__ __forceinline__ void move_narrow(const DevRect& r, uint32_t tile_in_rect) {
  constexpr int U = M::kUnroll;
  const uint32_t sub = r.src_unit_bytes, dub = r.dst_unit_bytes;
  const uint32_t upr = r.units_per_row;
  const uint32_t magic = r.magic;
  const uint32_t row0 = tile_in_rect * r.split;
  const uint32_t nrows = min(r.split, r.rows - row0);
  const uint32_t total = nrows * upr;
  const int64_t ss0 = r.n_outer ? r.src_stride[0] : 0;
  const int64_t ds0 = r.n_outer ? r.dst_stride[0] : 0;
  const char* __restrict__ src = reinterpret_cast<const char*>(r.src) + static_cast<int64_t>(row0) * ss0;
  char* __restrict__ dst = reinterpret_cast<char*>(r.dst) + static_cast<int64_t>(row0) * ds0;
  for (uint32_t i = threadIdx.x; i < total; i += kThreads * U) {
    typename M::Reg v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const uint32_t idx = i + k * kThreads;
      if (idx < total) {
        const uint32_t rr = magic ? __umulhi(idx, magic) : idx;
        const uint32_t c = idx - rr * upr;
        v[k] = M::ld(src + static_cast<int64_t>(rr) * ss0 + static_cast<int64_t>(c) * sub);
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const uint32_t idx = i + k * kThreads;
      if (idx < total) {
        const uint32_t rr = magic ? __umulhi(idx, magic) : idx;
        const uint32_t c = idx - rr * upr;
        M::st(dst + static_cast<int64_t>(rr) * ds0 + static_cast<int64_t>(c) * dub, v[k]);
      }
    }
  }
}

// General N-D narrow rows (3 or more collapsed dims): rare, kept simple.
template <typename M>
__device__ __noinline__ void move_narrow_nd(const DevRect& r, uint32_t tile_in_rect) {
  const uint32_t sub = r.src_unit_bytes, dub = r.dst_unit_bytes;
  const uint32_t upr = r.units_per_row;
  const uint32_t magic = r.magic;
  const uint32_t row0 = tile_in_rect * r.split;
  const uint32_t nrows = min(r.split, r.rows - row0);
  const uint32_t total = nrows * upr;
  const char* __restrict__ src = reinterpret_cast<const char*>(r.src);
  char* __restrict__ dst = reinterpret_cast<char*>(r.dst);
  for (uint32_t idx = threadIdx.x; idx < total; idx += kThreads) {
    const uint32_t rr = magic ? __umulhi(idx, magic) : idx;
    const uint32_t c = idx - rr * upr;
    int64_t so, dof;
    row_offsets(r, row0 + rr, so, dof);
    typename M::Reg v = M::ld(src + so + static_cast<int64_t>(c) * sub);
    M::st(dst + dof + static_cast<int64_t>(c) * dub, v);
  }
}

// Out-of-line wrappers for the generic (mixed-mode) kernel: one ABI call per tile keeps the
// 60-odd instantiations from sharing one register allocation.
template <typename M>
__device__ __noinline__ void move_wide_ool(const DevRect& r, uint32_t t, uint32_t tile_units) { move_wide<M>(r, t, tile_units); }
template <typename M>
__device__ __noinline__ void move_narrow_ool(const DevRect& r, uint32_t t) { move_narrow<M>(r, t); }

template <typename M, bool kInline>
__device__ __forceinline__ void move_tile(const DevRect& r, uint32_t tile_in_rect, uint32_t tile_units) {
  if (r.wide) {
    if (kInline) move_wide<M>(r, tile_in_rect, tile_units);
    else move_wide_ool<M>(r, tile_in_rect, tile_units);
  } else if (r.n_outer <= 1) {
    if (kInline) move_narrow<M>(r, tile_in_rect);
    else move_narrow_ool<M>(r, tile_in_rect);
  } else {
    move_narrow_nd<M>(r, tile_in_rect);
  }
}

// KIND selects a kernel specialisation chosen by the plan compiler:
//   KIND_GENERIC  any mix of modes (per-tile dispatch, out-of-line movers)
//   KIND_B16      every rect moves 16-byte units: the weight-sync case, fully inlined
//   KIND_F32_BF16 every rect is the vector fp32->bf16 cast (transfer_dtype=bf16), fully inlined
template <int KIND>
__device__ __forceinline__ void process_tile(const DevRect& r, uint32_t tile_in_rect) {
  const uint32_t tile_units = r.tile_units;
  if (KIND == KIND_B16) {
    move_tile<MoveB16, true>(r, tile_in_rect, tile_units);
    return;
  }
  if (KIND == KIND_F32_BF16) {
    move_tile<CastNarrowV8<__nv_bfloat16>, true>(r, tile_in_rect, tile_units);
    return;
  }
  switch (r.mode) {
    case MODE_B16: move_tile<MoveB16, false>(r, tile_in_rect, tile_units); break;
    case MODE_B8: move_tile<MoveSmall<uint2>, false>(r, tile_in_rect, tile_units); break;
    case MODE_B4: move_tile<MoveSmall<uint32_t>, false>(r, tile_in_rect, tile_units); break;
    case MODE_B2: move_tile<MoveSmall<uint16_t>, false>(r, tile_in_rect, tile_units); break;
    case MODE_B1: move_tile<MoveSmall<uint8_t>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F32_BF16_V8: move_tile<CastNarrowV8<__nv_bfloat16>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F32_BF16_S: move_tile<CastScalar<float, __nv_bfloat16>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F32_F16_V8: move_tile<CastNarrowV8<__half>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F32_F16_S: move_tile<CastScalar<float, __half>, false>(r, tile_in_rect, tile_units); break;
    case MODE_BF16_F32_V8: move_tile<CastWidenV8<__nv_bfloat16>, false>(r, tile_in_rect, tile_units); break;
    case MODE_BF16_F32_S: move_tile<CastScalar<__nv_bfloat16, float>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F16_F32_V8: move_tile<CastWidenV8<__half>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F16_F32_S: move_tile<CastScalar<__half, float>, false>(r, tile_in_rect, tile_units); break;
    case MODE_BF16_F16_V8: move_tile<CastHalfV8<__nv_bfloat16, __half>, false>(r, tile_in_rect, tile_units); break;
    case MODE_BF16_F16_S: move_tile<CastScalar<__nv_bfloat16, __half>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F16_BF16_V8: move_tile<CastHalfV8<__half, __nv_bfloat16>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F16_BF16_S: move_tile<CastScalar<__half, __nv_bfloat16>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F64_F32_S: move_tile<CastScalar<double, float>, false>(r, tile_in_rect, tile_units); break;
    case MODE_F32_F64_S: move_tile<CastScalar<float, double>, false>(r, tile_in_rect, tile_units); break;
    default: break;
  }
}

// Stage one DevRect (global -> shared) with 16-byte cp.async issued by the first few lanes.
__device__ __forceinline__ void stage_rect(DevRect* sdst, const DevRect* gsrc) {
  constexpr uint32_t kChunks = sizeof(DevRect) / 16;
  if (threadIdx.x < kChunks) {
    const uint32_t saddr = static_cast<uint32_t>(__cvta_generic_to_shared(reinterpret_cast<char*>(sdst) + threadIdx.x * 16));
    const char* g = reinterpret_cast<const char*>(gsrc) + threadIdx.x * 16;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
  }
}
__device__ __forceinline__ void stage_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// barrier of the 8 copy warps only (the link warp never joins it)
__device__ __forceinline__ void copy_warps_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kCopyThreads) : "memory"); }

// ---- link warp: TMA bulk ring over NVLink ----------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }

constexpr uint32_t kMaxLinkStages = 8;

struct alignas(16) LinkMeta {  // what the store half needs to know about the chunk parked in a stage
  uint64_t dst;
  int64_t dst_stride;  // bytes between rows in the destination
  uint32_t nrows;
  uint32_t row_bytes;
};

// One chunk == one link tile == at most one ring stage: a segment of a wide row, or a group of whole
// narrow rows packed back to back in shared memory.  Loads run S-2 stages ahead of stores; the stage
// about to be refilled was stored two commits ago, so wait_group.read 1 frees it.
__device__ __forceinline__ void link_warp_run(const LaunchParams& p, unsigned char* ring, uint64_t* bars, LinkMeta* meta) {
  const uint32_t lane = threadIdx.x - kCopyThreads;
  const uint32_t S = p.link_stages, SB = p.link_stage_bytes, n = p.num_link_tiles;
  const uint32_t lag = S - 2;
  if (lane == 0) {
    for (uint32_t s = 0; s < S; ++s) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();
  uint32_t issued = 0, stored = 0, phase_bits = 0;

  auto store_one = [&]() {
    const uint32_t s = stored % S;
    mbar_wait(&bars[s], (phase_bits >> s) & 1u);
    phase_bits ^= 1u << s;
    const LinkMeta m = meta[s];
    unsigned char* stage = ring + s * SB;
    if (m.nrows == 1 || m.dst_stride == static_cast<int64_t>(m.row_bytes)) {
      if (lane == 0) bulk_s2g(reinterpret_cast<void*>(m.dst), stage, m.nrows * m.row_bytes);
    } else {
      for (uint32_t j = lane; j < m.nrows; j += kLinkThreads)
        bulk_s2g(reinterpret_cast<char*>(m.dst) + static_cast<int64_t>(j) * m.dst_stride, stage + j * m.row_bytes, m.row_bytes);
    }
    bulk_commit();
    ++stored;
  };

  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(p.sched + 2, kLinkBatch);
  base = __shfl_sync(0xffffffffu, base, 0);
  while (base < n) {
    uint32_t next_base = 0;
    if (lane == 0) next_base = atomicAdd(p.sched + 2, kLinkBatch);  // consumed after this batch: latency hidden
    const uint32_t cnt = min(kLinkBatch, n - base);
    DevTile mine{0u, 0u};
    if (lane < cnt) mine = p.link_tiles[base + lane];
    for (uint32_t i = 0; i < cnt; ++i) {
      const uint32_t rect_id = __shfl_sync(0xffffffffu, mine.rect, i);
      const uint32_t tir = __shfl_sync(0xffffffffu, mine.tile_in_rect, i);
      const DevRect& r = p.rects[rect_id];
      const uint32_t s = issued % S;
      if (issued >= S) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      __syncwarp();
      int64_t so = 0, dof = 0, ss = 0, ds = 0;
      uint32_t nrows, row_bytes;
      if (r.wide) {
        const uint32_t row = tir / r.split;
        const uint32_t seg = tir - row * r.split;
        const uint32_t ustart = seg * r.tile_units;
        row_offsets(r, row, so, dof);
        so += static_cast<int64_t>(ustart) * 16;
        dof += static_cast<int64_t>(ustart) * 16;
        nrows = 1;
        row_bytes = min(r.tile_units, r.units_per_row - ustart) * 16u;
      } else {  // n_outer <= 1 by construction (plan.cu keeps N-D narrow rects in the copy queue)
        const uint32_t row0 = tir * r.split;
        ss = r.n_outer ? r.src_stride[0] : 0;
        ds = r.n_outer ? r.dst_stride[0] : 0;
        so = static_cast<int64_t>(row0) * ss;
        dof = static_cast<int64_t>(row0) * ds;
        nrows = min(r.split, r.rows - row0);
        row_bytes = r.units_per_row * 16u;
      }
      if (lane == 0) {
        meta[s] = LinkMeta{r.dst + static_cast<uint64_t>(dof), ds, nrows, row_bytes};
        mbar_expect_tx(&bars[s], nrows * row_bytes);
      }
      const char* src = reinterpret_cast<const char*>(r.src) + so;
      unsigned char* stage = ring + s * SB;
      for (uint32_t j = lane; j < nrows; j += kLinkThreads)
        bulk_g2s(stage + j * row_bytes, src + static_cast<int64_t>(j) * ss, row_bytes, &bars[s]);
      ++issued;
      __syncwarp();
      if (issued - stored > lag) store_one();
    }
    base = __shfl_sync(0xffffffffu, next_base, 0);
  }
  while (stored < issued) store_one();
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Tile scheduling of the copy queue.  Every CTA owns the first three tiles of its column statically
// (b, b+grid, b+2*grid: their headers can be prefetched at once); after that tiles are claimed
// from a global atomic counter, so CTAs that happened to draw slow tiles (short remainders, peer
// destinations) simply claim fewer -- no tail imbalance when tile costs are heterogeneous.  The
// claim for tile k+3 is issued before tile k's payload moves and only consumed after it, so the
// atomic's round trip is never exposed.  The claimed index is broadcast through a slot that is
// double-buffered by iteration parity (a warp still reading iteration k's slot cannot see the write
// of iteration k+1).  The last CTA to finish resets the counters, which keeps a sync at one kernel
// launch (a plan must not run concurrently with itself).
template <int KIND>
__global__ void __launch_bounds__(kCopyThreads + kLinkThreads, 3) copy_rects_kernel(LaunchParams p) {
  extern __shared__ __align__(128) unsigned char link_ring[];
  __shared__ DevRect srect[2];
  __shared__ uint32_t s_claim[2];
  __shared__ uint64_t link_bars[kMaxLinkStages];
  __shared__ LinkMeta link_meta[kMaxLinkStages];
  const uint32_t grid = gridDim.x;
  const uint32_t n = p.num_tiles;
  const bool dynamic = p.sched != nullptr;
  if (threadIdx.x >= kCopyThreads) {
    link_warp_run(p, link_ring, link_bars, link_meta);
  } else {
    uint32_t i0 = blockIdx.x;          // index (into p.tiles) of the current tile
    uint32_t i1 = i0 + grid;           // next
    uint32_t i2 = i1 + grid;           // the one after
    if (i0 < n) {
      DevTile cur = p.tiles[i0];
      DevTile nxt = cur;
      if (i1 < n) nxt = p.tiles[i1];
      stage_rect(&srect[0], &p.rects[cur.rect]);
      stage_wait();
      copy_warps_sync();

      int buf = 0;
      while (true) {
        const bool has_next = i1 < n;
        DevTile nn = nxt;
        uint32_t claimed = i2 + grid;  // static fallback: keep striding
        if (has_next) {
          // header pipeline: rect of tile k+1 -> smem, tile entry k+2 -> registers, claim of tile
          // k+3 -> in flight, all while tile k's payload moves
          stage_rect(&srect[buf ^ 1], &p.rects[nxt.rect]);
          if (i2 < n) nn = p.tiles[i2];
          if (dynamic && threadIdx.x == 0) claimed = atomicAdd(p.sched, 1u) + 3u * grid;
        }
        process_tile<KIND>(srect[buf], cur.tile_in_rect);
        if (!has_next) break;
        if (dynamic && threadIdx.x == 0) s_claim[buf] = claimed;
        stage_wait();
        copy_warps_sync();
        if (dynamic) claimed = s_claim[buf];  // this iteration's slot; the other one takes the next write
        cur = nxt;
        nxt = nn;
        i1 = i2;
        i2 = claimed;
        buf ^= 1;
      }
    }
  }
  if (dynamic) {
    __syncthreads();  // copy warps and link warp of this CTA are both done
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(p.sched + 1, 1u) == grid - 1) {  // last CTA out: re-arm for the next launch
        p.sched[0] = 0;
        p.sched[1] = 0;
        p.sched[2] = 0;
        __threadfence();
      }
    }
  }
}

std::atomic<uint64_t> g_launches{0};

template <int KIND>
cudaError_t prepare_kernel() {
  // the link ring plus the static tables exceed the 48 KiB default shared memory limit; function
  // attributes are per device (context), so set it once on every device the kernel runs on
  static std::atomic<uint64_t> prepared{0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const uint64_t bit = 1ull << (dev & 63);
  if (prepared.load(std::memory_order_acquire) & bit) return cudaSuccess;
  e = cudaFuncSetAttribute(copy_rects_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           static_cast<int>(kMaxLinkStages * 16384));
  if (e == cudaSuccess) prepared.fetch_or(bit, std::memory_order_release);
  return e;
}

template <int KIND>
cudaError_t occupancy(bool with_link, uint32_t smem, int* n) {
  cudaError_t e = prepare_kernel<KIND>();
  if (e != cudaSuccess) return e;
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(n, copy_rects_kernel<KIND>,
                                                       static_cast<int>(kCopyThreads + (with_link ? kLinkThreads : 0u)), smem);
}

template <int KIND>
cudaError_t launch(const LaunchParams& p, uint32_t grid, cudaStream_t stream) {
  cudaError_t e = prepare_kernel<KIND>();
  if (e != cudaSuccess) return e;
  const bool with_link = p.num_link_tiles != 0;
  const uint32_t block = kCopyThreads + (with_link ? kLinkThreads : 0u);
  const size_t smem = with_link ? static_cast<size_t>(p.link_stages) * p.link_stage_bytes : 0;
  copy_rects_kernel<KIND><<<grid, block, smem, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int max_ctas_per_sm(uint32_t kind, bool with_link, uint32_t link_smem_bytes, int* out) {
  int n = 0;
  cudaError_t e;
  const uint32_t smem = with_link ? link_smem_bytes : 0u;
  switch (kind) {
    case KIND_B16: e = occupancy<KIND_B16>(with_link, smem, &n); break;
    case KIND_F32_BF16: e = occupancy<KIND_F32_BF16>(with_link, smem, &n); break;
    default: e = occupancy<KIND_GENERIC>(with_link, smem, &n); break;
  }
  if (e != cudaSuccess) return cuda_fail(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
  *out = n;
  return TSB_OK;
}

int launch_copy_rects(const LaunchParams& p, uint32_t grid, cudaStream_t stream) {
  if (p.num_tiles == 0 && p.num_link_tiles == 0) return TSB_OK;
  if (p.num_link_tiles != 0) {
    if (p.sched == nullptr) return fail(TSB_ERR_INVALID, "copy_rects: the link queue needs the dynamic scheduler");
    if (p.link_stages < 3 || p.link_stages > kMaxLinkStages || p.link_stage_bytes < 1024 || p.link_stage_bytes > 16384 ||
        p.link_stage_bytes % 16)
      return fail(TSB_ERR_INVALID, "copy_rects: bad link ring geometry");
  }
  cudaError_t e;
  switch (p.kind) {
    case KIND_B16: e = launch<KIND_B16>(p, grid, stream); break;
    case KIND_F32_BF16: e = launch<KIND_F32_BF16>(p, grid, stream); break;
    default: e = launch<KIND_GENERIC>(p, grid, stream); break;
  }
  if (e != cudaSuccess) return cuda_fail(e, "copy_rects_kernel launch");
  count_launch();
  return TSB_OK;
}

}  // namespace tsb

extern "C" uint64_t tsb_launch_count(void) { return tsb::g_launches.load(std::memory_order_relaxed); }
