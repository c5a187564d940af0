// Plan compiler: turns a list of tsb_rect_t (N-D rectangles, element extents, byte strides) into
// the device-resident tables the copy_rects kernel walks: one DevRect per (possibly split)
// rectangle and one DevTile per <= tile_units units of work, ordered so that consecutive tiles
// pull from different source GPUs.
//
// This is the native counterpart of DirectWeightSyncDest._build_plan's cached op list
// (reference direct_weight_sync.py:221-317,334-335) and of the per-sub-request copy loop of
// the store path (transport/shared_memory.py:438-480): built once, replayed every sync.

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "tsb_internal.h"

namespace tsb {

namespace {

// Device tables of one plan live in ONE allocation: {sched[4] | rects | copy tiles | link tiles}.
constexpr size_t kSchedBytes = 256;  // 4 counters, padded so the rect table stays 256-byte aligned

struct TableLayout {
  size_t rects_off = 0, tiles_off = 0, link_off = 0, total = 0;
};

TableLayout table_layout(size_t n_rects, size_t n_tiles, size_t n_link) {
  TableLayout l;
  l.rects_off = kSchedBytes;
  l.tiles_off = l.rects_off + n_rects * sizeof(DevRect);
  l.link_off = l.tiles_off + n_tiles * sizeof(DevTile);
  l.total = l.link_off + n_link * sizeof(DevTile);
  if (l.total < kSchedBytes + 16) l.total = kSchedBytes + 16;
  return l;
}

struct Plan {
  int device = 0;
  char* d_block = nullptr;
  TableLayout layout;
  uint32_t num_tiles = 0;
  uint32_t num_link_tiles = 0;
  uint32_t kind = KIND_GENERIC;
  // scaled fp8 plans: runs them from d_block (QuantPlan::launch); empty for copy plans, which d_block's
  // {sched | rects | copy tiles | link tiles} drive through the copy_rects kernel
  std::function<int(char*, cudaStream_t)> quant;
  uint32_t link_stage_bytes = 0;
  uint32_t link_stages = 0;
  tsb_plan_info_t info{};
  // fenced launches (tsb_plan_launch): created on first use, reused every sync
  cudaEvent_t ev_fence = nullptr, ev_start = nullptr, ev_done = nullptr;
  bool launched = false;
};

// Recycled {pinned host, device} table buffers for one-shot copies (tsb_copy_rects): the tables
// are uploaded with cudaMemcpyAsync on the SAME stream as the kernel, so ordering is by stream and
// no cudaMalloc/cudaFree (= device-wide sync) happens per call once the pool is warm.
struct PoolBlock {
  int device = 0;
  char* d = nullptr;
  char* h = nullptr;
  size_t cap = 0;
  cudaEvent_t done = nullptr;
  bool in_flight = false;
};

struct PlanRegistry {
  std::mutex mu;
  std::unordered_map<uint64_t, Plan*> plans;
  std::vector<PoolBlock*> pool;
  uint64_t next_id = 1;
  uint64_t pool_allocs = 0, pool_reuses = 0;
};

PlanRegistry& R() {
  static PlanRegistry r;
  return r;
}

uint32_t dtype_size(uint32_t dt) {
  switch (dt) {
    case TSB_U8: case TSB_F8E4M3: case TSB_F8E5M2: return 1;
    case TSB_U16: case TSB_F16: case TSB_BF16: return 2;
    case TSB_U32: case TSB_F32: return 4;
    case TSB_U64: case TSB_F64: return 8;
    default: return 0;
  }
}

// (vector mode, scalar mode, elements per vector unit) for a cross-dtype pair, or false
bool cast_modes(uint32_t s, uint32_t d, uint32_t* vmode, uint32_t* smode, uint32_t* velems = nullptr) {
  struct Row { uint32_t s, d, v, sc, ve; };
  static const Row table[] = {
      {TSB_F32, TSB_BF16, MODE_F32_BF16_V8, MODE_F32_BF16_S, 8},         {TSB_F32, TSB_F16, MODE_F32_F16_V8, MODE_F32_F16_S, 8},
      {TSB_BF16, TSB_F32, MODE_BF16_F32_V8, MODE_BF16_F32_S, 8},         {TSB_F16, TSB_F32, MODE_F16_F32_V8, MODE_F16_F32_S, 8},
      {TSB_BF16, TSB_F16, MODE_BF16_F16_V8, MODE_BF16_F16_S, 8},         {TSB_F16, TSB_BF16, MODE_F16_BF16_V8, MODE_F16_BF16_S, 8},
      {TSB_F64, TSB_F32, 0xffffffffu, MODE_F64_F32_S, 0},                {TSB_F32, TSB_F64, 0xffffffffu, MODE_F32_F64_S, 0},
      {TSB_F32, TSB_F8E4M3, MODE_F32_E4M3_V16, MODE_F32_E4M3_S, 16},     {TSB_F32, TSB_F8E5M2, MODE_F32_E5M2_V16, MODE_F32_E5M2_S, 16},
      {TSB_BF16, TSB_F8E4M3, MODE_BF16_E4M3_V16, MODE_BF16_E4M3_S, 16},  {TSB_BF16, TSB_F8E5M2, MODE_BF16_E5M2_V16, MODE_BF16_E5M2_S, 16},
      {TSB_F16, TSB_F8E4M3, MODE_F16_E4M3_V16, MODE_F16_E4M3_S, 16},     {TSB_F16, TSB_F8E5M2, MODE_F16_E5M2_V16, MODE_F16_E5M2_S, 16},
      {TSB_F8E4M3, TSB_F32, MODE_E4M3_F32_V16, MODE_E4M3_F32_S, 16},     {TSB_F8E5M2, TSB_F32, MODE_E5M2_F32_V16, MODE_E5M2_F32_S, 16},
      {TSB_F8E4M3, TSB_BF16, MODE_E4M3_BF16_V16, MODE_E4M3_BF16_S, 16},  {TSB_F8E5M2, TSB_BF16, MODE_E5M2_BF16_V16, MODE_E5M2_BF16_S, 16},
      {TSB_F8E4M3, TSB_F16, MODE_E4M3_F16_V16, MODE_E4M3_F16_S, 16},     {TSB_F8E5M2, TSB_F16, MODE_E5M2_F16_V16, MODE_E5M2_F16_S, 16},
  };
  for (const Row& r : table)
    if (r.s == s && r.d == d) {
      *vmode = r.v;
      *smode = r.sc;
      if (velems) *velems = r.ve;
      return true;
    }
  return false;
}

struct Dim {
  int64_t extent, ss, ds;
};

constexpr uint32_t kMaxRows = 1u << 30;
constexpr uint64_t kMaxUnitsPerRow = 1ull << 30;

struct Tuning {
  uint32_t tile_units = 4096;       // copy queue: 64 KiB tiles
  // link queue: one ring stage per tile.  3 stages x 4 KiB (8 KiB of loads in flight per CTA): deeper
  // rings only lengthen the queues at a source GPU whose HBM is busy with its own copy.  The multi-GPU
  // ring geometry has not been re-measured on H100; TSB_LINK_STAGES / TSB_LINK_STAGE_BYTES override it.
  uint32_t link_tile_units = 256;
  uint32_t link_stages = 3;
  bool link_stages_auto = true;     // no TSB_LINK_STAGES: pick the depth from the number of source GPUs
  bool link = true;
  bool link_all = false;  // TSB_LINK=2: local sources too (exercises the link warp on one GPU)
};

uint32_t env_u32(const char* name, uint32_t dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  long x = strtol(v, nullptr, 10);
  return x >= 0 ? static_cast<uint32_t>(x) : dflt;
}

Tuning default_tuning() {
  Tuning t;
  uint32_t bytes = env_u32("TSB_TILE_BYTES", 65536);
  t.tile_units = std::min<uint32_t>(32768u, std::max<uint32_t>(64u, bytes / 16));
  uint32_t sb = env_u32("TSB_LINK_STAGE_BYTES", 4096);
  sb = std::min<uint32_t>(16384u, std::max<uint32_t>(1024u, sb)) / 16 * 16;
  t.link_tile_units = sb / 16;
  t.link_stages = std::min<uint32_t>(8u, std::max<uint32_t>(3u, env_u32("TSB_LINK_STAGES", 3)));
  t.link_stages_auto = getenv("TSB_LINK_STAGES") == nullptr;
  const uint32_t lk = env_u32("TSB_LINK", 1);
  t.link = lk != 0;
  t.link_all = lk == 2;
  return t;
}

struct Compiler {
  Tuning tune;
  int plan_device;
  std::vector<DevRect> rects;
  std::vector<int32_t> rect_src_device;
  std::vector<uint32_t> rect_tiles;
  tsb_plan_info_t info{};

  // Emit one DevRect for (src, dst, outer dims, run of `units` units); splits oversize shapes.
  void emit(uint64_t src, uint64_t dst, std::vector<Dim> outer, uint64_t units, uint32_t mode,
            uint32_t sub, uint32_t dub, int32_t src_device) {
    if (units > kMaxUnitsPerRow) {
      // split the run into column chunks
      for (uint64_t u0 = 0; u0 < units; u0 += kMaxUnitsPerRow) {
        uint64_t n = std::min<uint64_t>(kMaxUnitsPerRow, units - u0);
        emit(src + u0 * sub, dst + u0 * dub, outer, n, mode, sub, dub, src_device);
      }
      return;
    }
    uint64_t rows = 1;
    for (const Dim& d : outer) rows *= static_cast<uint64_t>(d.extent);
    if (rows > kMaxRows) {
      // split the outermost dim that is > 1 in halves
      size_t k = 0;
      while (k < outer.size() && outer[k].extent == 1) ++k;
      Dim d = outer[k];
      int64_t h = d.extent / 2;
      std::vector<Dim> a = outer, b = outer;
      a[k].extent = h;
      b[k].extent = d.extent - h;
      emit(src, dst, a, units, mode, sub, dub, src_device);
      emit(src + static_cast<uint64_t>(h * d.ss), dst + static_cast<uint64_t>(h * d.ds), b, units, mode, sub, dub, src_device);
      return;
    }
    DevRect r;
    memset(&r, 0, sizeof(r));
    r.src = src;
    r.dst = dst;
    // drop unit extents created by splitting
    std::vector<Dim> o;
    for (const Dim& d : outer)
      if (d.extent != 1) o.push_back(d);
    r.n_outer = static_cast<uint32_t>(o.size());
    for (size_t i = 0; i < o.size(); ++i) {
      r.ext[i] = static_cast<uint32_t>(o[i].extent);
      r.src_stride[i] = o[i].ss;
      r.dst_stride[i] = o[i].ds;
    }
    r.rows = static_cast<uint32_t>(rows);
    r.units_per_row = static_cast<uint32_t>(units);
    r.magic = units == 1 ? 0u : static_cast<uint32_t>(((1ull << 32) + units - 1) / units);
    r.mode = mode;
    r.src_unit_bytes = sub;
    r.dst_unit_bytes = dub;
    const bool remote = src_device >= 0 && src_device != plan_device;
    // Link queue: 16-byte-unit moves out of another GPU's HBM whose rows are either wide or
    // addressed by ONE outer stride (what the link warp's per-lane row copies can express) and
    // whose strides are non-negative multiples of 16.  Everything else stays with the copy warps.
    bool link = tune.link && (remote || tune.link_all) && mode == MODE_B16;
    if (link && units < tune.link_tile_units && o.size() > 1) link = false;
    r.tile_units = link ? tune.link_tile_units : tune.tile_units;
    r.link = link ? 1u : 0u;
    uint64_t ntiles;
    if (units >= r.tile_units) {
      r.wide = 1;
      r.split = static_cast<uint32_t>((units + r.tile_units - 1) / r.tile_units);
      ntiles = rows * r.split;
    } else {
      r.wide = 0;
      r.split = std::max<uint32_t>(1u, r.tile_units / static_cast<uint32_t>(units));
      ntiles = (rows + r.split - 1) / r.split;
    }
    rects.push_back(r);
    rect_src_device.push_back(src_device);
    rect_tiles.push_back(static_cast<uint32_t>(ntiles));
    info.payload_bytes += rows * units * dub;
    info.src_bytes += rows * units * sub;
    if (remote) info.remote_src_bytes += rows * units * sub;
    if (link) info.link_bytes += rows * units * sub;
    if (is_vector_mode(mode)) info.num_vector_rects++;
  }

  int add(const tsb_rect_t& in, uint64_t index) {
    const std::string where = "rect " + std::to_string(index) + ": ";
    if (in.ndim < 1 || in.ndim > TSB_MAX_DIMS) return fail(TSB_ERR_INVALID, where + "ndim must be in [1, " + std::to_string(TSB_MAX_DIMS) + "]");
    const uint32_t es = dtype_size(in.src_dtype), ed = dtype_size(in.dst_dtype);
    if (!es || !ed) return fail(TSB_ERR_INVALID, where + "unknown dtype");
    uint32_t vmode = 0, smode = 0, velems = 0;
    const bool is_cast = in.src_dtype != in.dst_dtype;
    if (is_cast && !cast_modes(in.src_dtype, in.dst_dtype, &vmode, &smode, &velems))
      return fail(TSB_ERR_UNSUPPORTED, where + "dtype cast " + std::to_string(in.src_dtype) + " -> " + std::to_string(in.dst_dtype) + " is not implemented");

    std::vector<Dim> dims;
    for (uint32_t i = 0; i < in.ndim; ++i) {
      if (in.extent[i] < 0) return fail(TSB_ERR_INVALID, where + "negative extent");
      if (in.extent[i] == 0) return TSB_OK;  // empty rect: nothing to move
      if (in.extent[i] == 1) continue;
      dims.push_back({in.extent[i], in.src_stride[i], in.dst_stride[i]});
    }
    if (in.src == 0 || in.dst == 0) return fail(TSB_ERR_INVALID, where + "NULL src/dst");

    // innermost contiguous run, in elements
    int64_t run = 1;
    if (!dims.empty() && dims.back().ss == static_cast<int64_t>(es) && dims.back().ds == static_cast<int64_t>(ed)) {
      run = dims.back().extent;
      dims.pop_back();
      while (!dims.empty() && dims.back().ss == run * static_cast<int64_t>(es) && dims.back().ds == run * static_cast<int64_t>(ed)) {
        run *= dims.back().extent;
        dims.pop_back();
      }
    }
    // merge adjacent outer dims that are jointly contiguous on both sides
    for (size_t i = dims.size(); i >= 2; --i) {
      Dim& outer = dims[i - 2];
      Dim& inner = dims[i - 1];
      if (outer.ss == inner.ss * inner.extent && outer.ds == inner.ds * inner.extent) {
        outer.extent *= inner.extent;
        outer.ss = inner.ss;
        outer.ds = inner.ds;
        dims.erase(dims.begin() + static_cast<long>(i) - 1);
      }
    }

    auto all_aligned = [&](uint64_t a) {
      if (in.src % a || in.dst % a) return false;
      for (const Dim& d : dims)
        if (static_cast<uint64_t>(d.ss < 0 ? -d.ss : d.ss) % a || static_cast<uint64_t>(d.ds < 0 ? -d.ds : d.ds) % a) return false;
      return true;
    };

    if (!is_cast) {
      const uint64_t run_bytes = static_cast<uint64_t>(run) * es;
      uint32_t vec = 16;
      while (vec > 1 && (!all_aligned(vec) || run_bytes % vec)) vec >>= 1;
      uint32_t mode = vec == 16 ? MODE_B16 : vec == 8 ? MODE_B8 : vec == 4 ? MODE_B4 : vec == 2 ? MODE_B2 : MODE_B1;
      emit(in.src, in.dst, dims, run_bytes / vec, mode, vec, vec, in.src_device);
    } else {
      if (in.src % es || in.dst % ed) return fail(TSB_ERR_INVALID, where + "src/dst not aligned to their element size");
      for (const Dim& d : dims)
        if (d.ss % static_cast<int64_t>(es) || d.ds % static_cast<int64_t>(ed)) return fail(TSB_ERR_INVALID, where + "stride not a multiple of the element size");
      // vector unit: 8 elements (16-bit/32-bit pairs) or 16 (fp8 pairs: the fp8 side is one 16-byte access)
      if (vmode != 0xffffffffu && all_aligned(16) && run % velems == 0) {
        emit(in.src, in.dst, dims, static_cast<uint64_t>(run) / velems, vmode, velems * es, velems * ed, in.src_device);
      } else {
        emit(in.src, in.dst, dims, static_cast<uint64_t>(run), smode, es, ed, in.src_device);
      }
    }
    return TSB_OK;
  }

  uint32_t kind() const {
    if (rects.empty()) return KIND_GENERIC;
    bool all_b16 = true, all_cast = true, all_fp8 = true;
    for (const DevRect& r : rects) {
      all_b16 = all_b16 && r.mode == MODE_B16;
      all_cast = all_cast && r.mode == MODE_F32_BF16_V8;
      all_fp8 = all_fp8 && r.mode == MODE_BF16_E4M3_V16;
    }
    return all_b16 ? KIND_B16 : all_cast ? KIND_F32_BF16 : all_fp8 ? KIND_BF16_E4M3 : KIND_GENERIC;
  }

  // Tile order of one queue: proportional interleave over source devices, starting after the
  // plan's own device, in granules of `granule` consecutive tiles of one rect (the link queue
  // claims kLinkBatch tiles per atomic).  Group g's j-th granule sits at fractional position
  // (j + 0.5) / n_g of the queue, so every source GPU is drained at a constant rate for the whole
  // kernel: all inbound NVSwitch paths stay busy and the destinations do not gang up on one source.
  void order(bool link_queue, uint32_t flags, uint32_t granule, std::vector<DevTile>* out) const {
    uint64_t total = 0;
    std::vector<uint32_t> ids;
    for (uint32_t r = 0; r < rects.size(); ++r)
      if ((rects[r].link != 0) == link_queue) {
        ids.push_back(r);
        total += rect_tiles[r];
      }
    out->clear();
    out->reserve(total);
    if (flags & TSB_PLAN_NO_INTERLEAVE) {
      for (uint32_t r : ids)
        for (uint32_t t = 0; t < rect_tiles[r]; ++t) out->push_back({r, t});
      return;
    }
    std::map<int32_t, std::vector<uint32_t>> by_src;  // device -> rect ids
    for (uint32_t r : ids) by_src[rect_src_device[r]].push_back(r);
    struct Cursor {
      const std::vector<uint32_t>* rect_ids;
      size_t ri = 0;
      uint32_t ti = 0;
    };
    std::vector<Cursor> cursors;
    // rotate: first the device after ours, ..., ours last (local traffic does not need a port)
    std::vector<int32_t> keys;
    for (auto& kv : by_src) keys.push_back(kv.first);
    std::stable_sort(keys.begin(), keys.end(), [&](int32_t a, int32_t b) {
      auto rot = [&](int32_t k) -> int64_t {
        if (k < 0) return 1 << 20;
        int64_t d = static_cast<int64_t>(k) - plan_device - 1;
        if (d < 0) d += 1 << 16;
        return d;
      };
      return rot(a) < rot(b);
    });
    for (int32_t k : keys) cursors.push_back({&by_src[k]});
    std::vector<uint64_t> group_tiles(cursors.size(), 0);
    for (size_t g = 0; g < cursors.size(); ++g)
      for (uint32_t rid : *cursors[g].rect_ids) group_tiles[g] += rect_tiles[rid];
    std::vector<uint64_t> emitted(cursors.size(), 0);
    uint64_t k = 0;
    while (k < total) {
      size_t best = cursors.size();
      // pick the group that is furthest behind its schedule: minimise (2*emitted+1)/(2*n)
      for (size_t g = 0; g < cursors.size(); ++g) {
        if (emitted[g] >= group_tiles[g]) continue;
        if (best == cursors.size()) { best = g; continue; }
        const unsigned __int128 lhs = static_cast<unsigned __int128>(2 * emitted[g] + 1) * group_tiles[best];
        const unsigned __int128 rhs = static_cast<unsigned __int128>(2 * emitted[best] + 1) * group_tiles[g];
        if (lhs < rhs) best = g;
      }
      Cursor& c = cursors[best];
      for (uint32_t q = 0; q < granule && emitted[best] < group_tiles[best]; ++q) {
        while (c.ti >= rect_tiles[(*c.rect_ids)[c.ri]]) {
          ++c.ri;
          c.ti = 0;
        }
        out->push_back({(*c.rect_ids)[c.ri], c.ti++});
        ++emitted[best];
        ++k;
      }
    }
  }
};

struct Compiled {
  Compiler c;
  std::vector<DevTile> tiles, link_tiles;
};

int compile(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, const Tuning& tune, Compiled* out) {
  Compiler& c = out->c;
  c.tune = tune;
  c.plan_device = device;
  for (uint64_t i = 0; i < n; ++i) {
    int st = c.add(rects[i], i);
    if (st) return st;
  }
  uint64_t total = 0;
  for (uint32_t t : c.rect_tiles) total += t;
  if (total >= (1ull << 32)) return fail(TSB_ERR_UNSUPPORTED, "plan has more than 2^32 tiles");
  if (c.tune.link_stages_auto) {
    // Ring depth by fan-in: with many source GPUs each NVSwitch path carries a small share of the stream and
    // a deeper ring keeps enough bytes in flight; with <= 3 sources the deeper ring only lengthens the
    // queues at the busy sources.
    std::set<int32_t> sources;
    for (size_t i = 0; i < c.rects.size(); ++i)
      if (c.rects[i].link) sources.insert(c.rect_src_device[i]);
    c.tune.link_stages = sources.size() >= 4 ? 6u : 3u;
  }
  c.order(false, flags, 1, &out->tiles);
  c.order(true, flags, kLinkBatch, &out->link_tiles);
  c.info.num_rects = c.rects.size();
  c.info.num_tiles = out->tiles.size();
  c.info.num_link_tiles = out->link_tiles.size();
  c.info.tile_bytes = tune.tile_units * 16;
  c.info.link_tile_bytes = tune.link_tile_units * 16;
  c.info.link_stages = c.tune.link_stages;
  c.info.block = kCopyThreads + (out->link_tiles.empty() ? 0u : kLinkThreads);
  return TSB_OK;
}

// Persistent grid: SMs x CTAs/SM, never more than can be co-resident, never more than there is work.
int choose_grid(int device, uint32_t kind, const Compiled& cp, uint32_t* out_grid) {
  int sm = 0;
  int st = device_sm_count(device, &sm);
  if (st) return st;
  uint32_t per_sm = env_u32("TSB_CTAS_PER_SM", 3);
  if (per_sm == 0) per_sm = 3;
  const bool with_link = !cp.link_tiles.empty();
  {
    DeviceGuard guard(device);
    int resident = 0;
    if (guard.ok && max_ctas_per_sm(kind, with_link, cp.c.tune.link_stages * cp.c.tune.link_tile_units * 16, &resident) == TSB_OK &&
        resident > 0 && per_sm > static_cast<uint32_t>(resident))
      per_sm = static_cast<uint32_t>(resident);
  }
  uint64_t work = std::max<uint64_t>(cp.tiles.size(), (cp.link_tiles.size() + kLinkBatch - 1) / kLinkBatch);
  uint64_t grid = static_cast<uint64_t>(sm) * per_sm;
  if (grid > work) grid = work;
  // TSB_MAX_GRID caps the CTAs per launch (tests and ablations: a grid of 1 walks the whole queue in
  // one CTA); 0 or unset means no cap
  const uint32_t max_grid = env_u32("TSB_MAX_GRID", 0);
  if (max_grid && grid > max_grid) grid = max_grid;
  if (grid == 0) grid = 1;
  *out_grid = static_cast<uint32_t>(grid);
  return TSB_OK;
}

// Serialise {sched | rects | tiles | link tiles} into `dst` (layout.total bytes).
void fill_block(char* dst, const TableLayout& l, const Compiled& cp) {
  memset(dst, 0, kSchedBytes);
  if (!cp.c.rects.empty()) memcpy(dst + l.rects_off, cp.c.rects.data(), cp.c.rects.size() * sizeof(DevRect));
  if (!cp.tiles.empty()) memcpy(dst + l.tiles_off, cp.tiles.data(), cp.tiles.size() * sizeof(DevTile));
  if (!cp.link_tiles.empty()) memcpy(dst + l.link_off, cp.link_tiles.data(), cp.link_tiles.size() * sizeof(DevTile));
}

LaunchParams make_params(char* d_block, const TableLayout& l, uint32_t n_tiles, uint32_t n_link, uint32_t kind,
                         uint32_t link_stage_bytes, uint32_t link_stages) {
  LaunchParams lp{};
  lp.tiles = reinterpret_cast<const DevTile*>(d_block + l.tiles_off);
  lp.rects = reinterpret_cast<const DevRect*>(d_block + l.rects_off);
  lp.link_tiles = n_link ? reinterpret_cast<const DevTile*>(d_block + l.link_off) : nullptr;
  lp.num_tiles = n_tiles;
  lp.num_link_tiles = n_link;
  lp.kind = kind;
  lp.link_stage_bytes = link_stage_bytes;
  lp.link_stages = link_stages;
  lp.sched = reinterpret_cast<uint32_t*>(d_block);
  return lp;
}

void free_plan(Plan* p) {
  DeviceGuard guard(p->device);
  if (p->ev_fence) cudaEventDestroy(p->ev_fence);
  if (p->ev_start) cudaEventDestroy(p->ev_start);
  if (p->ev_done) cudaEventDestroy(p->ev_done);
  if (p->d_block) cudaFree(p->d_block);  // synchronises with outstanding work that uses the tables
  delete p;
}

// ---- one-shot table pool ---------------------------------------------------------------------------
constexpr size_t kPoolMinBytes = 256 << 10;
constexpr size_t kPoolMaxBlocks = 64;

PoolBlock* pool_acquire_locked(PlanRegistry& reg, int device, size_t bytes, int* status) {
  *status = TSB_OK;
  for (PoolBlock* b : reg.pool) {
    if (b->device != device || b->cap < bytes) continue;
    if (b->in_flight) {
      cudaError_t e = cudaEventQuery(b->done);
      if (e == cudaErrorNotReady) {
        cudaGetLastError();
        continue;
      }
      b->in_flight = false;
    }
    ++reg.pool_reuses;
    return b;
  }
  if (reg.pool.size() >= kPoolMaxBlocks) {
    // drop one idle block that is too small (or belongs to another device) to make room
    for (size_t i = 0; i < reg.pool.size(); ++i) {
      PoolBlock* b = reg.pool[i];
      if (b->in_flight && cudaEventQuery(b->done) == cudaErrorNotReady) {
        cudaGetLastError();
        continue;
      }
      DeviceGuard g(b->device);
      cudaFree(b->d);
      cudaFreeHost(b->h);
      cudaEventDestroy(b->done);
      delete b;
      reg.pool.erase(reg.pool.begin() + static_cast<long>(i));
      break;
    }
  }
  PoolBlock* b = new PoolBlock();
  b->device = device;
  b->cap = std::max(kPoolMinBytes, (bytes + 65535) / 65536 * 65536);
  cudaError_t e = cudaMalloc(&b->d, b->cap);
  if (e == cudaSuccess) e = cudaHostAlloc(&b->h, b->cap, cudaHostAllocPortable);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&b->done, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    if (b->d) cudaFree(b->d);
    if (b->h) cudaFreeHost(b->h);
    delete b;
    *status = cuda_fail(e, "table pool allocation");
    return nullptr;
  }
  ++reg.pool_allocs;
  reg.pool.push_back(b);
  return b;
}

int find_plan(tsb_plan_t plan, Plan** out) {
  PlanRegistry& reg = R();
  std::lock_guard<std::mutex> lk(reg.mu);
  auto it = reg.plans.find(plan);
  if (it == reg.plans.end()) return fail(TSB_ERR_NOTFOUND, "unknown plan");
  *out = it->second;
  return TSB_OK;
}

int run_plan(Plan* p, cudaStream_t s) {
  if (p->quant) return p->quant(p->d_block, s);
  uint32_t kind = p->kind;
  if (getenv("TSB_FORCE_GENERIC")) kind = KIND_GENERIC;
  LaunchParams lp = make_params(p->d_block, p->layout, p->num_tiles, p->num_link_tiles, kind, p->link_stage_bytes, p->link_stages);
  if (getenv("TSB_STATIC_SCHED") && p->num_link_tiles == 0) lp.sched = nullptr;
  return launch_copy_rects(lp, p->info.grid, s);
}

// Upload a plan's serialised tables, create its launch events and register it; frees `p` on failure.
int register_plan(Plan* p, const std::vector<char>& host, tsb_plan_t* out) {
  int st;
  {
    // upload on the device's copy stream and wait for it: after this returns the tables are in
    // HBM whatever stream the plan is later run on
    cudaStream_t up;
    if ((st = copy_stream(p->device, &up))) {
      delete p;
      return st;
    }
    DeviceGuard guard(p->device);
    if (!guard.ok) { delete p; return cuda_fail(guard.err, "cudaSetDevice"); }
    cudaError_t e = cudaMalloc(&p->d_block, host.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(p->d_block, host.data(), host.size(), cudaMemcpyHostToDevice, up);
    if (e == cudaSuccess) e = cudaStreamSynchronize(up);
    // the events of tsb_plan_launch belong to the plan and exist from the start (no lazy creation that
    // two threads launching the same plan could race on)
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_fence, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreate(&p->ev_start);
    if (e == cudaSuccess) e = cudaEventCreate(&p->ev_done);
    if (e != cudaSuccess) {
      cuda_fail(e, "plan upload");
      free_plan(p);
      return TSB_ERR_CUDA;
    }
  }
  PlanRegistry& reg = R();
  std::lock_guard<std::mutex> lk(reg.mu);
  uint64_t id = reg.next_id++;
  reg.plans[id] = p;
  *out = id;
  return TSB_OK;
}

}  // namespace

namespace {

int check_quant_flags(const char* fn, uint32_t flags, uint32_t accepted) {
  if (flags & ~accepted)
    return fail(TSB_ERR_INVALID, std::string(fn) + (accepted ? ": flags must be 0 or TSB_QUANT_UE8M0" : ": flags must be 0"));
  return TSB_OK;
}

}  // namespace

int quant_plan_create(const char* fn, int device, uint32_t flags, uint32_t accepted, tsb_plan_t* out, const QuantCompile& compile) {
  if (!out) return fail(TSB_ERR_INVALID, std::string(fn) + ": NULL argument");
  if (int st = check_quant_flags(fn, flags, accepted)) return st;
  QuantPlan q;
  q.ue8m0 = (flags & TSB_QUANT_UE8M0) != 0;
  int st = compile(&q);
  if (st) return st;
  Plan* p = new Plan();
  p->device = device;
  p->num_tiles = static_cast<uint32_t>(q.info.num_tiles);
  p->info = q.info;
  p->quant = std::move(q.launch);
  return register_plan(p, q.tables, out);
}

int quant_compile_host(const char* fn, uint32_t flags, uint32_t accepted, const QuantCompile& compile,
                       std::initializer_list<TableOut> outs, uint64_t* out_n_groups) {
  if (int st = check_quant_flags(fn, flags, accepted)) return st;
  QuantPlan q;
  q.ue8m0 = (flags & TSB_QUANT_UE8M0) != 0;
  int st = compile(&q);
  if (st) return st;
  size_t k = 0;
  for (const TableOut& o : outs) {
    if (o.n) *o.n = q.sections[k].count;
    ++k;
  }
  if (out_n_groups) *out_n_groups = q.n_groups;
  k = 0;
  for (const TableOut& o : outs) {
    const QuantPlan::Section& t = q.sections[k++];
    if (!o.out) continue;
    if (t.count > o.cap) return fail(TSB_ERR_NOMEM, std::string(o.name) + " too small");
    if (t.count) memcpy(o.out, q.tables.data() + t.off, t.bytes);
  }
  return TSB_OK;
}

int plans_shutdown() {
  PlanRegistry& reg = R();
  std::lock_guard<std::mutex> lk(reg.mu);
  for (auto& kv : reg.plans) free_plan(kv.second);
  reg.plans.clear();
  for (PoolBlock* b : reg.pool) {
    DeviceGuard g(b->device);
    if (b->in_flight) cudaEventSynchronize(b->done);
    cudaFree(b->d);
    cudaFreeHost(b->h);
    cudaEventDestroy(b->done);
    delete b;
  }
  reg.pool.clear();
  return TSB_OK;
}

}  // namespace tsb

using namespace tsb;

extern "C" {

int tsb_cast_supported(uint32_t src_dtype, uint32_t dst_dtype) {
  if (!dtype_size(src_dtype) || !dtype_size(dst_dtype)) return 0;
  if (src_dtype == dst_dtype) return 1;
  uint32_t v, s;
  return cast_modes(src_dtype, dst_dtype, &v, &s) ? 1 : 0;
}

// Host-only: compile rects and copy the tables out (no CUDA call).  Used by the CPU test-suite to
// check the index math of the plan compiler against the oracle without a GPU.  `out_rects` points
// at n_rect_cap records of 192 bytes (DevRect), `out_tiles` at n_tile_cap pairs of uint32: the
// copy queue followed by the link queue (out_info->num_tiles / num_link_tiles entries).
int tsb_plan_compile_host(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, uint32_t tile_units,
                          void* out_rects, uint64_t n_rect_cap, uint64_t* out_n_rects, void* out_tiles,
                          uint64_t n_tile_cap, uint64_t* out_n_tiles, tsb_plan_info_t* out_info) {
  if (n && !rects) return fail(TSB_ERR_INVALID, "rects is NULL");
  Tuning tune = default_tuning();
  if (tile_units != 0) tune.tile_units = tile_units;
  if (tune.tile_units > 32768) return fail(TSB_ERR_INVALID, "tile_units must be <= 32768");
  Compiled cp;
  int st = compile(device, rects, n, flags, tune, &cp);
  if (st) return st;
  const uint64_t n_tiles = cp.tiles.size() + cp.link_tiles.size();
  if (out_n_rects) *out_n_rects = cp.c.rects.size();
  if (out_n_tiles) *out_n_tiles = n_tiles;
  if (out_info) *out_info = cp.c.info;
  if (out_rects) {
    if (cp.c.rects.size() > n_rect_cap) return fail(TSB_ERR_NOMEM, "out_rects too small");
    memcpy(out_rects, cp.c.rects.data(), cp.c.rects.size() * sizeof(DevRect));
  }
  if (out_tiles) {
    if (n_tiles > n_tile_cap) return fail(TSB_ERR_NOMEM, "out_tiles too small");
    char* o = static_cast<char*>(out_tiles);
    memcpy(o, cp.tiles.data(), cp.tiles.size() * sizeof(DevTile));
    memcpy(o + cp.tiles.size() * sizeof(DevTile), cp.link_tiles.data(), cp.link_tiles.size() * sizeof(DevTile));
  }
  return TSB_OK;
}

int tsb_plan_create(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, tsb_plan_t* out) {
  if (!out || (n && !rects)) return fail(TSB_ERR_INVALID, "tsb_plan_create: NULL argument");
  Compiled cp;
  int st = compile(device, rects, n, flags, default_tuning(), &cp);
  if (st) return st;
  Plan* p = new Plan();
  p->device = device;
  p->num_tiles = static_cast<uint32_t>(cp.tiles.size());
  p->num_link_tiles = static_cast<uint32_t>(cp.link_tiles.size());
  p->info = cp.c.info;
  p->kind = cp.c.kind();
  p->link_stage_bytes = cp.c.tune.link_tile_units * 16;
  p->link_stages = cp.c.tune.link_stages;
  if ((st = choose_grid(device, p->kind, cp, &p->info.grid))) {
    delete p;
    return st;
  }
  p->layout = table_layout(cp.c.rects.size(), cp.tiles.size(), cp.link_tiles.size());
  std::vector<char> host(p->layout.total);
  fill_block(host.data(), p->layout, cp);
  return register_plan(p, host, out);
}

int tsb_plan_info(tsb_plan_t plan, tsb_plan_info_t* out) {
  if (!out) return fail(TSB_ERR_INVALID, "out is NULL");
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  *out = p->info;
  return TSB_OK;
}

int tsb_plan_run(tsb_plan_t plan, void* stream) {
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  if (p->num_tiles == 0 && p->num_link_tiles == 0) return TSB_OK;
  cudaStream_t s = resolve_stream(p->device, stream, &st);
  if (st) return st;
  DeviceGuard guard(p->device);
  if (!guard.ok) return cuda_fail(guard.err, "cudaSetDevice");
  return run_plan(p, s);
}

// One call per sync: [caller stream -> fence] start, kernel, done [-> caller stream waits].
int tsb_plan_launch(tsb_plan_t plan, void* caller_stream) { return tsb_plan_launch_flags(plan, caller_stream, TSB_LAUNCH_DEFAULT); }

int tsb_plan_launch_flags(tsb_plan_t plan, void* caller_stream, uint32_t flags) {
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  cudaStream_t s;
  if ((st = copy_stream(p->device, &s))) return st;
  DeviceGuard guard(p->device);
  if (!guard.ok) return cuda_fail(guard.err, "cudaSetDevice");
  cudaStream_t cs = reinterpret_cast<cudaStream_t>(caller_stream);
  if (cs) {
    TSB_CUDA(cudaEventRecord(p->ev_fence, cs));
    TSB_CUDA(cudaStreamWaitEvent(s, p->ev_fence, 0));
  }
  TSB_CUDA(cudaEventRecord(p->ev_start, s));
  if (p->num_tiles || p->num_link_tiles) {
    if ((st = run_plan(p, s))) return st;
  }
  TSB_CUDA(cudaEventRecord(p->ev_done, s));
  if (cs && !(flags & TSB_LAUNCH_NO_FENCE_OUT)) TSB_CUDA(cudaStreamWaitEvent(cs, p->ev_done, 0));
  p->launched = true;
  return TSB_OK;
}

int tsb_plan_poll(tsb_plan_t plan, int* out_done) {
  if (!out_done) return fail(TSB_ERR_INVALID, "out_done is NULL");
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  if (!p->launched) {
    *out_done = 1;
    return TSB_OK;
  }
  cudaError_t e = cudaEventQuery(p->ev_done);
  if (e == cudaSuccess) {
    *out_done = 1;
    return TSB_OK;
  }
  if (e == cudaErrorNotReady) {
    cudaGetLastError();
    *out_done = 0;
    return TSB_OK;
  }
  return cuda_fail(e, "cudaEventQuery");
}

int tsb_plan_wait(tsb_plan_t plan) {
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  if (!p->launched) return TSB_OK;
  TSB_CUDA(cudaEventSynchronize(p->ev_done));
  return TSB_OK;
}

int tsb_plan_elapsed_ms(tsb_plan_t plan, float* out_ms) {
  if (!out_ms) return fail(TSB_ERR_INVALID, "out_ms is NULL");
  Plan* p;
  int st = find_plan(plan, &p);
  if (st) return st;
  if (!p->launched) return fail(TSB_ERR_INVALID, "plan was never launched with tsb_plan_launch");
  TSB_CUDA(cudaEventElapsedTime(out_ms, p->ev_start, p->ev_done));
  return TSB_OK;
}

int tsb_plan_destroy(tsb_plan_t plan) {
  PlanRegistry& reg = R();
  Plan* p;
  {
    std::lock_guard<std::mutex> lk(reg.mu);
    auto it = reg.plans.find(plan);
    if (it == reg.plans.end()) return fail(TSB_ERR_NOTFOUND, "unknown plan");
    p = it->second;
    reg.plans.erase(it);
  }
  free_plan(p);
  return TSB_OK;
}

// One-shot: compile, upload and launch on ONE stream; the tables come from a recycled pool.
int tsb_copy_rects(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, void* stream) {
  if (n && !rects) return fail(TSB_ERR_INVALID, "tsb_copy_rects: NULL argument");
  Compiled cp;
  int st = compile(device, rects, n, flags, default_tuning(), &cp);
  if (st) return st;
  if (cp.tiles.empty() && cp.link_tiles.empty()) return TSB_OK;
  const uint32_t kind = getenv("TSB_FORCE_GENERIC") ? static_cast<uint32_t>(KIND_GENERIC) : cp.c.kind();
  uint32_t grid = 1;
  if ((st = choose_grid(device, kind, cp, &grid))) return st;
  cudaStream_t s = resolve_stream(device, stream, &st);
  if (st) return st;
  DeviceGuard guard(device);
  if (!guard.ok) return cuda_fail(guard.err, "cudaSetDevice");
  const TableLayout l = table_layout(cp.c.rects.size(), cp.tiles.size(), cp.link_tiles.size());
  PlanRegistry& reg = R();
  std::lock_guard<std::mutex> lk(reg.mu);
  PoolBlock* b = pool_acquire_locked(reg, device, l.total, &st);
  if (!b) return st;
  fill_block(b->h, l, cp);
  TSB_CUDA(cudaMemcpyAsync(b->d, b->h, l.total, cudaMemcpyHostToDevice, s));
  LaunchParams lp = make_params(b->d, l, static_cast<uint32_t>(cp.tiles.size()), static_cast<uint32_t>(cp.link_tiles.size()), kind,
                                cp.c.tune.link_tile_units * 16, cp.c.tune.link_stages);
  b->in_flight = true;  // even if the launch fails the upload may still be queued
  st = launch_copy_rects(lp, grid, s);
  cudaError_t e = cudaEventRecord(b->done, s);
  if (st) return st;
  if (e != cudaSuccess) return cuda_fail(e, "cudaEventRecord");
  return TSB_OK;
}

int tsb_pool_stats(uint64_t* out_blocks, uint64_t* out_allocs, uint64_t* out_reuses) {
  PlanRegistry& reg = R();
  std::lock_guard<std::mutex> lk(reg.mu);
  if (out_blocks) *out_blocks = reg.pool.size();
  if (out_allocs) *out_allocs = reg.pool_allocs;
  if (out_reuses) *out_reuses = reg.pool_reuses;
  return TSB_OK;
}

}  // extern "C"
