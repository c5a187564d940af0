// Internal declarations shared by the translation units of libtstore_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <string>
#include <vector>

#include "tstore_b200.h"

namespace tsb {

// ---- error plumbing -----------------------------------------------------------------------
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);

#define TSB_CUDA(expr)                                   \
  do {                                                   \
    cudaError_t _e = (expr);                             \
    if (_e != cudaSuccess) return ::tsb::cuda_fail(_e, #expr); \
  } while (0)

// RAII: switch the calling thread to `device`, restore on scope exit (torch owns the
// thread's current device; we must not disturb it).
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  bool had_context = true;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device);  // runtime.cu
  ~DeviceGuard() {
    // restore only if this thread had a context before: on a fresh thread (the actor-server thread)
    // "restoring" device 0 would create a primary context on GPU 0 in every rank's process
    if (ok && had_context && prev >= 0 && prev != cur) cudaSetDevice(prev);
  }
  int cur = -1;
};

// ---- per-device state -----------------------------------------------------------------------
int device_sm_count(int device, int* out);
int copy_stream(int device, cudaStream_t* out);
cudaStream_t resolve_stream(int device, void* stream, int* status);

// ---- kernel-side structures -------------------------------------------------------------------
// Copy modes of a compiled rect: how one "unit" (the thing a thread moves per step) is defined.
enum : uint32_t {
  MODE_B1 = 0,   // unit = 1 byte
  MODE_B2 = 1,
  MODE_B4 = 2,
  MODE_B8 = 3,
  MODE_B16 = 4,  // unit = 16 bytes (LDG.128 / STG.128)
  // casts: unit = 8 elements (vector) or 1 element (scalar)
  MODE_F32_BF16_V8 = 8,
  MODE_F32_BF16_S = 9,
  MODE_F32_F16_V8 = 10,
  MODE_F32_F16_S = 11,
  MODE_BF16_F32_V8 = 12,
  MODE_BF16_F32_S = 13,
  MODE_F16_F32_V8 = 14,
  MODE_F16_F32_S = 15,
  MODE_BF16_F16_V8 = 16,
  MODE_BF16_F16_S = 17,
  MODE_F16_BF16_V8 = 18,
  MODE_F16_BF16_S = 19,
  MODE_F64_F32_S = 20,
  MODE_F32_F64_S = 21,
  // fp8 casts: unit = 16 elements (vector: the fp8 side is one 16-byte access) or 1 element (scalar)
  MODE_F32_E4M3_V16 = 22,
  MODE_F32_E4M3_S = 23,
  MODE_F32_E5M2_V16 = 24,
  MODE_F32_E5M2_S = 25,
  MODE_BF16_E4M3_V16 = 26,
  MODE_BF16_E4M3_S = 27,
  MODE_BF16_E5M2_V16 = 28,
  MODE_BF16_E5M2_S = 29,
  MODE_F16_E4M3_V16 = 30,
  MODE_F16_E4M3_S = 31,
  MODE_F16_E5M2_V16 = 32,
  MODE_F16_E5M2_S = 33,
  MODE_E4M3_F32_V16 = 34,
  MODE_E4M3_F32_S = 35,
  MODE_E5M2_F32_V16 = 36,
  MODE_E5M2_F32_S = 37,
  MODE_E4M3_BF16_V16 = 38,
  MODE_E4M3_BF16_S = 39,
  MODE_E5M2_BF16_V16 = 40,
  MODE_E5M2_BF16_S = 41,
  MODE_E4M3_F16_V16 = 42,
  MODE_E4M3_F16_S = 43,
  MODE_E5M2_F16_V16 = 44,
  MODE_E5M2_F16_S = 45,
};

// modes whose units are 16-byte accesses on both sides (plan info: num_vector_rects)
constexpr bool is_vector_mode(uint32_t m) {
  return m == MODE_B16 || (m >= MODE_F32_BF16_V8 && m <= MODE_F16_BF16_V8 && m % 2 == 0) ||
         (m >= MODE_F32_E4M3_V16 && m <= MODE_E5M2_F16_V16 && m % 2 == 0);
}

constexpr int kMaxOuter = TSB_MAX_DIMS;  // outer (row) dims after splitting off the run

// Device-resident compiled rect.  16-byte aligned, size multiple of 16 so that a few lanes can
// stage it into shared memory with cp.async.
struct alignas(16) DevRect {
  uint64_t src;
  uint64_t dst;
  int64_t src_stride[kMaxOuter];  // bytes, outermost first; only [0, n_outer) valid
  int64_t dst_stride[kMaxOuter];
  uint32_t ext[kMaxOuter];        // extents of the outer dims
  uint32_t n_outer;               // 0 => a single row
  uint32_t rows;                  // prod(ext[0..n_outer))
  uint32_t units_per_row;         // U
  uint32_t magic;                 // ceil(2^32 / U) (0 when U == 1)
  uint32_t wide;                  // 1: tiles are segments of one row; 0: tiles are groups of whole rows
  uint32_t split;                 // wide: tiles per row; narrow: rows per tile
  uint32_t mode;
  uint32_t src_unit_bytes;        // bytes one unit spans in src
  uint32_t dst_unit_bytes;        // bytes one unit spans in dst
  uint32_t tile_units;            // tile size of THIS rect (link rects use the TMA stage size)
  uint32_t link;                  // 1: tiles of this rect are in the link queue (TMA bulk over NVLink)
  uint32_t pad_[3];
};
static_assert(sizeof(DevRect) == 192, "DevRect layout changed: keep it a multiple of 16 bytes");

struct DevTile {
  uint32_t rect;
  uint32_t tile_in_rect;
};

// kernel specialisations (see copy_rects.cu)
enum : uint32_t { KIND_GENERIC = 0, KIND_B16 = 1, KIND_F32_BF16 = 2, KIND_BF16_E4M3 = 3 };

// Two work queues per plan (see copy_rects.cu):
//   copy queue  tiles moved by the CTA's 8 copy warps with LDG.128/STG.128 (local HBM sources,
//               casts, misaligned rects, peer destinations)
//   link queue  tiles whose source is another GPU's HBM and that move 16-byte units: driven by one
//               extra "link warp" per CTA through a ring of TMA bulk copies
//               (peer global -> shared -> local global), fully asynchronous to the copy warps
struct LaunchParams {
  const DevTile* tiles;       // copy queue
  const DevRect* rects;
  const DevTile* link_tiles;  // link queue (nullptr when empty)
  uint32_t num_tiles;
  uint32_t num_link_tiles;
  uint32_t kind;
  uint32_t link_stage_bytes;  // bytes per ring stage (== tile size of link rects)
  uint32_t link_stages;       // ring depth S (stores trail loads by S-2 stages)
  uint32_t* sched;  // {copy claim, finished CTAs, link claim, pad}; nullptr = fully static striding (no link queue)
};

constexpr uint32_t kCopyThreads = 256;
constexpr uint32_t kLinkThreads = 32;
constexpr uint32_t kLinkBatch = 8;  // link tiles claimed per atomic

// defined in copy_rects.cu
int launch_copy_rects(const LaunchParams& p, uint32_t grid, cudaStream_t stream);
void count_launch();
int max_ctas_per_sm(uint32_t kind, bool with_link, uint32_t link_smem_bytes, int* out);

// ---- scaled fp8 plans: what every kind shares ---------------------------------------------------------
constexpr uint32_t kQuantThreads = 256;  // CTA size of every scaled fp8 kernel

inline uint32_t round16(uint64_t x) { return static_cast<uint32_t>((x + 15u) & ~uint64_t(15)); }

// rows from p, `stride` bytes apart, all start 16-byte aligned
inline bool aligned16(uint64_t p, int64_t stride, uint64_t rows) { return p % 16 == 0 && (rows == 1 || stride % 16 == 0); }

// ... and rows of `cols` elements of `es` bytes are whole 16-byte units: 16-byte accesses cover them
inline bool vec_ok(uint64_t p, int64_t stride, uint64_t rows, uint64_t cols, uint32_t es) {
  return aligned16(p, stride, rows) && (cols * es) % 16 == 0;
}

// The byte counts of tsb_plan_info_t a scaled fp8 compiler accumulates.
struct PlanBytes {
  uint64_t src_bytes = 0, remote_src_bytes = 0, payload_bytes = 0;
  // `bytes` read by a plan of `device` from a source on `src_device` (< 0: not a GPU)
  void read(uint64_t bytes, int32_t src_device, int device) {
    src_bytes += bytes;
    if (src_device >= 0 && src_device != device) remote_src_bytes += bytes;
  }
};

// A scaled fp8 grid as the compilers validate it: `batch` [rows, cols] matrices of `es`-byte elements at `base`
// and global offset (row0, col0), with their float32 scales at `scale`.  `null`: one of its pointers is NULL.
struct Grid {
  uint64_t base, scale, batch, rows, cols, row0, col0;
  uint32_t es, granularity, pad;
  bool null;
};
// What differs between the compilers' checks of their grids.
struct GridRules {
  const char* noun;          // "target" / "source": messages start "<noun> N: "
  const char* null_msg;      // the message for `null`
  const char* base_name;     // names the base in the element-alignment message
  const char* scale_name;    // names the scale in the 4-byte-alignment message
  uint32_t granularities;    // the accepted TSB_SCALE_* as bits 1 << g; 0: the grid has no granularity
  uint64_t max_cols;         // cols must stay below this
};
// TSB_ERR_INVALID naming grid `index` unless it passes `rules` (block_fp8.cu).
int check_grid(const GridRules& rules, uint64_t index, const Grid& g);

// Exact coverage of one [rows, cols] matrix by `boxes` (anything with r0, er, c0, ec; sorted by r0): between two
// consecutive box row boundaries y and y1 the boxes spanning those rows, sorted by column, must cut [0, cols) into
// contiguous, disjoint runs.  Checks in time proportional to the boxes, not the elements.  Calls band(y, y1, sorted)
// for each band of rows that passes, and returns gap(y, c) at the first that does not, c being the first column not
// covered exactly once (clamped to cols - 1); a non-zero status of either ends the sweep.
template <class Box, class Band, class Gap>
int sweep_cover(uint64_t rows, uint64_t cols, const Box* const* boxes, size_t nb, Band&& band, Gap&& gap) {
  std::vector<const Box*> act, sorted;
  size_t i = 0;
  for (uint64_t y = 0; y < rows;) {
    while (i < nb && boxes[i]->r0 == y) act.push_back(boxes[i++]);
    act.erase(std::remove_if(act.begin(), act.end(), [y](const Box* x) { return x->r0 + x->er <= y; }), act.end());
    uint64_t y1 = i < nb ? boxes[i]->r0 : rows;
    for (const Box* x : act) y1 = std::min(y1, x->r0 + x->er);
    sorted = act;
    std::sort(sorted.begin(), sorted.end(), [](const Box* a, const Box* b) { return a->c0 < b->c0; });
    uint64_t c = 0;
    bool ok = true;
    for (const Box* x : sorted) {
      if (x->c0 != c) {
        ok = false;
        c = std::min(c, x->c0);
        break;
      }
      c += x->ec;
    }
    if (!ok || c != cols) return gap(y, std::min(c, cols - 1));
    if (int st = band(y, y1, sorted)) return st;
    y = y1;
  }
  return TSB_OK;
}

// One sealed scaled fp8 plan, as its kind's .cu file describes it to plan.cu: only that file knows the tables'
// layout and how to launch from them.
struct QuantPlan {
  struct Section {
    size_t off;      // byte offset in `tables`
    uint64_t count;  // records
    size_t bytes;    // count * record size
  };
  std::vector<char> tables;       // every table back to back, then the zeroed amax words
  std::vector<Section> sections;  // the tables, in the order of the kind's tsb_*_compile_host outputs
  uint32_t n_groups = 0;          // amax words
  bool ue8m0 = false;             // TSB_QUANT_UE8M0: the launch runs the power-of-two scale kernels (tables unchanged)
  bool int8 = false;              // TSB_I8 destinations: the launch runs the int8 kernels (tables unchanged)
  tsb_plan_info_t info{};
  std::function<int(char* d, cudaStream_t)> launch;  // runs the plan from its tables' device copy at d

  // Append a table; returns its byte offset.
  template <class T>
  size_t add(const std::vector<T>& v) {
    const size_t off = tables.size();
    tables.resize(off + v.size() * sizeof(T));
    if (!v.empty()) memcpy(tables.data() + off, v.data(), v.size() * sizeof(T));
    sections.push_back({off, v.size(), v.size() * sizeof(T)});
    return off;
  }
  // After the last table: `groups` zeroed amax words (at the returned offset), at least 16 bytes in all.
  size_t seal(uint32_t groups) {
    const size_t off = tables.size();
    n_groups = groups;
    tables.resize(std::max<size_t>(16, off + 4ull * groups), 0);
    return off;
  }
  // tsb_plan_info_t: `inputs` rects (or targets), one kQuantThreads CTA per each of `ctas` records
  void describe(uint64_t inputs, uint32_t ctas, uint32_t tile_bytes, const PlanBytes& b) {
    info.num_rects = inputs;
    info.num_tiles = ctas;
    info.grid = ctas;
    info.block = kQuantThreads;
    info.tile_bytes = tile_bytes;
    info.payload_bytes = b.payload_bytes;
    info.src_bytes = b.src_bytes;
    info.remote_src_bytes = b.remote_src_bytes;
  }
};
using QuantCompile = std::function<int(QuantPlan*)>;
// The bodies of tsb_*_plan_create and tsb_*_compile_host (plan.cu): `fn` names the entry in its argument errors,
// `accepted` the TSB_QUANT_* bits the kind takes in `flags` (any other bit is TSB_ERR_INVALID); compile() sees
// them in QuantPlan::ue8m0.
int quant_plan_create(const char* fn, int device, uint32_t flags, uint32_t accepted, tsb_plan_t* out, const QuantCompile& compile);
struct TableOut {
  void* out;          // NULL: not wanted
  uint64_t cap;       // records out can take
  uint64_t* n;        // the table's record count (if not NULL)
  const char* name;   // the argument, for TSB_ERR_NOMEM
};
int quant_compile_host(const char* fn, uint32_t flags, uint32_t accepted, const QuantCompile& compile,
                       std::initializer_list<TableOut> outs, uint64_t* out_n_groups);

// After a kernel launch: its launch error, or count it.
inline int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, what);
  count_launch();
  return TSB_OK;
}

// ---- scaled fp8 destinations: the rect -> [batch, rows, cols] mapping (block_fp8.cu) ----------------
// Where a quantised destination lives: `batch` contiguous [rows, cols] float8_e4m3fn matrices at dst.
struct TargetGeom {
  uint64_t dst, batch, rows, cols;
};
// A rect after mapping onto its target: an [er, ec] box of matrix b at (r0, c0), source rows contiguous.
struct TargetBox {
  uint64_t src;
  int64_t row_stride;  // source bytes between rows (0 for a single row)
  uint64_t target, b, r0, c0, er, ec;
  uint32_t dtype;
  int32_t src_device;
  uint32_t rstep = 1;  // grid rows between the box's rows: 2 for a rotary head half mapped by its source, else 1
};
uint32_t quant_src_bytes(uint32_t dtype);  // 4 / 2 for TSB_F32 / TSB_BF16, TSB_F16; 0 otherwise
// Append one box per combination of the rect's batch dims to `out` (nothing for an empty rect).
int rect_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* targets, uint64_t n_targets,
               std::vector<TargetBox>* out);
// The same mapping from the other side: the rect's *source* is located on the fp8 grids (its
// TargetGeom::dst is the grid's base), and a box's `src` / `row_stride` / `dtype` describe the
// destination side.  Destination columns must be contiguous.  A row dim that steps two grid rows (a rotary
// head half, read in interleaved order) gives a box of rows r0, r0 + 2, ... (TargetBox::rstep 2).
int rect_source_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* grids, uint64_t n_grids,
                      std::vector<TargetBox>* out);
// Whether the rects of a quantising pull (each already checked by rect_boxes) write int8 (TSB_I8) rather than
// float8_e4m3fn: TSB_ERR_INVALID when they mix the two, or for int8 with TSB_QUANT_UE8M0 (`ue8m0`).
int quant_dst_int8(const tsb_rect_t* rects, uint64_t n, bool ue8m0, bool* int8);
// rect_boxes for requantising pulls: float8_e4m3fn on both sides; a box's `src` / `row_stride` are the
// source's fp8 bytes.
int rect_requant_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* targets, uint64_t n_targets,
                       std::vector<TargetBox>* out);

// ---- block-scaled fp8 (block_fp8.cu) ---------------------------------------------------------------
constexpr uint32_t kBqBlock = 128;  // block edge (elements)

// One 128x128 (or partial edge) block of a target: CTA-sized unit of work.
struct alignas(16) BqBlock {
  uint64_t dst;          // fp8 element (0, 0) of the block
  uint64_t scale;        // its float32 scale_inv
  uint32_t pitch;        // destination row pitch (bytes == elements)
  uint16_t rows, cols;   // real extent of the block
  uint32_t piece0;       // first piece
  uint16_t n_pieces;
  uint16_t src_dtype;    // TSB_F32 / TSB_BF16 / TSB_F16, the same for every piece of the block
};
static_assert(sizeof(BqBlock) == 32, "BqBlock is part of tsb_block_fp8_compile_host's output");

// A source rectangle inside one block.
struct alignas(16) BqPiece {
  uint64_t src;          // source element (row0, col0) of the piece
  int64_t src_stride;    // bytes between source rows
  uint16_t row0, col0;   // position inside the block
  uint16_t rows, cols;
  uint32_t vec;          // 1: source address, stride, column offset and width allow 16-byte accesses
  uint32_t pad_;
};
static_assert(sizeof(BqPiece) == 32, "BqPiece is part of tsb_block_fp8_compile_host's output");

struct BqTables : PlanBytes {
  std::vector<BqBlock> blocks;
  std::vector<BqPiece> pieces;
  uint32_t max_src_bytes = 2;  // largest source element size: sizes the shared-memory stage
};

// ---- per-channel / per-tensor scaled fp8 (scaled_fp8.cu) -------------------------------------------
// Shared-memory stage of the row-staged kernel: a per-channel row whose source bytes (rounded up to 16)
// fit takes the one-read path.  32 KiB admits a bf16 row of K = 14336 (28 KiB) and four of K = 4096,
// stays under the 48 KiB default (no opt-in), and leaves room for 6 CTAs of 256 threads per SM.
constexpr uint32_t kSqStageBytes = 32768;
constexpr uint32_t kSqBandRows = 256;      // most rows one CTA stages (one per thread in the reduction)
constexpr uint32_t kSqTileElems = 16384;   // most elements of one two-pass tile (one CTA per pass)

// Row-staged path: a band of whole rows of one per-channel matrix.
struct alignas(8) SqBand {
  uint64_t dst;          // fp8 element (0, 0) of the band
  uint64_t scale;        // float32 scale_inv of its first row (one per row, contiguous)
  uint32_t cols;         // row length (elements == destination pitch in bytes)
  uint32_t rows;
  uint32_t piece0, n_pieces;
  uint32_t src_dtype;    // the same for every piece of the band
  uint32_t pad_;
};
static_assert(sizeof(SqBand) == 40, "SqBand is part of tsb_scaled_fp8_compile_host's output");

// A source rectangle inside one band.
struct alignas(8) SqPiece {
  uint64_t src;          // source element (row0, col0) of the piece
  int64_t src_stride;    // bytes between source rows
  uint32_t row0, col0;   // position inside the band
  uint32_t rows, cols;
  uint32_t vec;          // 1: source address, stride, column offset and width allow 16-byte accesses
  uint32_t pad_;
};
static_assert(sizeof(SqPiece) == 40, "SqPiece is part of tsb_scaled_fp8_compile_host's output");

// Two-pass path: a rectangle of one group (a per-tensor matrix or a long per-channel row), read once
// per pass by one CTA.
struct alignas(8) SqTile {
  uint64_t src;          // source element (0, 0) of the tile
  int64_t src_stride;    // bytes between source rows
  uint64_t dst;          // its fp8 element (0, 0)
  uint64_t scale;        // the group's float32 scale_inv if this tile writes it (one tile per group), else 0
  uint32_t dst_pitch;    // destination row pitch (bytes == elements)
  uint32_t rows, cols;
  uint32_t group;        // index of the group's amax word
  uint32_t src_dtype;
  uint32_t vec;          // as SqPiece::vec
};
static_assert(sizeof(SqTile) == 56, "SqTile is part of tsb_scaled_fp8_compile_host's output");

struct SqTables : PlanBytes {
  std::vector<SqBand> bands;
  std::vector<SqPiece> pieces;
  std::vector<SqTile> tiles;
  uint32_t n_groups = 0;        // amax words of the two-pass path
  uint32_t stage_bytes = 0;     // largest band stage (dynamic shared memory of the row-staged kernel)
};
struct SqLaunch {
  const SqBand* bands;
  const SqPiece* pieces;
  const SqTile* tiles;
  uint32_t* amax;  // n_groups words, cleared by the launch
  uint32_t n_bands, n_tiles, n_groups, stage_bytes;
  bool ue8m0;      // power-of-two scales (QuantPlan::ue8m0)
  bool int8;       // int8 destinations (QuantPlan::int8)
};
int launch_scaled_fp8(const SqLaunch& l, cudaStream_t stream);

// ---- dequantising pulls: scaled fp8 sources -> f32 / bf16 / f16 (dequant_fp8.cu) --------------------
constexpr uint32_t kDqTileElems = 16384;  // most elements of one tile (one CTA; 4 16-element chunks per thread)
constexpr uint32_t kDqTileRows = 256;     // most rows of one tile (one staged scale per row)

// A rectangle of one source read under one scale (block, tensor) or one scale per row (channel).
struct alignas(8) DqTile {
  uint64_t src;          // fp8 element (0, 0) of the tile
  uint64_t dst;          // its destination element
  uint64_t scale;        // float32 scale of row 0
  int64_t src_stride;    // bytes between source rows
  int64_t dst_stride;    // bytes between destination rows
  uint32_t rows, cols;
  uint16_t scale_step;   // bytes between the scales of consecutive rows: 4 * source row step (channel) or 0
  uint8_t dst_dtype;     // TSB_F32 / TSB_BF16 / TSB_F16
  uint8_t vec;           // 1: source and destination rows start 16-byte aligned (16-element chunks vectorise)
  uint32_t pad_;
};
static_assert(sizeof(DqTile) == 56, "DqTile is part of tsb_dequant_fp8_compile_host's output");

struct DqTables : PlanBytes {
  std::vector<DqTile> tiles;
};
// Validate scaled fp8 source shards (TSB_ERR_INVALID naming the source) -> their fp8 grids.
int dq_source_geoms(const tsb_dq_source_t* sources, uint64_t n_sources, std::vector<TargetGeom>* out);

// ---- requantising pulls: scaled fp8 sources -> block / channel / tensor scaled fp8 (requant_fp8.cu) -----

// Staged path, one CTA each: a 128x128 block of a block-scaled target (one group), or a band of whole rows
// of a per-channel target whose row fits kSqStageBytes (one group per row).
struct alignas(8) RqUnit {
  uint64_t dst;          // fp8 element (0, 0) of the unit
  uint64_t scale_inv;    // float32 scale_inv of the block, or of the band's first row (one per row, contiguous)
  uint32_t pitch;        // destination row pitch (bytes == elements)
  uint32_t rows, cols;
  uint32_t piece0, n_pieces;
  uint32_t per_row;      // 1: one group per row (band), 0: one group (block)
};
static_assert(sizeof(RqUnit) == 40, "RqUnit is part of tsb_requant_fp8_compile_host's output");

// A source rectangle inside one unit, read under one source scale (tensor), one per row (channel) or one per 128
// source columns (block: the rows of a piece lie in one block row of the source).
struct alignas(8) RqPiece {
  uint64_t src;          // fp8 source element (row0, col0) of the piece
  int64_t src_stride;    // bytes between source rows
  uint64_t scale;        // float32 source scale of the piece's first element
  uint32_t row0, col0;   // position inside the unit
  uint32_t rows, cols;
  uint32_t scale_step;   // bytes between the source scales of consecutive rows: 4 * row step (channel) or 0
  uint32_t vec;          // 1: source address, stride, column offset, width and column phase allow 16-byte accesses
  uint32_t col_phase;    // col_blocks: column of the piece's first element inside its source block
  uint32_t col_blocks;   // 1: the scale advances 4 bytes every 128 columns from col_phase on (block sources), else 0
};
static_assert(sizeof(RqPiece) == 56, "RqPiece is part of tsb_requant_fp8_compile_host's output");

// Two-pass path: a rectangle of one destination group (a per-tensor matrix or a long per-channel row) under
// one source scale (or one per row), read once per pass by one CTA.
struct alignas(8) RqTile {
  uint64_t src;          // fp8 source element (0, 0) of the tile
  int64_t src_stride;
  uint64_t scale;        // float32 source scale of row 0
  uint64_t dst;          // its fp8 destination element
  uint64_t scale_inv;    // the group's float32 scale_inv if this tile writes it (one tile per group), else 0
  uint32_t dst_pitch;
  uint32_t rows, cols;
  uint32_t group;        // index of the group's amax word
  uint32_t scale_step;   // as RqPiece::scale_step
  uint32_t vec;          // 1: source rows start 16-byte aligned (whole 16-element chunks vectorise)
};
static_assert(sizeof(RqTile) == 64, "RqTile is part of tsb_requant_fp8_compile_host's output");

struct RqTables : PlanBytes {
  std::vector<RqUnit> units;
  std::vector<RqPiece> pieces;
  std::vector<RqTile> tiles;
  uint32_t n_groups = 0;     // amax words of the two-pass path
  uint32_t stage_bytes = 0;  // largest unit stage (dynamic shared memory of the staged kernel)
};

// ---- source-side quantisation: live bf16/f16/f32 shards -> scaled fp8 staging (source_quant.cu) ---------
constexpr uint32_t kSrcQChunks = 4;  // 16-element chunks per thread: a unit holds at most 4 * 256 of them (a 128x128 block)

// One CTA's work: one group of a block-scaled shard (its part of a global 128x128 block), or a band of whole rows of
// a per-channel shard (one group per row) of at most kSqStageBytes source bytes and kSrcQChunks * kQuantThreads
// 16-element chunks.  Source and destination are the shard's own contiguous rows.
struct alignas(8) SrcQUnit {
  uint64_t src;          // source element (0, 0) of the unit
  uint64_t dst;          // its fp8 element
  uint64_t scale_inv;    // float32 scale_inv of the block, or of the band's first row (one per row, contiguous)
  uint32_t src_pitch;    // bytes between source rows
  uint32_t dst_pitch;    // bytes between destination rows
  uint32_t rows, cols;
  uint32_t per_row;      // 1: one group per row (band), 0: one group (block)
  uint16_t src_dtype;    // TSB_F32 / TSB_BF16 / TSB_F16
  uint16_t vec;          // 1: source address, pitch and row width allow 16-byte loads
};
static_assert(sizeof(SrcQUnit) == 48, "SrcQUnit is part of tsb_source_quant_compile_host's output");

struct SrcQTables : PlanBytes {
  std::vector<SrcQUnit> units;  // grouped by source dtype: bf16, then f16, then f32 (one kernel launch each)
  std::vector<SqTile> tiles;    // two-pass path: per-tensor groups and long per-channel rows
  uint32_t n_groups = 0;        // amax words of the two-pass path
  uint32_t n_units[3] = {};     // units per source dtype, in the order above
  uint32_t unit_bytes = 0;      // largest unit's source bytes
};

}  // namespace tsb
