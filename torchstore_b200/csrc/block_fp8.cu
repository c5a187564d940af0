// Block-scaled FP8 pulls (sm_90a, H100): gather bf16/f16/f32 source rectangles into float8_e4m3fn
// destinations stored the way DeepSeek-V3 / vLLM (weight_block_size=[128, 128]) keep FP8 weights, one
// float32 scale_inv per 128x128 block, quantising on the way.  Each source byte is read once.
//
// Host side: the plan compiler maps every rect onto its target's [batch, rows, cols] grid, cuts it
// at block boundaries into pieces, sorts the pieces by block and checks that they tile every block
// exactly (an uncovered element would leave the block's amax undefined).
// Device side: one CTA of 256 threads per block.
//   phase 1  the block's pieces (from any shard, local or peer-mapped) land in shared memory in their
//            source dtype, 16-byte loads where address, stride and width allow it, and every thread
//            folds |x| into a running max as the data arrives.  |x| is compared as an integer (sign
//            bit cleared): for non-negative floats that orders finite < Inf < NaN, so a NaN anywhere
//            makes the block's amax NaN (fmaxf would drop it).
//   reduce   warp max, then one thread: amax_c = max(amax, 1e-4f), scale = 448 / amax_c and
//            scale_inv = amax_c / 448, both correctly rounded (__fdiv_rn); with TSB_QUANT_UE8M0 scale_inv is
//            rounded up to a power of two and scale = 1 / scale_inv (fp8_quant.cuh).
//   phase 2  shared -> e4m3fn: x * scale (__fmul_rn), torch-exact narrowing (fp8_cvt.cuh), 16
//            destination bytes per thread and step (one STG.128 when aligned, byte stores at ragged edges).
// int8 destinations (TSB_I8 rects) run the same kernel with the int8 format of fp8_quant.cuh: scale step 127
// instead of 448, and a round-to-nearest-even saturating int8 narrowing (NaN -> 0).  The tables are the same.

#include <algorithm>
#include <atomic>
#include <cstring>

#include "fp8_quant.cuh"
#include "tsb_internal.h"

namespace tsb {

uint32_t quant_src_bytes(uint32_t dt) {
  switch (dt) {
    case TSB_F32: return 4;
    case TSB_BF16: case TSB_F16: return 2;
    default: return 0;
  }
}

namespace {

// A dim of a rect: extent, the step on the side that is not the fp8 grid (ss), the step on the grid (ds).
struct Dim {
  int64_t e, ss, ds;
};

// What differs between mapping a rect by its destination (quantising pulls) or by its source
// (dequantising pulls).
struct Side {
  bool by_src;            // the fp8 grid is the rect's source
  const char* no_grid;    // the grid pointer lies in no grid
  const char* not_a_box;  // its grid strides describe no box
  int contig_code;        // the other side's columns are strided
  const char* contig;
  const char* unaligned;  // the other side is not aligned to its element size
};

constexpr Side kByDst{false, "dst is inside no target", "its destination strides do not describe a box of the target",
                      TSB_ERR_UNSUPPORTED, "scaled fp8 pulls read contiguous source rows",
                      "source not aligned to its element size"};
constexpr Side kBySrc{true, "src is inside no source", "its source strides do not describe a box of the source",
                      TSB_ERR_INVALID, "dequantising pulls write contiguous destination rows",
                      "destination not aligned to its element size"};

// The mapping of rect_boxes / rect_source_boxes once the dtypes are checked; `es` is the element size
// of the side that is not the grid.
int map_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* targets, uint64_t n_targets, const Side& side,
              uint32_t es, std::vector<TargetBox>* out) {
  const std::string where = "rect " + std::to_string(index) + ": ";
  std::vector<Dim> work;
  for (uint32_t i = 0; i < in.ndim; ++i) {
    if (in.extent[i] < 0) return fail(TSB_ERR_INVALID, where + "negative extent");
    if (in.extent[i] == 0) return TSB_OK;
    if (in.extent[i] > 1)
      work.push_back(side.by_src ? Dim{in.extent[i], in.dst_stride[i], in.src_stride[i]}
                                 : Dim{in.extent[i], in.src_stride[i], in.dst_stride[i]});
  }
  if (in.src == 0 || in.dst == 0) return fail(TSB_ERR_INVALID, where + "NULL src/dst");
  const uint64_t grid_ptr = side.by_src ? in.src : in.dst, other_ptr = side.by_src ? in.dst : in.src;
  uint64_t t = 0;
  while (t < n_targets && !(grid_ptr >= targets[t].dst && grid_ptr - targets[t].dst < targets[t].batch * targets[t].rows * targets[t].cols)) ++t;
  if (t == n_targets) return fail(TSB_ERR_INVALID, where + side.no_grid);
  const int64_t R = static_cast<int64_t>(targets[t].rows), C = static_cast<int64_t>(targets[t].cols);
  const int64_t B = static_cast<int64_t>(targets[t].batch);
  const uint64_t o = grid_ptr - targets[t].dst;
  const int64_t b0 = static_cast<int64_t>(o / (R * C)), r0 = static_cast<int64_t>(o % (R * C)) / C, c0 = static_cast<int64_t>(o % C);
  // Classify every dim by its grid step: columns (1), rows (C) or whole matrices (multiple of
  // R*C).  A collapsed dim that runs past the end of a row (or of a matrix) is split back.
  int64_t er = 1, ec = 1, row_ss = 0, col_ss = es, rstep = 1;
  bool have_row = false, have_col = false;
  std::vector<Dim> batch;
  const std::string bad = where + side.not_a_box;
  while (!work.empty()) {
    const Dim d = work.back();
    work.pop_back();
    if (d.ds == 1 && C > 1) {
      if (c0 + d.e <= C) {
        if (have_col) return fail(TSB_ERR_INVALID, bad);
        have_col = true;
        ec = d.e;
        col_ss = d.ss;
      } else if (c0 == 0 && d.e % C == 0) {
        work.push_back({d.e / C, d.ss * C, C});
        work.push_back({C, d.ss, 1});
      } else {
        return fail(TSB_ERR_INVALID, bad);
      }
    } else if (d.ds == C && R > 1) {
      if (r0 + d.e <= R) {
        if (have_row) return fail(TSB_ERR_INVALID, bad);
        have_row = true;
        er = d.e;
        row_ss = d.ss;
      } else if (r0 == 0 && d.e % R == 0) {
        work.push_back({d.e / R, d.ss * R, R * C});
        work.push_back({R, d.ss, C});
      } else {
        return fail(TSB_ERR_INVALID, bad);
      }
    } else if (side.by_src && d.ds == 2 * C && r0 + 2 * (d.e - 1) < R) {  // a rotary head half: every other row
      if (have_row) return fail(TSB_ERR_INVALID, bad);
      have_row = true;
      er = d.e;
      row_ss = d.ss;
      rstep = 2;
    } else if (d.ds > 0 && d.ds % (R * C) == 0) {
      batch.push_back({d.e, d.ss, d.ds / (R * C)});
    } else {
      return fail(TSB_ERR_INVALID, bad);
    }
  }
  int64_t b_last = b0;
  for (const Dim& d : batch) b_last += (d.e - 1) * d.ds;
  if (b_last >= B) return fail(TSB_ERR_INVALID, bad);
  if (have_col && col_ss != static_cast<int64_t>(es)) return fail(side.contig_code, where + side.contig);
  if (other_ptr % es || row_ss % es) return fail(TSB_ERR_INVALID, where + side.unaligned);
  for (const Dim& d : batch)
    if (d.ss % es) return fail(TSB_ERR_INVALID, where + side.unaligned);
  // one box per combination of the batch dims
  std::vector<int64_t> k(batch.size(), 0);
  while (true) {
    int64_t b = b0, so = 0;
    for (size_t i = 0; i < batch.size(); ++i) {
      b += k[i] * batch[i].ds;
      so += k[i] * batch[i].ss;
    }
    out->push_back({other_ptr + static_cast<uint64_t>(so), row_ss, t, static_cast<uint64_t>(b), static_cast<uint64_t>(r0),
                    static_cast<uint64_t>(c0), static_cast<uint64_t>(er), static_cast<uint64_t>(ec),
                    side.by_src ? in.dst_dtype : in.src_dtype, in.src_device, static_cast<uint32_t>(rstep)});
    size_t i = batch.size();
    while (i > 0 && ++k[i - 1] == batch[i - 1].e) k[--i] = 0;
    if (i == 0) break;
  }
  return TSB_OK;
}

}  // namespace

int check_grid(const GridRules& rules, uint64_t index, const Grid& g) {
  const std::string where = std::string(rules.noun) + " " + std::to_string(index) + ": ";
  if (g.null) return fail(TSB_ERR_INVALID, where + rules.null_msg);
  if (!g.batch || !g.rows || !g.cols) return fail(TSB_ERR_INVALID, where + "empty " + rules.noun);
  if (g.base % g.es) return fail(TSB_ERR_INVALID, where + rules.base_name + " is not aligned to its element size");
  if (g.scale % 4) return fail(TSB_ERR_INVALID, where + rules.scale_name + " is not 4-byte aligned");
  if (rules.granularities && !(g.granularity < 32 && (rules.granularities >> g.granularity) & 1)) {
    // "must be A or B" / "must be A, B or C", in the order block, channel, tensor
    const uint32_t codes[] = {TSB_SCALE_PER_BLOCK, TSB_SCALE_PER_CHANNEL, TSB_SCALE_PER_TENSOR};
    const char* const code_names[] = {"TSB_SCALE_PER_BLOCK", "TSB_SCALE_PER_CHANNEL", "TSB_SCALE_PER_TENSOR"};
    std::vector<std::string> names;
    for (int k = 0; k < 3; ++k)
      if ((rules.granularities >> codes[k]) & 1) names.push_back(code_names[k]);
    std::string list = names[0];
    for (size_t i = 1; i < names.size(); ++i) list += (i + 1 == names.size() ? " or " : ", ") + names[i];
    return fail(TSB_ERR_INVALID, where + "granularity must be " + list + ", not " + std::to_string(g.granularity));
  }
  if (g.pad) return fail(TSB_ERR_INVALID, where + "pad must be 0");
  if (g.cols >= rules.max_cols || g.rows >= (1ull << 31) || g.batch >= (1ull << 31) || g.batch * g.rows >= (1ull << 40) / g.cols ||
      g.row0 >= (1ull << 40) || g.col0 >= (1ull << 40))
    return fail(TSB_ERR_INVALID, where + rules.noun + " too large");
  return TSB_OK;
}

int rect_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* targets, uint64_t n_targets,
               std::vector<TargetBox>* out) {
  const std::string where = "rect " + std::to_string(index) + ": ";
  if (in.ndim < 1 || in.ndim > TSB_MAX_DIMS) return fail(TSB_ERR_INVALID, where + "ndim must be in [1, 6]");
  const uint32_t es = quant_src_bytes(in.src_dtype);
  if (!es) return fail(TSB_ERR_UNSUPPORTED, where + "scaled fp8 pulls read f32, bf16 or f16 sources");
  if (in.dst_dtype != TSB_F8E4M3 && in.dst_dtype != TSB_I8)
    return fail(TSB_ERR_UNSUPPORTED, where + "scaled destinations are float8_e4m3fn or int8");
  return map_boxes(in, index, targets, n_targets, kByDst, es, out);
}

int quant_dst_int8(const tsb_rect_t* rects, uint64_t n, bool ue8m0, bool* int8) {
  *int8 = n && rects[0].dst_dtype == TSB_I8;
  for (uint64_t i = 1; i < n; ++i)
    if ((rects[i].dst_dtype == TSB_I8) != *int8)
      return fail(TSB_ERR_INVALID, "rect " + std::to_string(i) + ": the rects of one plan write one destination dtype, "
                                   "float8_e4m3fn or int8");
  if (*int8 && ue8m0) return fail(TSB_ERR_INVALID, "int8 destinations take float32 scales: TSB_QUANT_UE8M0 is refused");
  return TSB_OK;
}

int rect_source_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* grids, uint64_t n_grids,
                      std::vector<TargetBox>* out) {
  const std::string where = "rect " + std::to_string(index) + ": ";
  if (in.ndim < 1 || in.ndim > TSB_MAX_DIMS) return fail(TSB_ERR_INVALID, where + "ndim must be in [1, 6]");
  if (in.src_dtype != TSB_F8E4M3 && in.src_dtype != TSB_I8)
    return fail(TSB_ERR_INVALID, where + "dequantising pulls read float8_e4m3fn or int8 sources");
  const uint32_t es = quant_src_bytes(in.dst_dtype);
  if (!es) return fail(TSB_ERR_INVALID, where + "dequantising pulls write f32, bf16 or f16 destinations");
  return map_boxes(in, index, grids, n_grids, kBySrc, es, out);
}

int rect_requant_boxes(const tsb_rect_t& in, uint64_t index, const TargetGeom* targets, uint64_t n_targets,
                       std::vector<TargetBox>* out) {
  const std::string where = "rect " + std::to_string(index) + ": ";
  if (in.ndim < 1 || in.ndim > TSB_MAX_DIMS) return fail(TSB_ERR_INVALID, where + "ndim must be in [1, 6]");
  if (in.src_dtype != TSB_F8E4M3 || in.dst_dtype != TSB_F8E4M3)
    return fail(TSB_ERR_INVALID, where + "requantising pulls read and write float8_e4m3fn");
  return map_boxes(in, index, targets, n_targets, kByDst, 1, out);
}

namespace {

constexpr GridRules kTargetRules{"target", "NULL dst or scale_inv", "dst", "scale_inv", 0, 1ull << 31};

int block_fp8_compile(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets, uint64_t n_targets,
                      BqTables* out) {
  if ((n && !rects) || (n_targets && !targets)) return fail(TSB_ERR_INVALID, "block_fp8: NULL rects or targets");
  // block index of every target's first block
  std::vector<uint64_t> base(n_targets + 1, 0);
  for (uint64_t t = 0; t < n_targets; ++t) {
    const tsb_bq_target_t& T = targets[t];
    int st = check_grid(kTargetRules, t, {T.dst, T.scale_inv, T.batch, T.rows, T.cols, 0, 0, 1, 0, 0, !T.dst || !T.scale_inv});
    if (st) return st;
    const uint64_t nbr = (T.rows + kBqBlock - 1) / kBqBlock, nbc = (T.cols + kBqBlock - 1) / kBqBlock;
    base[t + 1] = base[t] + T.batch * nbr * nbc;
    out->payload_bytes += T.batch * T.rows * T.cols + 4 * T.batch * nbr * nbc;
  }
  if (base[n_targets] >= (1ull << 31)) return fail(TSB_ERR_UNSUPPORTED, "block_fp8: more than 2^31 blocks");
  std::vector<TargetGeom> geom(n_targets);
  for (uint64_t t = 0; t < n_targets; ++t) geom[t] = {targets[t].dst, targets[t].batch, targets[t].rows, targets[t].cols};
  std::vector<TargetBox> boxes;
  for (uint64_t i = 0; i < n; ++i) {
    int st = rect_boxes(rects[i], i, geom.data(), n_targets, &boxes);
    if (st) return st;
  }
  struct Keyed {
    uint64_t block;
    uint32_t dtype;
    BqPiece piece;
  };
  std::vector<Keyed> pieces;
  for (const TargetBox& x : boxes) {
    const tsb_bq_target_t& T = targets[x.target];
    const uint64_t nbr = (T.rows + kBqBlock - 1) / kBqBlock, nbc = (T.cols + kBqBlock - 1) / kBqBlock;
    const uint32_t es = quant_src_bytes(x.dtype);
    for (uint64_t br = x.r0 / kBqBlock; br <= (x.r0 + x.er - 1) / kBqBlock; ++br) {
      const uint64_t pr0 = std::max<uint64_t>(x.r0, br * kBqBlock), pr1 = std::min<uint64_t>(x.r0 + x.er, (br + 1) * kBqBlock);
      for (uint64_t bc = x.c0 / kBqBlock; bc <= (x.c0 + x.ec - 1) / kBqBlock; ++bc) {
        const uint64_t pc0 = std::max<uint64_t>(x.c0, bc * kBqBlock), pc1 = std::min<uint64_t>(x.c0 + x.ec, (bc + 1) * kBqBlock);
        BqPiece p;
        memset(&p, 0, sizeof(p));
        p.src = x.src + (pr0 - x.r0) * x.row_stride + (pc0 - x.c0) * es;
        p.src_stride = x.row_stride;
        p.row0 = static_cast<uint16_t>(pr0 - br * kBqBlock);
        p.col0 = static_cast<uint16_t>(pc0 - bc * kBqBlock);
        p.rows = static_cast<uint16_t>(pr1 - pr0);
        p.cols = static_cast<uint16_t>(pc1 - pc0);
        p.vec = (vec_ok(p.src, p.src_stride, p.rows, p.cols, es) && (p.col0 * es) % 16 == 0) ? 1u : 0u;
        pieces.push_back({base[x.target] + (x.b * nbr + br) * nbc + bc, x.dtype, p});
        out->read(static_cast<uint64_t>(p.rows) * p.cols * es, x.src_device, device);
        out->max_src_bytes = std::max(out->max_src_bytes, es);
      }
    }
  }
  std::stable_sort(pieces.begin(), pieces.end(), [](const Keyed& a, const Keyed& b) { return a.block < b.block; });
  out->blocks.resize(base[n_targets]);
  out->pieces.resize(pieces.size());
  size_t pi = 0;
  uint64_t t = 0;
  for (uint64_t blk = 0; blk < base[n_targets]; ++blk) {
    while (blk >= base[t + 1]) ++t;
    const tsb_bq_target_t& T = targets[t];
    const uint64_t nbr = (T.rows + kBqBlock - 1) / kBqBlock, nbc = (T.cols + kBqBlock - 1) / kBqBlock;
    const uint64_t local = blk - base[t], b = local / (nbr * nbc), br = (local / nbc) % nbr, bc = local % nbc;
    const uint32_t rows = static_cast<uint32_t>(std::min<uint64_t>(kBqBlock, T.rows - br * kBqBlock));
    const uint32_t cols = static_cast<uint32_t>(std::min<uint64_t>(kBqBlock, T.cols - bc * kBqBlock));
    const size_t first = pi;
    uint64_t area = 0;
    while (pi < pieces.size() && pieces[pi].block == blk) {
      area += static_cast<uint64_t>(pieces[pi].piece.rows) * pieces[pi].piece.cols;
      out->pieces[pi] = pieces[pi].piece;
      ++pi;
    }
    const std::string where = "target " + std::to_string(t) + " block (" + std::to_string(b) + ", " + std::to_string(br) + ", " +
                              std::to_string(bc) + "): ";
    if (area != static_cast<uint64_t>(rows) * cols)
      return fail(TSB_ERR_INVALID, where + "its elements are not all written exactly once (" + std::to_string(area) + " of " +
                                       std::to_string(rows * cols) + ")");
    for (size_t i = first + 1; i < pi; ++i)
      if (pieces[i].dtype != pieces[first].dtype) return fail(TSB_ERR_UNSUPPORTED, where + "sources of different dtypes");
    if (pi - first > 1) {  // equal area: exact tiling unless two pieces overlap
      uint64_t mask[kBqBlock][2] = {};
      for (size_t i = first; i < pi; ++i) {
        const BqPiece& p = out->pieces[i];
        uint64_t m[2] = {0, 0};
        for (uint32_t c = p.col0; c < static_cast<uint32_t>(p.col0) + p.cols; ++c) m[c >> 6] |= 1ull << (c & 63);
        for (uint32_t r = p.row0; r < static_cast<uint32_t>(p.row0) + p.rows; ++r) {
          if ((mask[r][0] & m[0]) | (mask[r][1] & m[1]))
            return fail(TSB_ERR_INVALID, where + "its elements are not all written exactly once (overlap)");
          mask[r][0] |= m[0];
          mask[r][1] |= m[1];
        }
      }
    }
    BqBlock& o = out->blocks[blk];
    memset(&o, 0, sizeof(o));
    o.dst = T.dst + b * T.rows * T.cols + br * kBqBlock * T.cols + bc * kBqBlock;
    o.scale = T.scale_inv + 4 * ((b * nbr + br) * nbc + bc);
    o.pitch = static_cast<uint32_t>(T.cols);
    o.rows = static_cast<uint16_t>(rows);
    o.cols = static_cast<uint16_t>(cols);
    o.piece0 = static_cast<uint32_t>(first);
    o.n_pieces = static_cast<uint16_t>(pi - first);
    o.src_dtype = static_cast<uint16_t>(pieces[first].dtype);
  }
  return TSB_OK;
}

// Phase 1: pieces -> shared memory (source dtype, block row pitch 128 elements); returns this
// thread's max |x| bits.
template <uint32_t DT>
__device__ __forceinline__ uint32_t stage_block(const BqBlock& blk, const BqPiece* __restrict__ pieces, unsigned char* smem) {
  constexpr uint32_t es = Src<DT>::kBytes;
  constexpr uint32_t spitch = kBqBlock * es;
  uint32_t m = 0;
  for (uint32_t q = 0; q < blk.n_pieces; ++q) {
    const BqPiece p = pieces[blk.piece0 + q];
    const char* src = reinterpret_cast<const char*>(p.src);
    unsigned char* s0 = smem + p.row0 * spitch + p.col0 * es;
    if (p.vec) {
      const uint32_t upr = p.cols * es / 16;  // 16-byte units per row
      const uint32_t total = p.rows * upr;
      for (uint32_t i = threadIdx.x; i < total; i += kQuantThreads * kUnroll) {
        uint4 v[kUnroll];
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
          const uint32_t idx = i + k * kQuantThreads;
          if (idx < total) {
            const uint32_t r = idx / upr, c = idx - r * upr;
            v[k] = ldg16(src + static_cast<int64_t>(r) * p.src_stride + c * 16);
          }
        }
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
          const uint32_t idx = i + k * kQuantThreads;
          if (idx < total) {
            const uint32_t r = idx / upr, c = idx - r * upr;
            m = fold16<DT>(m, v[k]);
            *reinterpret_cast<uint4*>(s0 + r * spitch + c * 16) = v[k];
          }
        }
      }
    } else {
      const uint32_t total = static_cast<uint32_t>(p.rows) * p.cols;
      for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
        const uint32_t r = idx / p.cols, c = idx - r * p.cols;
        const char* a = src + static_cast<int64_t>(r) * p.src_stride + c * es;
        unsigned char* s = s0 + r * spitch + c * es;
        if (es == 4) {
          const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(a));
          m = max(m, abs_bits(w));
          *reinterpret_cast<uint32_t*>(s) = w;
        } else {
          const unsigned short h = __ldg(reinterpret_cast<const unsigned short*>(a));
          m = max(m, abs_bits(Src<DT>::f32(h)));
          *reinterpret_cast<unsigned short*>(s) = h;
        }
      }
    }
  }
  return m;
}

// Phase 2: shared memory -> the destination format, 16 destination bytes per thread and step.
template <uint32_t DT, class Out>
__device__ __forceinline__ void quantise_block(const BqBlock& blk, const unsigned char* smem, float scale) {
  constexpr uint32_t es = Src<DT>::kBytes;
  constexpr uint32_t spitch = kBqBlock * es;
  const uint32_t cpr = (blk.cols + 15u) / 16u;
  const uint32_t total = blk.rows * cpr;
  for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
    const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
    const unsigned char* s = smem + r * spitch + c * es;
    char* d = reinterpret_cast<char*>(blk.dst) + static_cast<uint64_t>(r) * blk.pitch + c;
    const uint32_t nvalid = min(16u, static_cast<uint32_t>(blk.cols) - c);
    uint32_t f[16], o[4];
    load16_shared<DT>(s, nvalid, f);
    Out::narrow(f, scale, o);
    store16(d, nvalid, o);
  }
}

template <uint32_t DT, class Out>
__device__ __forceinline__ void run_block(const BqBlock& blk, const BqPiece* pieces, unsigned char* smem, uint32_t* s_red,
                                          float* s_scale) {
  cta_max(stage_block<DT>(blk, pieces, smem), s_red, [&](uint32_t a) {
    float scale, scale_inv;
    Out::scales(a, &scale, &scale_inv);
    *s_scale = scale;
    *reinterpret_cast<float*>(blk.scale) = scale_inv;
  });
  __syncthreads();
  quantise_block<DT, Out>(blk, smem, *s_scale);
}

// The CTA's block in destination format Out (fp8_quant.cuh), the body of the kernels below
template <class Out>
__device__ __forceinline__ void quantise_blocks(const BqBlock* __restrict__ blocks, const BqPiece* __restrict__ pieces,
                                                unsigned char* stage, uint32_t* s_red, float* s_scale) {
  const BqBlock blk = blocks[blockIdx.x];
  switch (blk.src_dtype) {
    case TSB_BF16: run_block<TSB_BF16, Out>(blk, pieces, stage, s_red, s_scale); break;
    case TSB_F16: run_block<TSB_F16, Out>(blk, pieces, stage, s_red, s_scale); break;
    default: run_block<TSB_F32, Out>(blk, pieces, stage, s_red, s_scale); break;
  }
}

// kUe8m0: power-of-two scales (TSB_QUANT_UE8M0)
template <bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads, 6) block_fp8_kernel(const BqBlock* __restrict__ blocks, const BqPiece* __restrict__ pieces) {
  extern __shared__ __align__(16) unsigned char stage[];
  __shared__ uint32_t s_red[kQuantThreads / 32];
  __shared__ float s_scale;
  quantise_blocks<E4m3Out<kUe8m0>>(blocks, pieces, stage, s_red, &s_scale);
}

// int8 destinations (TSB_I8)
__global__ void __launch_bounds__(kQuantThreads, 6) block_int8_kernel(const BqBlock* __restrict__ blocks, const BqPiece* __restrict__ pieces) {
  extern __shared__ __align__(16) unsigned char stage[];
  __shared__ uint32_t s_red[kQuantThreads / 32];
  __shared__ float s_scale;
  quantise_blocks<I8Out>(blocks, pieces, stage, s_red, &s_scale);
}

cudaError_t prepare() {
  // an f32 stage (64 KiB) exceeds the 48 KiB default; the attribute is per device (context)
  static std::atomic<uint64_t> prepared{0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const uint64_t bit = 1ull << (dev & 63);
  if (prepared.load(std::memory_order_acquire) & bit) return cudaSuccess;
  for (auto kernel : {block_fp8_kernel<false>, block_fp8_kernel<true>, block_int8_kernel}) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kBqBlock * kBqBlock * 4));
    if (e != cudaSuccess) return e;
  }
  prepared.fetch_or(bit, std::memory_order_release);
  return e;
}

int launch_block_fp8(const BqBlock* blocks, const BqPiece* pieces, uint32_t n_blocks, uint32_t max_src_bytes, bool ue8m0,
                     bool int8, cudaStream_t stream) {
  const cudaError_t e = prepare();
  if (e != cudaSuccess) return cuda_fail(e, "block_fp8_kernel launch");
  const auto kernel = int8 ? block_int8_kernel : ue8m0 ? block_fp8_kernel<true> : block_fp8_kernel<false>;
  kernel<<<n_blocks, kQuantThreads, kBqBlock * kBqBlock * max_src_bytes, stream>>>(blocks, pieces);
  return launched(int8 ? "block_int8_kernel launch" : "block_fp8_kernel launch");
}

// d = {BqBlock table | BqPiece table}, one CTA per block
int block_fp8_plan(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets, uint64_t n_targets,
                   QuantPlan* q) {
  BqTables tb;
  int st = block_fp8_compile(device, rects, n, targets, n_targets, &tb);
  if (st || (st = quant_dst_int8(rects, n, q->ue8m0, &q->int8))) return st;
  q->add(tb.blocks);
  const size_t pieces = q->add(tb.pieces);
  q->seal(0);
  q->describe(n, static_cast<uint32_t>(tb.blocks.size()), kBqBlock * kBqBlock, tb);
  q->launch = [pieces, n_blocks = static_cast<uint32_t>(tb.blocks.size()), es = tb.max_src_bytes, ue8m0 = q->ue8m0,
               int8 = q->int8](char* d, cudaStream_t s) {
    return launch_block_fp8(reinterpret_cast<const BqBlock*>(d), reinterpret_cast<const BqPiece*>(d + pieces), n_blocks, es, ue8m0,
                            int8, s);
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_block_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets,
                                         uint64_t n_targets, uint32_t flags, tsb_plan_t* out) {
  return quant_plan_create("tsb_block_fp8_plan_create", device, flags, TSB_QUANT_UE8M0, out,
                           [&](QuantPlan* q) { return block_fp8_plan(device, rects, n, targets, n_targets, q); });
}

extern "C" int tsb_block_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets,
                                          uint64_t n_targets, uint32_t flags, void* out_blocks, uint64_t block_cap,
                                          uint64_t* out_n_blocks, void* out_pieces, uint64_t piece_cap, uint64_t* out_n_pieces) {
  return quant_compile_host("tsb_block_fp8_compile_host", flags, TSB_QUANT_UE8M0,
                            [&](QuantPlan* q) { return block_fp8_plan(device, rects, n, targets, n_targets, q); },
                            {{out_blocks, block_cap, out_n_blocks, "out_blocks"}, {out_pieces, piece_cap, out_n_pieces, "out_pieces"}},
                            nullptr);
}
