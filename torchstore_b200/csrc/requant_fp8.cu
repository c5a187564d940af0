// Requantising pulls (sm_90a, H100): gather block-, channel- or tensor-scaled float8_e4m3fn source
// rectangles into block-, channel- or tensor-scaled float8_e4m3fn destinations.  Every element is first
// dequantised exactly as a dequantising pull into f32 would write it, x = f32(q) * s_src (dequant_fp8.cu),
// then quantised with the destination's formula as if x were an f32 source (block_fp8.cu, scaled_fp8.cu).
// The result equals that two-step route byte for byte, with no f32 temporary and one read of each source
// byte (two for per-tensor destinations).
//
// Host side: the plan compiler maps every rect onto its target's [batch, rows, cols] grid (rect_boxes), finds
// its source shard and the (matrix, row, column) of its first byte there, and cuts the box into segments
// whose rows share their source scales: block sources are cut at block rows (128, anchored at the global
// origin through the shard's (row0, col0)) and their scale steps 4 bytes every 128 columns; a per-channel
// segment carries the scale of its first row and a 4-byte step per row; per tensor the only cuts are the
// shard's matrices.  A row sweep per destination matrix then checks that the
// segments cover every element exactly once and the segments are cut again at the destination's groups:
//   block targets                      -> one unit per 128x128 block (staged kernel)
//   per-channel rows of <= 32 KiB      -> units of whole rows (staged kernel)
//   per-tensor matrices, longer rows   -> tiles of at most kSqTileElems elements (two-pass kernels)
// Device side:
//   requant_fp8_staged_kernel  one 256-thread CTA per unit.  Phase 1: the unit's pieces land in shared memory
//                              as fp8 bytes (16-byte loads where aligned); every chunk is dequantised on the
//                              fly and |x| folded into the block's max or its row's.  Phase 2: x recomputed
//                              from the staged bytes and the source scale, narrowed with the unit's scale
//                              (one STG.128 per 16 destination bytes where aligned).
//   requant_fp8_amax_kernel    pass 1 of a tile: max |x| over the tile, one atomicMax on its group's word.
//   requant_fp8_quant_kernel   pass 2: the group's scale, the tile re-read and quantised straight to HBM.
// The amax words live in the plan's allocation and are cleared on the launch stream before pass 1.

#include <algorithm>
#include <cstring>

#include "fp8_quant.cuh"
#include "tsb_internal.h"

namespace tsb {

namespace {

// A box of a destination matrix read from one source under one scale, or one per row.
struct Seg {
  uint64_t t, b, r0, c0, er, ec;  // target, matrix, first row and column, extent
  uint64_t src;                   // fp8 source byte of (r0, c0)
  int64_t stride;                 // source bytes between rows
  uint64_t scale;                 // float32 source scale of (r0, c0)
  uint32_t step;                  // bytes between the scales of consecutive rows (channel sources), else 0
  uint32_t cph;                   // block sources: column of c0 inside its source block (the scale steps 4 bytes
  uint32_t cblk;                  // every 128 columns from there; cblk = 1), else 0
  int32_t src_device;
};

// Locate box x (of rect `index`) in its source shard and cut it at the source's scale-group rows (block sources
// keep their rows whole: the scale steps along the columns).
int source_segments(const TargetBox& x, uint64_t index, const tsb_dq_source_t* sources, uint64_t n_sources,
                    std::vector<Seg>* out) {
  const std::string where = "rect " + std::to_string(index) + ": ";
  uint64_t s = 0;
  while (s < n_sources && !(x.src >= sources[s].src && x.src - sources[s].src < sources[s].batch * sources[s].rows * sources[s].cols)) ++s;
  if (s == n_sources) return fail(TSB_ERR_INVALID, where + "src is inside no source");
  const tsb_dq_source_t& S = sources[s];
  const std::string src_name = "source " + std::to_string(s);
  const uint64_t o = x.src - S.src, L0 = o / S.cols, j0 = o % S.cols;  // L: row index over the whole shard
  if (j0 + x.ec > S.cols) return fail(TSB_ERR_INVALID, where + "its source rows cross a row of " + src_name);
  uint64_t rk = 0;  // source rows per destination row
  if (x.er > 1) {
    if (x.row_stride <= 0 || x.row_stride % static_cast<int64_t>(S.cols))
      return fail(TSB_ERR_INVALID, where + "its source rows are not rows of " + src_name);
    rk = static_cast<uint64_t>(x.row_stride) / S.cols;
  }
  if (L0 + (x.er - 1) * rk >= S.batch * S.rows) return fail(TSB_ERR_INVALID, where + "it runs past the end of " + src_name);
  const bool block = S.granularity == TSB_SCALE_PER_BLOCK, channel = S.granularity == TSB_SCALE_PER_CHANNEL;
  const uint64_t br0 = S.row0 / kBqBlock, bc0 = S.col0 / kBqBlock;
  const uint64_t nbr = (S.row0 + S.rows + kBqBlock - 1) / kBqBlock - br0, nbc = (S.col0 + S.cols + kBqBlock - 1) / kBqBlock - bc0;
  for (uint64_t y = 0; y < x.er;) {
    const uint64_t L = L0 + y * rk, sb = L / S.rows, i = L % S.rows;
    uint64_t n = x.er - y;  // rows under the same source group
    if (!channel && rk) {
      const uint64_t lim = block ? std::min(S.rows, ((S.row0 + i) / kBqBlock + 1) * kBqBlock - S.row0) : S.rows;
      n = std::min(n, (lim - i + rk - 1) / rk);
    }
    uint64_t scale;
    if (block)
      scale = S.scale + 4 * ((sb * nbr + (S.row0 + i) / kBqBlock - br0) * nbc + (S.col0 + j0) / kBqBlock - bc0);
    else if (channel)
      scale = S.scale + 4 * L;
    else
      scale = S.scale + 4 * sb;
    out->push_back({x.target, x.b, x.r0 + y, x.c0, n, x.ec, x.src + y * x.row_stride, x.row_stride, scale,
                    channel ? static_cast<uint32_t>(4 * rk) : 0u, block ? static_cast<uint32_t>((S.col0 + j0) % kBqBlock) : 0u,
                    block ? 1u : 0u, x.src_device});
    y += n;
  }
  return TSB_OK;
}

struct Compiler {
  int device;
  const tsb_sq_target_t* targets;
  RqTables* out;

  void count(uint64_t elems, const Seg& x) { out->read(elems, x.src_device, device); }

  // rows [y0, y0 + h) and columns [c0, c0 + w) of segment x as a piece at (row0, col0) of a unit
  void piece(const Seg& x, uint64_t y0, uint64_t h, uint64_t c0, uint64_t w, uint64_t row0, uint64_t col0) {
    RqPiece p;
    memset(&p, 0, sizeof(p));
    const uint64_t j = x.cph + (c0 - x.c0);  // column inside the segment's first source block
    p.src = x.src + (y0 - x.r0) * x.stride + (c0 - x.c0);
    p.src_stride = x.stride;
    p.scale = x.scale + (y0 - x.r0) * x.step + (x.cblk ? 4 * (j / kBqBlock) : 0);
    p.scale_step = x.step;
    p.col_phase = x.cblk ? static_cast<uint32_t>(j % kBqBlock) : 0u;
    p.col_blocks = x.cblk;
    p.row0 = static_cast<uint32_t>(row0);
    p.col0 = static_cast<uint32_t>(col0);
    p.rows = static_cast<uint32_t>(h);
    p.cols = static_cast<uint32_t>(w);
    p.vec = (vec_ok(p.src, p.src_stride, h, w, 1) && col0 % 16 == 0 && p.col_phase % 16 == 0) ? 1u : 0u;
    out->pieces.push_back(p);
    count(h * w, x);
  }

  void unit(uint64_t dst, uint64_t scale_inv, uint64_t pitch, uint64_t rows, uint64_t cols, size_t piece0, bool per_row) {
    RqUnit u;
    memset(&u, 0, sizeof(u));
    u.dst = dst;
    u.scale_inv = scale_inv;
    u.pitch = static_cast<uint32_t>(pitch);
    u.rows = static_cast<uint32_t>(rows);
    u.cols = static_cast<uint32_t>(cols);
    u.piece0 = static_cast<uint32_t>(piece0);
    u.n_pieces = static_cast<uint32_t>(out->pieces.size() - piece0);
    u.per_row = per_row ? 1u : 0u;
    out->units.push_back(u);
    out->stage_bytes = std::max(out->stage_bytes, static_cast<uint32_t>(rows) * round16(static_cast<uint32_t>(cols)));
  }

  // rows [y0, y0 + h) of segment x as two-pass tiles of group g; the tile holding the group's first element
  // writes `scale_inv`
  void tiles(const Seg& x, uint64_t y0, uint64_t h, uint32_t g, bool first_row, uint64_t scale_inv) {
    const tsb_sq_target_t& T = targets[x.t];
    const uint64_t w = x.ec;
    for (uint64_t c = 0; c < w;) {  // column runs of one source scale, at most kSqTileElems wide
      uint64_t c1 = std::min<uint64_t>(w, c + kSqTileElems);
      if (x.cblk) c1 = std::min<uint64_t>(c1, c + kBqBlock - (x.cph + c) % kBqBlock);
      const uint64_t cols = c1 - c, tr = cols >= kSqTileElems ? 1 : kSqTileElems / cols;
      for (uint64_t r = 0; r < h; r += tr) {
        RqTile t;
        memset(&t, 0, sizeof(t));
        const uint64_t rows = std::min(tr, h - r);
        t.src = x.src + (y0 + r - x.r0) * x.stride + c;
        t.src_stride = x.stride;
        t.scale = x.scale + (y0 + r - x.r0) * x.step + (x.cblk ? 4 * ((x.cph + c) / kBqBlock) : 0);
        t.scale_step = x.step;
        t.dst = T.dst + (x.b * T.rows + y0 + r) * T.cols + x.c0 + c;
        t.dst_pitch = static_cast<uint32_t>(T.cols);
        t.rows = static_cast<uint32_t>(rows);
        t.cols = static_cast<uint32_t>(cols);
        t.group = g;
        t.vec = aligned16(t.src, t.src_stride, rows) ? 1u : 0u;
        t.scale_inv = first_row && r == 0 && x.c0 + c == 0 ? scale_inv : 0;
        out->tiles.push_back(t);
        count(rows * cols, x);
      }
      c = c1;
    }
  }

  // Exact coverage of matrix b of target t by its segments (sorted by first row).
  int check_cover(uint64_t t, uint64_t b, const Seg* const* segs, size_t ns) {
    const tsb_sq_target_t& T = targets[t];
    return sweep_cover(
        T.rows, T.cols, segs, ns, [](uint64_t, uint64_t, const std::vector<const Seg*>&) { return 0; },
        [&](uint64_t y, uint64_t c) {
          std::string grp = "target " + std::to_string(t) + " group (" + std::to_string(b);
          if (T.granularity == TSB_SCALE_PER_BLOCK)
            grp += ", " + std::to_string(y / kBqBlock) + ", " + std::to_string(c / kBqBlock);
          else if (T.granularity == TSB_SCALE_PER_CHANNEL)
            grp += ", " + std::to_string(y);
          return fail(TSB_ERR_INVALID, grp + "): its elements are not all written exactly once (at row " + std::to_string(y) +
                                           ", column " + std::to_string(c) + ")");
        });
  }

  // Emit the work of matrix b of target t.
  void matrix(uint64_t t, uint64_t b, const Seg* const* segs, size_t ns) {
    const tsb_sq_target_t& T = targets[t];
    if (T.granularity == TSB_SCALE_PER_BLOCK) {
      const uint64_t nbr = (T.rows + kBqBlock - 1) / kBqBlock, nbc = (T.cols + kBqBlock - 1) / kBqBlock;
      std::vector<std::vector<const Seg*>> by_block(nbr * nbc);
      for (size_t k = 0; k < ns; ++k) {
        const Seg& x = *segs[k];
        for (uint64_t br = x.r0 / kBqBlock; br <= (x.r0 + x.er - 1) / kBqBlock; ++br)
          for (uint64_t bc = x.c0 / kBqBlock; bc <= (x.c0 + x.ec - 1) / kBqBlock; ++bc) by_block[br * nbc + bc].push_back(&x);
      }
      for (uint64_t blk = 0; blk < nbr * nbc; ++blk) {
        const uint64_t br = blk / nbc, bc = blk % nbc, R0 = br * kBqBlock, C0 = bc * kBqBlock;
        const uint64_t R1 = std::min(T.rows, R0 + kBqBlock), C1 = std::min(T.cols, C0 + kBqBlock);
        const size_t first = out->pieces.size();
        for (const Seg* x : by_block[blk]) {
          const uint64_t y0 = std::max(x->r0, R0), y1 = std::min(x->r0 + x->er, R1);
          const uint64_t c0 = std::max(x->c0, C0), c1 = std::min(x->c0 + x->ec, C1);
          piece(*x, y0, y1 - y0, c0, c1 - c0, y0 - R0, c0 - C0);
        }
        unit(T.dst + (b * T.rows + R0) * T.cols + C0, T.scale_inv + 4 * ((b * nbr + br) * nbc + bc), T.cols, R1 - R0,
             C1 - C0, first, false);
      }
      return;
    }
    if (T.granularity == TSB_SCALE_PER_CHANNEL && T.cols <= kSqStageBytes) {
      const uint64_t per_band = std::min<uint64_t>(kSqBandRows, kSqStageBytes / round16(static_cast<uint32_t>(T.cols)));
      std::vector<const Seg*> act;
      size_t next = 0;
      for (uint64_t r = 0; r < T.rows; r += per_band) {
        const uint64_t r1 = std::min(T.rows, r + per_band);
        act.erase(std::remove_if(act.begin(), act.end(), [r](const Seg* x) { return x->r0 + x->er <= r; }), act.end());
        while (next < ns && segs[next]->r0 < r1) act.push_back(segs[next++]);
        const size_t first = out->pieces.size();
        for (const Seg* x : act) {
          const uint64_t y0 = std::max(x->r0, r), y1 = std::min(x->r0 + x->er, r1);
          piece(*x, y0, y1 - y0, x->c0, x->ec, y0 - r, x->c0);
        }
        unit(T.dst + (b * T.rows + r) * T.cols, T.scale_inv + 4 * (b * T.rows + r), T.cols, r1 - r, T.cols, first, true);
      }
      return;
    }
    if (T.granularity == TSB_SCALE_PER_TENSOR) {
      const uint32_t g = out->n_groups++;
      for (size_t k = 0; k < ns; ++k) tiles(*segs[k], segs[k]->r0, segs[k]->er, g, segs[k]->r0 == 0, T.scale_inv + 4 * b);
      return;
    }
    // per-channel rows longer than the stage: one two-pass group per row
    const uint32_t g0 = out->n_groups;
    out->n_groups += static_cast<uint32_t>(T.rows);
    for (size_t k = 0; k < ns; ++k) {
      const Seg& x = *segs[k];
      for (uint64_t y = x.r0; y < x.r0 + x.er; ++y)
        tiles(x, y, 1, g0 + static_cast<uint32_t>(y), true, T.scale_inv + 4 * (b * T.rows + y));
    }
  }
};

constexpr GridRules kTargetRules{"target", "NULL dst or scale_inv", "dst", "scale_inv",
                                 (1u << TSB_SCALE_PER_BLOCK) | (1u << TSB_SCALE_PER_CHANNEL) | (1u << TSB_SCALE_PER_TENSOR), 1ull << 31};

int requant_fp8_compile(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources, uint64_t n_sources,
                        const tsb_sq_target_t* targets, uint64_t n_targets, RqTables* out) {
  if ((n && !rects) || (n_sources && !sources) || (n_targets && !targets))
    return fail(TSB_ERR_INVALID, "requant_fp8: NULL rects, sources or targets");
  std::vector<TargetGeom> sgeom;
  int st = dq_source_geoms(sources, n_sources, &sgeom);
  if (st) return st;
  std::vector<TargetGeom> geom(n_targets);
  std::vector<uint64_t> base(n_targets + 1, 0);  // matrix index of every target's first matrix
  for (uint64_t t = 0; t < n_targets; ++t) {
    const tsb_sq_target_t& T = targets[t];
    if ((st = check_grid(kTargetRules, t, {T.dst, T.scale_inv, T.batch, T.rows, T.cols, 0, 0, 1, T.granularity, T.pad,
                                           !T.dst || !T.scale_inv})))
      return st;
    geom[t] = {T.dst, T.batch, T.rows, T.cols};
    base[t + 1] = base[t] + T.batch;
    const uint64_t groups = T.granularity == TSB_SCALE_PER_BLOCK ? ((T.rows + kBqBlock - 1) / kBqBlock) * ((T.cols + kBqBlock - 1) / kBqBlock)
                            : T.granularity == TSB_SCALE_PER_CHANNEL ? T.rows : 1;
    out->payload_bytes += T.batch * (T.rows * T.cols + 4 * groups);
  }
  std::vector<TargetBox> boxes;
  std::vector<Seg> segs;
  for (uint64_t i = 0; i < n; ++i) {
    boxes.clear();
    if ((st = rect_requant_boxes(rects[i], i, geom.data(), n_targets, &boxes))) return st;
    for (const TargetBox& x : boxes)
      if ((st = source_segments(x, i, sources, n_sources, &segs))) return st;
  }
  // segments grouped by matrix, each matrix's sorted by first row
  std::vector<const Seg*> order(segs.size());
  for (size_t i = 0; i < segs.size(); ++i) order[i] = &segs[i];
  std::stable_sort(order.begin(), order.end(), [&](const Seg* a, const Seg* c) {
    const uint64_t ma = base[a->t] + a->b, mc = base[c->t] + c->b;
    return ma != mc ? ma < mc : a->r0 < c->r0;
  });
  Compiler cc{device, targets, out};
  size_t i = 0;
  for (uint64_t t = 0; t < n_targets; ++t) {
    for (uint64_t b = 0; b < targets[t].batch; ++b) {
      const size_t first = i;
      while (i < order.size() && order[i]->t == t && order[i]->b == b) ++i;
      if ((st = cc.check_cover(t, b, order.data() + first, i - first))) return st;
      cc.matrix(t, b, order.data() + first, i - first);
      if (out->units.size() >= (1ull << 31) || out->tiles.size() >= (1ull << 31) || out->pieces.size() >= (1ull << 32) ||
          out->n_groups >= (1u << 31))
        return fail(TSB_ERR_UNSUPPORTED, "requant_fp8: more than 2^31 units, tiles or groups");
    }
  }
  return TSB_OK;
}

// max abs_bits of the 16 scaled elements of v
__device__ __forceinline__ uint32_t fold_scaled16(uint32_t m, const uint4& v, float scale) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (uint32_t j = 0; j < 8; ++j) {
    uint32_t lo, hi;
    scaled_e4m3x2(w[j >> 1] >> (16 * (j & 1)), scale, &lo, &hi);
    m = max(m, max(abs_bits(lo), abs_bits(hi)));
  }
  return m;
}

// the f32 bits of the 16 scaled elements of v, in element order
__device__ __forceinline__ void widen_scaled16(const uint4& v, float scale, uint32_t f[16]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (uint32_t j = 0; j < 8; ++j) scaled_e4m3x2(w[j >> 1] >> (16 * (j & 1)), scale, &f[2 * j], &f[2 * j + 1]);
}

// one scaled element
__device__ __forceinline__ uint32_t scaled1(uint32_t byte, float scale) {
  uint32_t lo, hi;
  scaled_e4m3x2(byte, scale, &lo, &hi);
  return lo;
}

// the float32 source scale of row r of a tile (scale0: that of row 0)
__device__ __forceinline__ float row_scale(uint64_t scale, uint32_t step, uint32_t r, float scale0) {
  return step ? __ldg(reinterpret_cast<const float*>(scale + static_cast<uint64_t>(r) * step)) : scale0;
}

// the float32 source scale of element (r, c) of a piece
__device__ __forceinline__ float source_scale(const RqPiece& p, uint32_t r, uint32_t c) {
  return __ldg(reinterpret_cast<const float*>(p.scale + static_cast<uint64_t>(r) * p.scale_step +
                                              (p.col_blocks ? 4u * ((p.col_phase + c) / kBqBlock) : 0u)));
}

// Phase 1: the unit's pieces -> shared memory (row pitch spitch), |x| folded into s_amax[row] (kPerRow) or into
// the returned per-thread max.
template <bool kPerRow>
__device__ __forceinline__ uint32_t stage_unit(const RqUnit& u, const RqPiece* __restrict__ pieces, unsigned char* smem,
                                               uint32_t spitch, uint32_t* s_amax) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  uint32_t mt = 0;
  for (uint32_t q = 0; q < u.n_pieces; ++q) {
    const RqPiece p = pieces[u.piece0 + q];
    const char* src = reinterpret_cast<const char*>(p.src);
    unsigned char* s0 = smem + p.row0 * spitch + p.col0;
    uint32_t* rmax = s_amax + p.row0;
    if (p.vec) {
      // each warp takes 32 * kUnroll consecutive 16-byte units per step (coalesced 512-byte loads)
      const uint32_t upr = p.cols / 16;
      const uint32_t total = p.rows * upr;
      for (uint32_t base = warp * 32 * kUnroll; base < total; base += kQuantThreads * kUnroll) {
        uint4 v[kUnroll];
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
          const uint32_t idx = base + k * 32 + lane;
          if (idx < total) {
            const uint32_t r = idx / upr, c = idx - r * upr;
            v[k] = ldg16(src + static_cast<int64_t>(r) * p.src_stride + c * 16);
          }
        }
        const uint32_t rf = base / upr, rl = (min(base + 32 * kUnroll, total) - 1) / upr;
        uint32_t m = 0;
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
          const uint32_t idx = base + k * 32 + lane;
          if (idx < total) {
            const uint32_t r = idx / upr, c = idx - r * upr;
            *reinterpret_cast<uint4*>(s0 + r * spitch + c * 16) = v[k];
            const uint32_t mk = fold_scaled16(0u, v[k], source_scale(p, r, c * 16));
            if (!kPerRow || rf == rl)
              m = max(m, mk);
            else
              atomicMax(rmax + r, mk);
          }
        }
        if (kPerRow) {
          if (rf == rl) {
            m = __reduce_max_sync(0xffffffffu, m);
            if (lane == 0) atomicMax(rmax + rf, m);
          }
        } else {
          mt = max(mt, m);
        }
      }
    } else {
      const uint32_t total = p.rows * p.cols;
      for (uint32_t base = warp * 32; base < total; base += kQuantThreads) {
        const uint32_t idx = base + lane;
        const uint32_t rf = base / p.cols, rl = (min(base + 32, total) - 1) / p.cols;
        uint32_t m = 0;
        if (idx < total) {
          const uint32_t r = idx / p.cols, c = idx - r * p.cols;
          const unsigned char q8 = __ldg(reinterpret_cast<const unsigned char*>(src + static_cast<int64_t>(r) * p.src_stride + c));
          s0[r * spitch + c] = q8;
          m = abs_bits(scaled1(q8, source_scale(p, r, c)));
          if (kPerRow && rf != rl) atomicMax(rmax + r, m);
        }
        if (kPerRow) {
          if (rf == rl) {
            m = __reduce_max_sync(0xffffffffu, m);
            if (lane == 0) atomicMax(rmax + rf, m);
          }
        } else {
          mt = max(mt, m);
        }
      }
    }
  }
  return mt;
}

// Phase 2: staged bytes -> x -> e4m3fn with the unit's scale (s_scale[row] or s_scale[0]).
template <bool kPerRow>
__device__ __forceinline__ void quantise_unit(const RqUnit& u, const RqPiece* __restrict__ pieces, const unsigned char* smem,
                                              uint32_t spitch, const float* s_scale) {
  for (uint32_t q = 0; q < u.n_pieces; ++q) {
    const RqPiece p = pieces[u.piece0 + q];
    const uint32_t cpr = (p.cols + 15u) / 16u;
    const uint32_t total = p.rows * cpr;
    for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
      const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
      const uint32_t nvalid = min(16u, p.cols - c);
      const uint32_t row = p.row0 + r, col = p.col0 + c;
      const unsigned char* s = smem + row * spitch + col;
      // one source scale for the 16 elements unless they straddle a source block
      const bool one_scale = !p.col_blocks || (p.col_phase + c) % kBqBlock <= kBqBlock - 16;
      uint32_t f[16], o[4];
      if (nvalid == 16 && (col & 15u) == 0 && one_scale) {
        widen_scaled16(*reinterpret_cast<const uint4*>(s), source_scale(p, r, c), f);
      } else {
        for (uint32_t j = 0; j < 16; ++j) f[j] = j < nvalid ? scaled1(s[j], source_scale(p, r, c + j)) : 0u;
      }
      narrow16(f, s_scale[kPerRow ? row : 0], o);
      store16(reinterpret_cast<char*>(u.dst) + static_cast<uint64_t>(row) * u.pitch + col, nvalid, o);
    }
  }
}

template <bool kPerRow, bool kUe8m0>
__device__ __forceinline__ void run_unit(const RqUnit& u, const RqPiece* pieces, unsigned char* smem, uint32_t* s_amax,
                                         float* s_scale, uint32_t* s_red) {
  const uint32_t spitch = (u.cols + 15u) & ~15u;
  if (kPerRow) {
    for (uint32_t r = threadIdx.x; r < u.rows; r += kQuantThreads) s_amax[r] = 0;
    __syncthreads();
  }
  uint32_t m = stage_unit<kPerRow>(u, pieces, smem, spitch, s_amax);
  if (kPerRow) {
    __syncthreads();
    for (uint32_t r = threadIdx.x; r < u.rows; r += kQuantThreads) {
      float scale, scale_inv;
      group_scales<kUe8m0>(s_amax[r], &scale, &scale_inv);
      s_scale[r] = scale;
      reinterpret_cast<float*>(u.scale_inv)[r] = scale_inv;
    }
  } else {
    cta_max(m, s_red, [&](uint32_t a) {
      float scale, scale_inv;
      group_scales<kUe8m0>(a, &scale, &scale_inv);
      s_scale[0] = scale;
      *reinterpret_cast<float*>(u.scale_inv) = scale_inv;
    });
  }
  __syncthreads();
  quantise_unit<kPerRow>(u, pieces, smem, spitch, s_scale);
}

// kUe8m0 (here and in requant_fp8_quant_kernel): power-of-two scales (TSB_QUANT_UE8M0)
template <bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads) requant_fp8_staged_kernel(const RqUnit* __restrict__ units,
                                                                        const RqPiece* __restrict__ pieces) {
  extern __shared__ __align__(16) unsigned char stage[];
  __shared__ uint32_t s_amax[kSqBandRows];
  __shared__ float s_scale[kSqBandRows];
  __shared__ uint32_t s_red[kQuantThreads / 32];
  const RqUnit u = units[blockIdx.x];
  if (u.per_row)
    run_unit<true, kUe8m0>(u, pieces, stage, s_amax, s_scale, s_red);
  else
    run_unit<false, kUe8m0>(u, pieces, stage, s_amax, s_scale, s_red);
}

__global__ void __launch_bounds__(kQuantThreads) requant_fp8_amax_kernel(const RqTile* __restrict__ tiles, uint32_t* amax) {
  __shared__ uint32_t s_red[kQuantThreads / 32];
  const RqTile t = tiles[blockIdx.x];
  const char* src = reinterpret_cast<const char*>(t.src);
  const float scale0 = __ldg(reinterpret_cast<const float*>(t.scale));
  const uint32_t cpr = (t.cols + 15u) / 16u;
  const uint32_t total = t.rows * cpr;
  uint32_t m = 0;
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
      const float scale = row_scale(t.scale, t.scale_step, r, scale0);
      if (t.vec && c + 16u <= t.cols) {
        m = fold_scaled16(m, v[k], scale);
      } else {
        const unsigned char* s = reinterpret_cast<const unsigned char*>(src + static_cast<int64_t>(r) * t.src_stride + c);
        const uint32_t nvalid = min(16u, t.cols - c);
        for (uint32_t j = 0; j < nvalid; ++j) m = max(m, abs_bits(scaled1(__ldg(s + j), scale)));
      }
    }
  }
  cta_max(m, s_red, [&](uint32_t a) {
    if (a) atomicMax(amax + t.group, a);
  });
}

template <bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads) requant_fp8_quant_kernel(const RqTile* __restrict__ tiles,
                                                                       const uint32_t* __restrict__ amax) {
  const RqTile t = tiles[blockIdx.x];
  float dscale, scale_inv;
  group_scales<kUe8m0>(amax[t.group], &dscale, &scale_inv);
  if (t.scale_inv && threadIdx.x == 0) *reinterpret_cast<float*>(t.scale_inv) = scale_inv;
  const char* src = reinterpret_cast<const char*>(t.src);
  const float scale0 = __ldg(reinterpret_cast<const float*>(t.scale));
  const uint32_t cpr = (t.cols + 15u) / 16u;
  const uint32_t total = t.rows * cpr;
  for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
    const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
    const uint32_t nvalid = min(16u, t.cols - c);
    const char* s = src + static_cast<int64_t>(r) * t.src_stride + c;
    const float scale = row_scale(t.scale, t.scale_step, r, scale0);
    uint32_t f[16], o[4];
    if (t.vec && nvalid == 16) {
      widen_scaled16(ldg16(s), scale, f);
    } else {
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) f[j] = j < nvalid ? scaled1(__ldg(reinterpret_cast<const unsigned char*>(s) + j), scale) : 0u;
    }
    narrow16(f, dscale, o);
    store16(reinterpret_cast<char*>(t.dst) + static_cast<uint64_t>(r) * t.dst_pitch + c, nvalid, o);
  }
}

// d = {RqUnit table | RqPiece table | RqTile table | amax words}, one CTA per unit and per tile (and pass)
int requant_fp8_plan(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources, uint64_t n_sources,
                     const tsb_sq_target_t* targets, uint64_t n_targets, QuantPlan* q) {
  RqTables tb;
  int st = requant_fp8_compile(device, rects, n, sources, n_sources, targets, n_targets, &tb);
  if (st) return st;
  q->add(tb.units);
  const size_t pieces = q->add(tb.pieces), tiles = q->add(tb.tiles), amax = q->seal(tb.n_groups);
  q->describe(n, static_cast<uint32_t>(tb.units.size() + tb.tiles.size()), tb.stage_bytes, tb);
  q->launch = [pieces, tiles, amax, n_units = static_cast<uint32_t>(tb.units.size()), n_tiles = static_cast<uint32_t>(tb.tiles.size()),
               n_groups = tb.n_groups, stage_bytes = tb.stage_bytes, ue8m0 = q->ue8m0](char* d, cudaStream_t s) -> int {
    if (n_units) {
      const auto staged = ue8m0 ? requant_fp8_staged_kernel<true> : requant_fp8_staged_kernel<false>;
      staged<<<n_units, kQuantThreads, stage_bytes, s>>>(reinterpret_cast<const RqUnit*>(d), reinterpret_cast<const RqPiece*>(d + pieces));
      if (int st = launched("requant_fp8_staged_kernel launch")) return st;
    }
    if (!n_tiles) return TSB_OK;
    return launch_two_pass(requant_fp8_amax_kernel, ue8m0 ? requant_fp8_quant_kernel<true> : requant_fp8_quant_kernel<false>,
                           "requant_fp8", reinterpret_cast<const RqTile*>(d + tiles), n_tiles, reinterpret_cast<uint32_t*>(d + amax),
                           n_groups, s);
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_requant_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                           uint64_t n_sources, const tsb_sq_target_t* targets, uint64_t n_targets, uint32_t flags,
                                           tsb_plan_t* out) {
  return quant_plan_create("tsb_requant_fp8_plan_create", device, flags, TSB_QUANT_UE8M0, out, [&](QuantPlan* q) {
    return requant_fp8_plan(device, rects, n, sources, n_sources, targets, n_targets, q);
  });
}

extern "C" int tsb_requant_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                            uint64_t n_sources, const tsb_sq_target_t* targets, uint64_t n_targets,
                                            uint32_t flags, void* out_units, uint64_t unit_cap, uint64_t* out_n_units,
                                            void* out_pieces, uint64_t piece_cap, uint64_t* out_n_pieces, void* out_tiles,
                                            uint64_t tile_cap, uint64_t* out_n_tiles, uint64_t* out_n_groups) {
  return quant_compile_host(
      "tsb_requant_fp8_compile_host", flags, TSB_QUANT_UE8M0,
      [&](QuantPlan* q) { return requant_fp8_plan(device, rects, n, sources, n_sources, targets, n_targets, q); },
      {{out_units, unit_cap, out_n_units, "out_units"}, {out_pieces, piece_cap, out_n_pieces, "out_pieces"},
       {out_tiles, tile_cap, out_n_tiles, "out_tiles"}},
      out_n_groups);
}
