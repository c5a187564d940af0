// Per-channel and per-tensor scaled FP8 pulls (sm_90a, H100): gather bf16/f16/f32 source rectangles into
// float8_e4m3fn destinations with one float32 scale_inv per row (compressed-tensors FP8 / fbgemm-fp8,
// weight_scale [N, 1]) or per matrix (vLLM quantization="fp8"), quantising on the way.  The formula is the
// block-scaled one (block_fp8.cu) over a different group.
//
// Host side: the plan compiler maps every rect onto its target's [batch, rows, cols] grid (rect_boxes,
// shared with block_fp8.cu) and sweeps each matrix's boxes by row: between two consecutive box row
// boundaries the boxes that span the rows must cut [0, cols) into contiguous, disjoint runs of one
// dtype.  That checks exact coverage of every group in time proportional to the boxes, not the
// elements, and hands out the work in group order:
//   per-channel rows of at most kSqStageBytes source bytes  -> bands of whole rows (row-staged kernel)
//   per-tensor matrices and longer per-channel rows          -> tiles of at most kSqTileElems (two-pass)
// Device side:
//   scaled_fp8_rows_kernel   one 256-thread CTA per band: its pieces land in shared memory (16-byte loads
//                            where alignment allows), each warp folding |x| into the row's max as the data
//                            arrives; one scale per row; quantise from shared memory with 16-byte stores.
//                            Each source byte is read once.
//   scaled_fp8_amax_kernel   pass 1, one CTA per tile: max |x| of the tile, one atomicMax on its group's
//                            amax word (|x| as an integer: finite < Inf < NaN, so a NaN poisons the group).
//   scaled_fp8_quant_kernel  pass 2, one CTA per tile: the group's scale from its amax, the tile re-read and
//                            quantised straight to HBM; the group's one designated tile writes scale_inv.
// int8 destinations (TSB_I8 rects) run scaled_int8_rows_kernel and scaled_int8_quant_kernel, the same kernels in
// the int8 format of fp8_quant.cuh (scale step 127, round-to-nearest-even saturating narrowing, NaN -> 0), after
// the same amax pass, from the same tables.
// The amax words live in the plan's device allocation and are cleared on the launch stream before pass 1,
// so a replayed plan starts from zero.

#include <algorithm>
#include <cstring>

#include "fp8_quant.cuh"
#include "tsb_internal.h"

namespace tsb {

namespace {

struct Compiler {
  int device;
  const tsb_sq_target_t* targets;
  SqTables* out;

  void count(uint64_t bytes, const TargetBox& x) { out->read(bytes, x.src_device, device); }

  // rows [y0, y1) of box x as two-pass tiles of group g; the tile holding the group's element (0, 0)
  // writes `scale`
  void tiles(const TargetBox& x, uint64_t y0, uint64_t y1, uint32_t g, uint64_t scale) {
    const tsb_sq_target_t& T = targets[x.target];
    const uint32_t es = quant_src_bytes(x.dtype);
    const uint64_t h = y1 - y0, w = x.ec;
    const uint64_t tr = w >= kSqTileElems ? 1 : kSqTileElems / w, tc = std::min<uint64_t>(w, kSqTileElems);
    for (uint64_t r = 0; r < h; r += tr) {
      for (uint64_t c = 0; c < w; c += tc) {
        SqTile t;
        memset(&t, 0, sizeof(t));
        const uint64_t rows = std::min(tr, h - r), cols = std::min(tc, w - c);
        t.src = x.src + (y0 + r - x.r0) * x.row_stride + c * es;
        t.src_stride = x.row_stride;
        t.dst = T.dst + (x.b * T.rows + y0 + r) * T.cols + x.c0 + c;
        t.dst_pitch = static_cast<uint32_t>(T.cols);
        t.rows = static_cast<uint32_t>(rows);
        t.cols = static_cast<uint32_t>(cols);
        t.group = g;
        t.src_dtype = x.dtype;
        t.vec = vec_ok(t.src, t.src_stride, rows, cols, es) ? 1u : 0u;
        const bool origin = (T.granularity == TSB_SCALE_PER_TENSOR ? y0 + r == 0 : r == 0) && x.c0 + c == 0;
        t.scale = origin ? scale : 0;
        out->tiles.push_back(t);
        count(rows * cols * es, x);
      }
    }
  }

  // rows [y0, y1) of a per-channel matrix, spanned by the boxes `act` (sorted by column)
  void channel_rows(const std::vector<const TargetBox*>& act, uint64_t y0, uint64_t y1) {
    const TargetBox& x0 = *act[0];
    const tsb_sq_target_t& T = targets[x0.target];
    const uint32_t es = quant_src_bytes(x0.dtype);
    const uint64_t scale0 = T.scale_inv + 4 * (x0.b * T.rows);
    if (T.cols * es > kSqStageBytes) {  // the row does not fit the stage: two passes, one group per row
      for (uint64_t y = y0; y < y1; ++y) {
        const uint32_t g = out->n_groups++;
        for (const TargetBox* x : act) tiles(*x, y, y + 1, g, scale0 + 4 * y);
      }
      return;
    }
    const uint32_t spitch = round16(static_cast<uint32_t>(T.cols) * es);
    const uint64_t per_band = std::min<uint64_t>(kSqBandRows, kSqStageBytes / spitch);
    for (uint64_t r = y0; r < y1; r += per_band) {
      SqBand b;
      memset(&b, 0, sizeof(b));
      b.rows = static_cast<uint32_t>(std::min(per_band, y1 - r));
      b.cols = static_cast<uint32_t>(T.cols);
      b.dst = T.dst + (x0.b * T.rows + r) * T.cols;
      b.scale = scale0 + 4 * r;
      b.piece0 = static_cast<uint32_t>(out->pieces.size());
      b.n_pieces = static_cast<uint32_t>(act.size());
      b.src_dtype = x0.dtype;
      out->stage_bytes = std::max(out->stage_bytes, b.rows * spitch);
      for (const TargetBox* x : act) {
        SqPiece p;
        memset(&p, 0, sizeof(p));
        p.src = x->src + (r - x->r0) * x->row_stride;
        p.src_stride = x->row_stride;
        p.row0 = 0;
        p.col0 = static_cast<uint32_t>(x->c0);
        p.rows = b.rows;
        p.cols = static_cast<uint32_t>(x->ec);
        p.vec = (vec_ok(p.src, p.src_stride, p.rows, p.cols, es) && (p.col0 * es) % 16 == 0) ? 1u : 0u;
        out->pieces.push_back(p);
        count(static_cast<uint64_t>(p.rows) * p.cols * es, *x);
      }
      out->bands.push_back(b);
    }
  }

  // Sweep the boxes of matrix b of target t (sorted by first row) and emit its work.
  int matrix(uint64_t t, uint64_t b, const TargetBox* const* boxes, size_t nb) {
    const tsb_sq_target_t& T = targets[t];
    const bool tensor = T.granularity == TSB_SCALE_PER_TENSOR;
    const auto group = [&](uint64_t y) {
      return "target " + std::to_string(t) + " group (" + std::to_string(b) + (tensor ? std::string(")") : ", " + std::to_string(y) + ")");
    };
    uint32_t g = 0;
    uint32_t dtype = nb ? boxes[0]->dtype : 0;
    return sweep_cover(
        T.rows, T.cols, boxes, nb,
        [&](uint64_t y, uint64_t y1, const std::vector<const TargetBox*>& sorted) -> int {
          if (!tensor) dtype = sorted[0]->dtype;
          for (const TargetBox* x : sorted)
            if (x->dtype != dtype) return fail(TSB_ERR_INVALID, group(y) + ": sources of different dtypes");
          if (tensor) {
            if (y == 0) g = out->n_groups++;
            for (const TargetBox* x : sorted) tiles(*x, y, y1, g, T.scale_inv + 4 * b);
          } else {
            channel_rows(sorted, y, y1);
          }
          return TSB_OK;
        },
        [&](uint64_t y, uint64_t) {
          return fail(TSB_ERR_INVALID, group(y) + ": its elements are not all written exactly once (at row " + std::to_string(y) + ")");
        });
  }
};

constexpr GridRules kTargetRules{"target", "NULL dst or scale_inv", "dst", "scale_inv",
                                 (1u << TSB_SCALE_PER_CHANNEL) | (1u << TSB_SCALE_PER_TENSOR), 1ull << 31};

int scaled_fp8_compile(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets,
                       uint64_t n_targets, SqTables* out) {
  if ((n && !rects) || (n_targets && !targets)) return fail(TSB_ERR_INVALID, "scaled_fp8: NULL rects or targets");
  std::vector<TargetGeom> geom(n_targets);
  std::vector<uint64_t> base(n_targets + 1, 0);  // matrix index of every target's first matrix
  for (uint64_t t = 0; t < n_targets; ++t) {
    const tsb_sq_target_t& T = targets[t];
    int st = check_grid(kTargetRules, t, {T.dst, T.scale_inv, T.batch, T.rows, T.cols, 0, 0, 1, T.granularity, T.pad, !T.dst || !T.scale_inv});
    if (st) return st;
    geom[t] = {T.dst, T.batch, T.rows, T.cols};
    base[t + 1] = base[t] + T.batch;
    out->payload_bytes += T.batch * T.rows * T.cols + 4 * T.batch * (T.granularity == TSB_SCALE_PER_CHANNEL ? T.rows : 1);
  }
  std::vector<TargetBox> boxes;
  for (uint64_t i = 0; i < n; ++i) {
    int st = rect_boxes(rects[i], i, geom.data(), n_targets, &boxes);
    if (st) return st;
  }
  // boxes grouped by matrix, each matrix's sorted by first row
  std::vector<const TargetBox*> order(boxes.size());
  for (size_t i = 0; i < boxes.size(); ++i) order[i] = &boxes[i];
  std::stable_sort(order.begin(), order.end(), [&](const TargetBox* a, const TargetBox* c) {
    const uint64_t ma = base[a->target] + a->b, mc = base[c->target] + c->b;
    return ma != mc ? ma < mc : a->r0 < c->r0;
  });
  Compiler cc{device, targets, out};
  size_t i = 0;
  for (uint64_t t = 0; t < n_targets; ++t) {
    for (uint64_t b = 0; b < targets[t].batch; ++b) {
      const size_t first = i;
      while (i < order.size() && order[i]->target == t && order[i]->b == b) ++i;
      int st = cc.matrix(t, b, order.data() + first, i - first);
      if (st) return st;
      if (out->bands.size() >= (1ull << 31) || out->tiles.size() >= (1ull << 31) || out->n_groups >= (1u << 31))
        return fail(TSB_ERR_UNSUPPORTED, "scaled_fp8: more than 2^31 bands, tiles or groups");
    }
  }
  return TSB_OK;
}

// max abs_bits of `a` (one word per lane, 0 for lanes without data) into s_amax[row] when the whole warp
// holds one row (warp-uniform `one_row`), else per lane
__device__ __forceinline__ void fold_rows(bool one_row, uint32_t row, uint32_t m, uint32_t* s_amax) {
  if (one_row) {
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31u) == 0) atomicMax(s_amax + row, m);
  }
}

// Band pieces -> shared memory (row pitch spitch bytes), every row's max |x| bits -> s_amax.
template <uint32_t DT>
__device__ __forceinline__ void stage_band(const SqBand& band, const SqPiece* __restrict__ pieces, unsigned char* smem,
                                           uint32_t spitch, uint32_t* s_amax) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  for (uint32_t q = 0; q < band.n_pieces; ++q) {
    const SqPiece p = pieces[band.piece0 + q];
    const char* src = reinterpret_cast<const char*>(p.src);
    unsigned char* s0 = smem + p.row0 * spitch + p.col0 * es;
    uint32_t* rmax = s_amax + p.row0;
    if (p.vec) {
      // each warp takes 32 * kUnroll consecutive 16-byte units per step (coalesced 512-byte loads)
      const uint32_t upr = p.cols * es / 16;
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
            if (rf == rl)
              m = fold16<DT>(m, v[k]);
            else
              atomicMax(rmax + r, fold16<DT>(0u, v[k]));
          }
        }
        fold_rows(rf == rl, rf, m, rmax);
      }
    } else {
      const uint32_t total = p.rows * p.cols;
      for (uint32_t base = warp * 32; base < total; base += kQuantThreads) {
        const uint32_t idx = base + lane;
        const uint32_t rf = base / p.cols, rl = (min(base + 32, total) - 1) / p.cols;
        uint32_t m = 0;
        if (idx < total) {
          const uint32_t r = idx / p.cols, c = idx - r * p.cols;
          const char* a = src + static_cast<int64_t>(r) * p.src_stride + c * es;
          unsigned char* s = s0 + r * spitch + c * es;
          uint32_t w;
          if (es == 4) {
            w = __ldg(reinterpret_cast<const uint32_t*>(a));
            *reinterpret_cast<uint32_t*>(s) = w;
          } else {
            const unsigned short h = __ldg(reinterpret_cast<const unsigned short*>(a));
            *reinterpret_cast<unsigned short*>(s) = h;
            w = h;
          }
          m = abs_bits(Src<DT>::f32(w));
          if (rf != rl) atomicMax(rmax + r, m);
        }
        fold_rows(rf == rl, rf, m, rmax);
      }
    }
  }
}

template <uint32_t DT, class Out>
__device__ __forceinline__ void run_band(const SqBand& band, const SqPiece* pieces, unsigned char* smem, uint32_t* s_amax,
                                         float* s_scale) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const uint32_t spitch = (band.cols * es + 15u) & ~15u;
  for (uint32_t r = threadIdx.x; r < band.rows; r += kQuantThreads) s_amax[r] = 0;
  __syncthreads();
  stage_band<DT>(band, pieces, smem, spitch, s_amax);
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < band.rows; r += kQuantThreads) {
    float scale, scale_inv;
    Out::scales(s_amax[r], &scale, &scale_inv);
    s_scale[r] = scale;
    reinterpret_cast<float*>(band.scale)[r] = scale_inv;
  }
  __syncthreads();
  const uint32_t cpr = (band.cols + 15u) / 16u;
  const uint32_t total = band.rows * cpr;
  for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
    const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
    const uint32_t nvalid = min(16u, band.cols - c);
    uint32_t f[16], o[4];
    load16_shared<DT>(smem + r * spitch + c * es, nvalid, f);
    Out::narrow(f, s_scale[r], o);
    store16(reinterpret_cast<char*>(band.dst) + static_cast<uint64_t>(r) * band.cols + c, nvalid, o);
  }
}

// The CTA's band in destination format Out (fp8_quant.cuh), the body of the row-staged kernels below
template <class Out>
__device__ __forceinline__ void quantise_bands(const SqBand* __restrict__ bands, const SqPiece* __restrict__ pieces,
                                               unsigned char* stage, uint32_t* s_amax, float* s_scale) {
  const SqBand band = bands[blockIdx.x];
  switch (band.src_dtype) {
    case TSB_BF16: run_band<TSB_BF16, Out>(band, pieces, stage, s_amax, s_scale); break;
    case TSB_F16: run_band<TSB_F16, Out>(band, pieces, stage, s_amax, s_scale); break;
    default: run_band<TSB_F32, Out>(band, pieces, stage, s_amax, s_scale); break;
  }
}

// kUe8m0 (here and in scaled_fp8_quant_kernel): power-of-two scales (TSB_QUANT_UE8M0)
template <bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads, 5) scaled_fp8_rows_kernel(const SqBand* __restrict__ bands,
                                                                       const SqPiece* __restrict__ pieces) {
  extern __shared__ __align__(16) unsigned char stage[];
  __shared__ uint32_t s_amax[kSqBandRows];
  __shared__ float s_scale[kSqBandRows];
  quantise_bands<E4m3Out<kUe8m0>>(bands, pieces, stage, s_amax, s_scale);
}

// int8 destinations (TSB_I8), here and in scaled_int8_quant_kernel
__global__ void __launch_bounds__(kQuantThreads, 5) scaled_int8_rows_kernel(const SqBand* __restrict__ bands,
                                                                        const SqPiece* __restrict__ pieces) {
  extern __shared__ __align__(16) unsigned char stage[];
  __shared__ uint32_t s_amax[kSqBandRows];
  __shared__ float s_scale[kSqBandRows];
  quantise_bands<I8Out>(bands, pieces, stage, s_amax, s_scale);
}

// this thread's max abs_bits over the tile
template <uint32_t DT>
__device__ __forceinline__ uint32_t tile_amax(const SqTile& t) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const char* src = reinterpret_cast<const char*>(t.src);
  uint32_t m = 0;
  if (t.vec) {
    const uint32_t upr = t.cols * es / 16;
    const uint32_t total = t.rows * upr;
    for (uint32_t i = threadIdx.x; i < total; i += kQuantThreads * kUnroll) {
      uint4 v[kUnroll];
#pragma unroll
      for (int k = 0; k < kUnroll; ++k) {
        const uint32_t idx = i + k * kQuantThreads;
        if (idx < total) {
          const uint32_t r = idx / upr, c = idx - r * upr;
          v[k] = ldg16(src + static_cast<int64_t>(r) * t.src_stride + c * 16);
        }
      }
#pragma unroll
      for (int k = 0; k < kUnroll; ++k)
        if (i + k * kQuantThreads < total) m = fold16<DT>(m, v[k]);
    }
  } else {
    const uint32_t total = t.rows * t.cols;
    for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
      const uint32_t r = idx / t.cols, c = idx - r * t.cols;
      m = max(m, abs_bits(elem<DT>(reinterpret_cast<const unsigned char*>(src + static_cast<int64_t>(r) * t.src_stride), c)));
    }
  }
  return m;
}

__global__ void __launch_bounds__(kQuantThreads) scaled_fp8_amax_kernel(const SqTile* __restrict__ tiles, uint32_t* amax) {
  __shared__ uint32_t s_red[kQuantThreads / 32];
  const SqTile t = tiles[blockIdx.x];
  uint32_t m;
  switch (t.src_dtype) {
    case TSB_BF16: m = tile_amax<TSB_BF16>(t); break;
    case TSB_F16: m = tile_amax<TSB_F16>(t); break;
    default: m = tile_amax<TSB_F32>(t); break;
  }
  cta_max(m, s_red, [&](uint32_t a) {
    if (a) atomicMax(amax + t.group, a);
  });
}

template <uint32_t DT, class Out>
__device__ __forceinline__ void quantise_tile(const SqTile& t, float scale) {
  constexpr uint32_t es = Src<DT>::kBytes;
  const uint32_t cpr = (t.cols + 15u) / 16u;
  const uint32_t total = t.rows * cpr;
  for (uint32_t idx = threadIdx.x; idx < total; idx += kQuantThreads) {
    const uint32_t r = idx / cpr, c = (idx - r * cpr) * 16u;
    const uint32_t nvalid = min(16u, t.cols - c);
    const char* s = reinterpret_cast<const char*>(t.src) + static_cast<int64_t>(r) * t.src_stride + c * es;
    uint32_t f[16], o[4];
    if (t.vec && nvalid == 16) {
      uint4 w[es];
#pragma unroll
      for (uint32_t i = 0; i < es; ++i) w[i] = ldg16(s + 16 * i);
      widen16<DT>(w, f);
    } else {
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) f[j] = j < nvalid ? elem<DT>(reinterpret_cast<const unsigned char*>(s), j) : 0u;
    }
    Out::narrow(f, scale, o);
    store16(reinterpret_cast<char*>(t.dst) + static_cast<uint64_t>(r) * t.dst_pitch + c, nvalid, o);
  }
}

// Pass 2 of the CTA's tile in destination format Out, the body of the quantise kernels below
template <class Out>
__device__ __forceinline__ void quantise_tiles(const SqTile* __restrict__ tiles, const uint32_t* __restrict__ amax) {
  const SqTile t = tiles[blockIdx.x];
  float scale, scale_inv;
  Out::scales(amax[t.group], &scale, &scale_inv);
  if (t.scale && threadIdx.x == 0) *reinterpret_cast<float*>(t.scale) = scale_inv;
  switch (t.src_dtype) {
    case TSB_BF16: quantise_tile<TSB_BF16, Out>(t, scale); break;
    case TSB_F16: quantise_tile<TSB_F16, Out>(t, scale); break;
    default: quantise_tile<TSB_F32, Out>(t, scale); break;
  }
}

template <bool kUe8m0>
__global__ void __launch_bounds__(kQuantThreads) scaled_fp8_quant_kernel(const SqTile* __restrict__ tiles,
                                                                    const uint32_t* __restrict__ amax) {
  quantise_tiles<E4m3Out<kUe8m0>>(tiles, amax);
}

__global__ void __launch_bounds__(kQuantThreads) scaled_int8_quant_kernel(const SqTile* __restrict__ tiles,
                                                                     const uint32_t* __restrict__ amax) {
  quantise_tiles<I8Out>(tiles, amax);
}

}  // namespace

int launch_scaled_fp8(const SqLaunch& l, cudaStream_t stream) {
  if (l.n_bands) {
    const auto rows_kernel = l.int8 ? scaled_int8_rows_kernel : l.ue8m0 ? scaled_fp8_rows_kernel<true> : scaled_fp8_rows_kernel<false>;
    rows_kernel<<<l.n_bands, kQuantThreads, l.stage_bytes, stream>>>(l.bands, l.pieces);
    if (int st = launched(l.int8 ? "scaled_int8_rows_kernel launch" : "scaled_fp8_rows_kernel launch")) return st;
  }
  if (!l.n_tiles) return TSB_OK;
  const auto quant_kernel = l.int8 ? scaled_int8_quant_kernel : l.ue8m0 ? scaled_fp8_quant_kernel<true> : scaled_fp8_quant_kernel<false>;
  return launch_two_pass(scaled_fp8_amax_kernel, quant_kernel, l.int8 ? "scaled_int8" : "scaled_fp8", l.tiles, l.n_tiles, l.amax,
                         l.n_groups, stream);
}

namespace {

// d = {SqBand table | SqPiece table | SqTile table | amax words}, one CTA per band and per tile (and pass)
int scaled_fp8_plan(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets, uint64_t n_targets,
                    QuantPlan* q) {
  SqTables tb;
  int st = scaled_fp8_compile(device, rects, n, targets, n_targets, &tb);
  if (st || (st = quant_dst_int8(rects, n, q->ue8m0, &q->int8))) return st;
  q->add(tb.bands);
  const size_t pieces = q->add(tb.pieces), tiles = q->add(tb.tiles), amax = q->seal(tb.n_groups);
  q->describe(n, static_cast<uint32_t>(tb.bands.size() + tb.tiles.size()), kSqStageBytes, tb);
  const SqLaunch l{nullptr, nullptr, nullptr, nullptr, static_cast<uint32_t>(tb.bands.size()), static_cast<uint32_t>(tb.tiles.size()),
                   tb.n_groups, tb.stage_bytes, q->ue8m0, q->int8};
  q->launch = [l, pieces, tiles, amax](char* d, cudaStream_t s) {
    SqLaunch x = l;
    x.bands = reinterpret_cast<const SqBand*>(d);
    x.pieces = reinterpret_cast<const SqPiece*>(d + pieces);
    x.tiles = reinterpret_cast<const SqTile*>(d + tiles);
    x.amax = reinterpret_cast<uint32_t*>(d + amax);
    return launch_scaled_fp8(x, s);
  };
  return TSB_OK;
}

}  // namespace

}  // namespace tsb

using namespace tsb;

extern "C" int tsb_scaled_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets,
                                          uint64_t n_targets, uint32_t flags, tsb_plan_t* out) {
  return quant_plan_create("tsb_scaled_fp8_plan_create", device, flags, TSB_QUANT_UE8M0, out,
                           [&](QuantPlan* q) { return scaled_fp8_plan(device, rects, n, targets, n_targets, q); });
}

extern "C" int tsb_scaled_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets,
                                           uint64_t n_targets, uint32_t flags, void* out_bands, uint64_t band_cap,
                                           uint64_t* out_n_bands, void* out_pieces, uint64_t piece_cap, uint64_t* out_n_pieces,
                                           void* out_tiles, uint64_t tile_cap, uint64_t* out_n_tiles, uint64_t* out_n_groups) {
  return quant_compile_host("tsb_scaled_fp8_compile_host", flags, TSB_QUANT_UE8M0,
                            [&](QuantPlan* q) { return scaled_fp8_plan(device, rects, n, targets, n_targets, q); },
                            {{out_bands, band_cap, out_n_bands, "out_bands"}, {out_pieces, piece_cap, out_n_pieces, "out_pieces"},
                             {out_tiles, tile_cap, out_n_tiles, "out_tiles"}},
                            out_n_groups);
}
