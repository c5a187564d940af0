/*
 * fp8_ref.c -- TEST INFRASTRUCTURE ONLY (CPU oracle, never shipped, never on the product path).
 *
 * The fp8 casts of the copy_rects kernel (float8_e4m3fn, float8_e5m2 <-> f32, bf16, f16), restated
 * in plain C as torch's .to() computes them, on top of the byte mover of copy_rects_ref.c.  That
 * file is compiled into this library unchanged (included below), so every pair it knows keeps its
 * exact behaviour here; this file adds the fp8 pairs, a rectangle mover that accepts them, and an
 * interpreter for compiled plan tables that knows the fp8 modes (22-45 of csrc/tsb_internal.h).
 *
 * The fp8 conversions restate c10/util/Float8_e4m3fn.h and Float8_e5m2.h (torch 2.11), which CPU
 * and CUDA share; they are pinned against torch by tests/golden/fp8_cast_vectors.npz.  nan_mode has
 * the meaning of copy_rects_ref.c and matters for fp8 only where the widening to f32 differs: CUDA's
 * f16 -> f32 (cvt.f32.f16, what torch's CUDA .to() widens through) makes every NaN positive, so with
 * nan_mode 1 a negative f16 NaN narrows to 0x7F instead of 0xFF.
 *
 * Build: oracle/fp8_oracle.py (gcc -O2 -shared -fPIC -pthread).
 */
#include "copy_rects_ref.c"

#include <math.h>

/* ---- fp8 conversions ---------------------------------------------------------------------- */
static float bits_f32(uint32_t x) { float f; memcpy(&f, &x, 4); return f; }
static uint32_t f32_bits(float f) { uint32_t x; memcpy(&x, &f, 4); return x; }

/* f32 -> float8_e4m3fn, round to nearest even; e4m3fn has no Inf: |x| >= 480 (everything that
 * rounds past 448), +-Inf and NaN give 0x7F|sign */
static uint8_t f32_to_e4m3(uint32_t x) {
  const uint32_t sign = x & 0x80000000u;
  uint32_t a = x ^ sign;
  uint8_t r;
  if (a >= (1087u << 20)) { /* 480.0f and above, Inf, NaN */
    r = 0x7f;
  } else if (a < (121u << 23)) { /* below 2^-6, the smallest normal: let the FPU round into the subnormals */
    const uint32_t denorm_mask = 141u << 23;
    r = (uint8_t)(f32_bits(bits_f32(a) + bits_f32(denorm_mask)) - denorm_mask);
  } else {
    const uint32_t mant_odd = (a >> 20) & 1u;
    a += ((uint32_t)(7 - 127) << 23) + 0x7ffffu + mant_odd;
    r = (uint8_t)(a >> 20);
  }
  return (uint8_t)(r | (sign >> 24));
}

/* f32 -> float8_e5m2, round to nearest even; |x| >= 61440 rounds to +-Inf, NaN gives 0x7F|sign */
static uint8_t f32_to_e5m2(uint32_t x) {
  const uint32_t sign = x & 0x80000000u;
  uint32_t a = x ^ sign;
  uint8_t r;
  if (a >= (143u << 23)) { /* 65536.0f and above, Inf, NaN */
    r = a > 0x7f800000u ? 0x7f : 0x7c;
  } else if (a < (113u << 23)) { /* below 2^-14, the smallest normal */
    const uint32_t denorm_mask = 134u << 23;
    r = (uint8_t)(f32_bits(bits_f32(a) + bits_f32(denorm_mask)) - denorm_mask);
  } else {
    const uint32_t mant_odd = (a >> 21) & 1u;
    a += ((uint32_t)(15 - 127) << 23) + 0xfffffu + mant_odd;
    r = (uint8_t)(a >> 21);
  }
  return (uint8_t)(r | (sign >> 24));
}

/* float8_e4m3fn -> f32 (exact; 0x7F|sign is NaN) */
static uint32_t e4m3_to_f32(uint8_t b) {
  const uint32_t sign = (uint32_t)(b & 0x80u) << 24;
  const uint32_t e = (b >> 3) & 0xfu, m = b & 7u;
  if (e == 15 && m == 7) return sign | 0x7fc00000u;
  const float mag = e ? ldexpf(1.0f + (float)m / 8.0f, (int)e - 7) : ldexpf((float)m, -9);
  return sign | f32_bits(mag);
}

/* float8_e5m2 -> f32 (exact: an e5m2 byte is the high byte of an f16) */
static uint32_t e5m2_to_f32(uint8_t b) { return f16_to_f32((uint16_t)((uint16_t)b << 8)); }

static int is_fp8(uint32_t dt) { return dt == TSB_F8E4M3 || dt == TSB_F8E5M2; }

static uint32_t fp8_dtype_size(uint32_t dt) { return is_fp8(dt) ? 1u : dtype_size(dt); }

/* a float element (f32, bf16, f16 or fp8) as f32 bits; -1 for another dtype */
static int load_f32(const uint8_t* s, uint32_t dt, uint32_t* out) {
  uint16_t h;
  switch (dt) {
    case TSB_F32: memcpy(out, s, 4); return 0;
    case TSB_BF16: memcpy(&h, s, 2); *out = bf16_to_f32(h); return 0;
    case TSB_F16: memcpy(&h, s, 2); *out = f16_to_f32(h); return 0;
    case TSB_F8E4M3: *out = e4m3_to_f32(*s); return 0;
    case TSB_F8E5M2: *out = e5m2_to_f32(*s); return 0;
    default: return -1;
  }
}

/* one element of any pair: the fp8 pairs {f32, bf16, f16} <-> {e4m3fn, e5m2} go through f32 like
 * torch (every step but the last is exact); every other pair is copy_rects_ref.c's convert_elem */
static int convert_elem_fp8(const uint8_t* s, uint32_t sdt, uint8_t* d, uint32_t ddt, int nan_mode) {
  if (!is_fp8(sdt) && !is_fp8(ddt)) return convert_elem(s, sdt, d, ddt, nan_mode);
  if (sdt == ddt) {
    *d = *s;
    return 0;
  }
  uint32_t w;
  uint16_t h;
  if (load_f32(s, sdt, &w)) return -1;
  if (nan_mode && sdt == TSB_F16 && (w & 0x7fffffffu) > 0x7f800000u) w = 0x7fffffffu;
  switch (ddt) {
    case TSB_F8E4M3: if (is_fp8(sdt)) return -1; *d = f32_to_e4m3(w); return 0;
    case TSB_F8E5M2: if (is_fp8(sdt)) return -1; *d = f32_to_e5m2(w); return 0;
    case TSB_F32: if (!is_fp8(sdt)) return -1; memcpy(d, &w, 4); return 0;
    case TSB_BF16: if (!is_fp8(sdt)) return -1; h = f32_to_bf16(w, nan_mode); memcpy(d, &h, 2); return 0;
    case TSB_F16: if (!is_fp8(sdt)) return -1; h = f32_to_f16(w, nan_mode); memcpy(d, &h, 2); return 0;
    default: return -1;
  }
}

/* Flat conversion of n elements of any supported pair, fp8 included. */
int oracle_fp8_convert(const void* src, uint32_t sdt, void* dst, uint32_t ddt, uint64_t n, int nan_mode) {
  const uint32_t es = fp8_dtype_size(sdt), ed = fp8_dtype_size(ddt);
  if (!es || !ed) return -1;
  const uint8_t* s = (const uint8_t*)src;
  uint8_t* d = (uint8_t*)dst;
  for (uint64_t i = 0; i < n; ++i)
    if (convert_elem_fp8(s + i * es, sdt, d + i * ed, ddt, nan_mode)) return -1;
  return 0;
}

/* Move every rect element by element (single thread), fp8 pairs included.  Returns 0 or -1. */
int oracle_fp8_copy_rects(const tsb_rect_t* rects, uint64_t n, int nan_mode) {
  for (uint64_t i = 0; i < n; ++i) {
    const tsb_rect_t* r = &rects[i];
    const uint32_t es = fp8_dtype_size(r->src_dtype), ed = fp8_dtype_size(r->dst_dtype);
    if (!es || !ed || r->ndim < 1 || r->ndim > TSB_MAX_DIMS) return -1;
    uint64_t total = 1;
    for (uint32_t k = 0; k < r->ndim; ++k) total *= (uint64_t)r->extent[k];
    for (uint64_t e = 0; e < total; ++e) {
      uint64_t rem = e;
      int64_t so = 0, dof = 0;
      for (int k = (int)r->ndim - 1; k >= 0; --k) {
        const uint64_t ext = (uint64_t)r->extent[k], idx = rem % ext;
        rem /= ext;
        so += (int64_t)idx * r->src_stride[k];
        dof += (int64_t)idx * r->dst_stride[k];
      }
      if (convert_elem_fp8((const uint8_t*)(uintptr_t)r->src + so, r->src_dtype, (uint8_t*)(uintptr_t)r->dst + dof,
                           r->dst_dtype, nan_mode))
        return -1;
    }
  }
  return 0;
}

/* mode -> (src dtype, dst dtype, elements per unit): the fp8 modes, then copy_rects_ref.c's table */
static void fp8_mode_dtypes(uint32_t mode, uint32_t* sdt, uint32_t* ddt, uint32_t* elems) {
  static const uint32_t pairs[12][2] = {
      {TSB_F32, TSB_F8E4M3},  {TSB_F32, TSB_F8E5M2},  {TSB_BF16, TSB_F8E4M3}, {TSB_BF16, TSB_F8E5M2},
      {TSB_F16, TSB_F8E4M3},  {TSB_F16, TSB_F8E5M2},  {TSB_F8E4M3, TSB_F32},  {TSB_F8E5M2, TSB_F32},
      {TSB_F8E4M3, TSB_BF16}, {TSB_F8E5M2, TSB_BF16}, {TSB_F8E4M3, TSB_F16},  {TSB_F8E5M2, TSB_F16},
  };
  if (mode >= 22 && mode <= 45) { /* even: vector unit of 16 elements, odd: one element */
    *sdt = pairs[(mode - 22) / 2][0];
    *ddt = pairs[(mode - 22) / 2][1];
    *elems = mode % 2 == 0 ? 16 : 1;
    return;
  }
  mode_dtypes(mode, sdt, ddt, elems);
}

/* Replay (DevRect, DevTile) tables from tsb_plan_compile_host with the kernel's arithmetic, like
 * oracle_replay_plan, for plans that may contain fp8 modes.  Link-queue rects are byte moves and are
 * replayed the same way (their extra constraints are checked by oracle_replay_plan). */
int oracle_fp8_replay_plan(const void* rect_table, uint64_t n_rects, const uint32_t* tiles, uint64_t n_tiles,
                           uint32_t tile_units, int nan_mode) {
  const dev_rect_t* rects = (const dev_rect_t*)rect_table;
  for (uint64_t t = 0; t < n_tiles; ++t) {
    const uint32_t ri = tiles[2 * t], tir = tiles[2 * t + 1];
    if (ri >= n_rects) return -2;
    const dev_rect_t* r = &rects[ri];
    uint32_t sdt, ddt, elems;
    fp8_mode_dtypes(r->mode, &sdt, &ddt, &elems);
    if (sdt == 0xff) return -3;
    const uint32_t es = fp8_dtype_size(sdt), ed = fp8_dtype_size(ddt);
    if (es * elems != r->src_unit_bytes || ed * elems != r->dst_unit_bytes) return -4;
    const uint32_t tu = r->tile_units ? r->tile_units : tile_units;
    if (r->wide) {
      const uint32_t row = tir / r->split, seg = tir - row * r->split;
      if (row >= r->rows) return -5;
      const uint32_t ustart = seg * tu;
      if (ustart >= r->units_per_row) return -6;
      uint32_t ucount = r->units_per_row - ustart;
      if (ucount > tu) ucount = tu;
      int64_t so, dof;
      dev_row_offsets(r, row, &so, &dof);
      const uint8_t* s = (const uint8_t*)(uintptr_t)r->src + so + (int64_t)ustart * r->src_unit_bytes;
      uint8_t* d = (uint8_t*)(uintptr_t)r->dst + dof + (int64_t)ustart * r->dst_unit_bytes;
      if (oracle_fp8_convert(s, sdt, d, ddt, (uint64_t)ucount * elems, nan_mode)) return -7;
    } else {
      const uint32_t row0 = tir * r->split;
      if (row0 >= r->rows) return -8;
      uint32_t nrows = r->rows - row0;
      if (nrows > r->split) nrows = r->split;
      const uint32_t total = nrows * r->units_per_row;
      for (uint32_t idx = 0; idx < total; ++idx) {
        const uint32_t rr = r->magic ? (uint32_t)(((uint64_t)idx * r->magic) >> 32) : idx;
        const uint32_t c = idx - rr * r->units_per_row;
        if (c >= r->units_per_row) return -9; /* multiply-high division must be exact */
        int64_t so, dof;
        dev_row_offsets(r, row0 + rr, &so, &dof);
        const uint8_t* s = (const uint8_t*)(uintptr_t)r->src + so + (int64_t)c * r->src_unit_bytes;
        uint8_t* d = (uint8_t*)(uintptr_t)r->dst + dof + (int64_t)c * r->dst_unit_bytes;
        if (oracle_fp8_convert(s, sdt, d, ddt, elems, nan_mode)) return -7;
      }
    }
  }
  return 0;
}
