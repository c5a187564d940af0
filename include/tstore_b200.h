/*
 * tstore_b200.h -- C-ABI of libtstore_b200.so: the H100-native data plane behind torchstore's
 * weight-sync hot path (ts.put/ts.get, put_state_dict/get_state_dict, direct_weight_sync).
 *
 * The reference (meta-pytorch/torchstore) is 100% Python and reaches native code only through
 * third-party wheels (monarch.rdma, torchcomms, torch shm storages).  This header is what a
 * ctypes / cffi binding on the reference side would bind *instead of* those: every entry point
 * names the reference call site(s) it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - plain C, no torch types; pointers are CUDA device virtual addresses passed as void* / uint64_t
 *   - every function returns int status: 0 == TSB_OK, anything else is an error and
 *     tsb_last_error() returns a thread-local human-readable message
 *     (mirrors "RDMA read failed: conn code {res}", transport/torchcomms/buffer.py:238-239)
 *   - every data-moving call is stream-asynchronous; completion is observed with the event API
 *   - `stream` is a cudaStream_t (== CUstream) as an opaque void*; NULL selects the library's
 *     per-device copy stream (a non-blocking side stream, so copies overlap the caller's compute)
 *   - there is NO CPU fallback: without a CUDA device every data call returns TSB_ERR_CUDA
 */
#ifndef TSTORE_B200_H
#define TSTORE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSB_ABI_VERSION 9
#define TSB_MAX_DIMS 6

/* `flags` bit of the quantising plan calls (tsb_block_fp8_*, tsb_scaled_fp8_*, tsb_requant_fp8_*,
 * tsb_source_quant_*): power-of-two (UE8M0) scales.  Per group, with t = amax_c / 448 correctly rounded,
 *   scale_inv = t                                      if t's mantissa bits are 0 (a power of two, or Inf)
 *               (bits(t) & 0x7f800000) + 0x00800000    otherwise (the next power of two up)
 *   dst = e4m3fn(rn(x * (1 / scale_inv)))              (1 / scale_inv is exact; 0 for Inf)
 * still stored as float32.  The flag selects the kernels only: *_compile_host returns the same tables with and
 * without it.  The dequantising calls refuse it (TSB_ERR_INVALID), as they refuse every other bit. */
#define TSB_QUANT_UE8M0 1u

enum {
  TSB_OK = 0,
  TSB_ERR_INVALID = 1,    /* bad argument (AssertionError / ValueError on the Python side) */
  TSB_ERR_CUDA = 2,       /* a CUDA runtime/driver call failed (RuntimeError) */
  TSB_ERR_UNSUPPORTED = 3,/* e.g. a dtype pair the cast kernel does not implement */
  TSB_ERR_NOMEM = 4,      /* arena exhausted */
  TSB_ERR_NOTFOUND = 5,   /* unknown handle / plan / arena */
};

/* element types understood by the copy/cast kernel (same-dtype copies are byte moves and accept
 * any of them; cross-dtype pairs are listed in tsb_cast_supported) */
enum {
  TSB_U8 = 0,  /* also used for "opaque bytes": int8, bool, and fp8 when it is only moved */
  TSB_U16 = 1, /* opaque 2-byte (int16) */
  TSB_U32 = 2, /* opaque 4-byte (int32) */
  TSB_U64 = 3, /* opaque 8-byte (int64, complex64) */
  TSB_F16 = 4,
  TSB_BF16 = 5,
  TSB_F32 = 6,
  TSB_F64 = 7,
  TSB_F8E4M3 = 8, /* float8_e4m3fn: one side of a cast (a same-dtype fp8 move is TSB_U8) */
  TSB_F8E5M2 = 9, /* float8_e5m2: likewise */
  TSB_I8 = 10,    /* int8, valid ONLY as the dst_dtype of the rects of tsb_block_fp8_* and tsb_scaled_fp8_*: the
                   * destination is quantised to symmetric int8 (see tsb_bq_target_t).  Every rect of one such plan
                   * writes one dtype, TSB_F8E4M3 or TSB_I8 (a mix is TSB_ERR_INVALID); TSB_I8 with TSB_QUANT_UE8M0
                   * is TSB_ERR_INVALID.  Also valid as the src_dtype of the rects of tsb_dequant_fp8_* (an int8
                   * source dequantised; one plan reads one source dtype) and as the dst_dtype of
                   * tsb_source_quant_*_as (int8 staging).  The copy plan, the fused casts (tsb_cast_supported),
                   * the requantising calls and the other sides refuse it; a plain int8 move is TSB_U8.
                   * *_compile_host returns the same tables for TSB_I8 as for TSB_F8E4M3: the dtype selects the
                   * kernels only.  Libraries that predate it refuse TSB_I8 rects with TSB_ERR_UNSUPPORTED (or
                   * TSB_ERR_INVALID), so callers can detect it without an ABI version change. */
};

/* ------------------------------------------------------------------------------------------ */
/* lifecycle                                                                                   */
/* ------------------------------------------------------------------------------------------ */

int tsb_abi_version(void);
/* Thread-local message for the last non-zero status returned on this thread. */
const char* tsb_last_error(void);
/* Idempotent; creates per-device copy streams lazily.  Returns TSB_ERR_CUDA without a GPU. */
int tsb_init(void);
int tsb_shutdown(void);
int tsb_device_count(int* out_n);
/* Enable bidirectional P2P between two devices owned by THIS process (single-process multi-GPU).
 * Cross-process access is enabled implicitly by tsb_import_region.  Replaces the RDMA
 * connection handshake (transport/torchcomms/uniflow_buffer.py:200-229). */
int tsb_enable_peer_access(int device, int peer_device);
/* Number of kernels this library has launched since load (bench.py's "gpu_launches"). */
uint64_t tsb_launch_count(void);

/* ------------------------------------------------------------------------------------------ */
/* memory registration: the RDMABuffer replacement                                             */
/*   reference: RDMABuffer(to_byte_view(buf))          direct_weight_sync.py:143               */
/*              rdma_buffer.read_into / drop            direct_weight_sync.py:174,339           */
/*              SharedMemoryDescriptor.from_tensor      transport/shared_memory.py:115-137      */
/* ------------------------------------------------------------------------------------------ */

/* A picklable (plain bytes) description of `nbytes` of device memory owned by some process. */
typedef struct tsb_region {
  uint8_t ipc_handle[64]; /* cudaIpcMemHandle_t of the enclosing allocation */
  uint64_t offset;        /* byte offset of the region inside that allocation */
  uint64_t nbytes;
  uint64_t alloc_bytes;   /* size of the enclosing allocation */
  uint64_t local_ptr;     /* address in the exporting process (used when importer == exporter) */
  int32_t device;         /* CUDA ordinal in the exporting process */
  int32_t pid;            /* exporting process */
  uint64_t boot_id;       /* random per-library-load id: disambiguates recycled pids */
  uint64_t epoch;         /* driver-unique id of the enclosing allocation (CU_POINTER_ATTRIBUTE_BUFFER_ID):
                           * a different epoch at the same exporter address means the old allocation was
                           * freed and the address reused -> importers drop the stale mapping
                           * (registration-cache eviction, transport/torchcomms/cache.py:150-186) */
} tsb_region_t;

/* Describe [ptr, ptr+nbytes) so another process/GPU can map it.  Works on any cudaMalloc-backed
 * pointer, including sub-allocations of torch's caching allocator (base found with
 * cuMemGetAddressRange).  Fails with TSB_ERR_UNSUPPORTED for VMM/expandable-segment memory. */
int tsb_export_region(const void* ptr, uint64_t nbytes, tsb_region_t* out);
/* Map a region into this process and return a pointer usable from kernels running on
 * `device`.  Same-process regions resolve to local_ptr (peer access is enabled if the devices
 * differ).  Mappings are cached per (boot_id, ipc_handle): importing twice is free, like
 * SharedMemoryCache.attach (transport/shared_memory.py:233-244). */
int tsb_import_region(const tsb_region_t* region, int device, void** out_ptr);
/* Drop one cached mapping (== rdma_buffer.drop(), SharedMemoryCache.delete). */
int tsb_release_region(const tsb_region_t* region);
/* Drop every cached mapping (== TransportContext.clear()). */
int tsb_release_all(void);
/* Import-cache counters: live mappings, and mappings evicted because the exporter re-used the
 * address range for a new allocation (epoch changed). */
int tsb_import_stats(uint64_t* out_live, uint64_t* out_stale_evictions);

/* ------------------------------------------------------------------------------------------ */
/* the hot path: batched N-D rectangle gather with optional fused dtype cast                   */
/*   reference: asyncio.gather(rdma_buffer.read_into(...))      direct_weight_sync.py:338-340   */
/*              dest[dest_slices].copy_(recv[src_slices])        direct_weight_sync.py:343-350   */
/*              client_tensor.copy_(shm_tensor)                  transport/shared_memory.py:473-476 */
/*              shm_tensor.copy_(tensor, non_blocking=True)      transport/shared_memory.py:373-374 */
/*              local.to(transfer_dtype) / staging.copy_(src)    direct_weight_sync.py:133,167-168 */
/* ------------------------------------------------------------------------------------------ */

/* One axis-aligned hyper-rectangle to move.  `extent` counts ELEMENTS per dimension, strides are
 * in BYTES (so src/dst may have different element sizes when casting).  Dimension ndim-1 is the
 * fastest varying.  src may be local HBM or a peer-mapped address returned by
 * tsb_import_region; dst must be memory of the device the plan runs on (or peer memory for
 * "push" style puts). */
typedef struct tsb_rect {
  uint64_t src;
  uint64_t dst;
  int64_t extent[TSB_MAX_DIMS];
  int64_t src_stride[TSB_MAX_DIMS];
  int64_t dst_stride[TSB_MAX_DIMS];
  uint32_t ndim;      /* 1..TSB_MAX_DIMS (0-d tensors are passed as ndim=1, extent={1}) */
  uint32_t src_dtype; /* TSB_* */
  uint32_t dst_dtype; /* TSB_*; != src_dtype selects the fused cast */
  int32_t src_device; /* device that physically holds src (for NVLink fairness ordering); -1 unknown */
} tsb_rect_t;

typedef uint64_t tsb_plan_t;

enum {
  TSB_PLAN_DEFAULT = 0,
  TSB_PLAN_NO_INTERLEAVE = 1, /* keep tiles in rect order (debug / ablation) */
};

typedef struct tsb_plan_info {
  uint64_t num_rects;
  uint64_t num_tiles;         /* copy queue: tiles moved by the copy warps (LDG.128/STG.128) */
  uint64_t payload_bytes;     /* sum over rects of bytes written to dst */
  uint64_t src_bytes;         /* sum over rects of bytes read from src */
  uint64_t remote_src_bytes;  /* part of src_bytes with src_device != plan device (NVLink bytes) */
  uint64_t num_link_tiles;    /* link queue: tiles moved by the link warp's TMA bulk ring */
  uint64_t link_bytes;        /* part of remote_src_bytes that travels through the link queue */
  uint32_t grid;              /* CTAs per launch */
  uint32_t block;             /* threads per CTA: 256 copy threads (+32 link threads) */
  uint32_t tile_bytes;        /* copy-queue tile size */
  uint32_t num_vector_rects;  /* rects moved with 16-byte accesses */
  uint32_t link_tile_bytes;   /* link-queue tile size == one ring stage */
  uint32_t link_stages;       /* ring depth */
} tsb_plan_info_t;

/* Is (src_dtype -> dst_dtype) implemented?  Same dtype is always supported.  The fused casts, all
 * bit-exact with torch's .to():
 *   f32 <-> bf16, f32 <-> f16, bf16 <-> f16, f64 <-> f32
 *   {f32, bf16, f16} -> {f8e4m3, f8e5m2}: round to nearest even; e4m3fn has no Inf, so |x| > 464,
 *     +-Inf and NaN give 0x7F|sign; e5m2 gives +-Inf (0x7C|sign) for |x| >= 61440 and 0x7F|sign for NaN
 *     (an f16 NaN gives 0x7F: its widening to f32 on the GPU drops the sign, as in torch's CUDA .to())
 *   {f8e4m3, f8e5m2} -> {f32, bf16, f16}: exact
 * Casts run on the GPU only (tsb_host_copy_rects moves bytes). */
int tsb_cast_supported(uint32_t src_dtype, uint32_t dst_dtype);

/* Compile a list of rects into a device-resident tile table for `device` (the cached transfer
 * plan of DirectWeightSyncDest._build_plan, direct_weight_sync.py:221-317,334-335). */
int tsb_plan_create(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, tsb_plan_t* out);
int tsb_plan_info(tsb_plan_t plan, tsb_plan_info_t* out);
/* One persistent-kernel launch that moves every rect of the plan.  Asynchronous. */
int tsb_plan_run(tsb_plan_t plan, void* stream);
/* The whole per-sync sequence of DirectWeightSyncDest.pull (direct_weight_sync.py:319-350) in one
 * call, on the device's copy stream: [copy stream waits for everything queued on caller_stream]
 * -> start event -> kernel -> done event -> [caller_stream waits for the done event].  The events
 * belong to the plan and are reused.  caller_stream == NULL skips both fences. */
int tsb_plan_launch(tsb_plan_t plan, void* caller_stream);
/* Same with flags: TSB_LAUNCH_NO_FENCE_OUT leaves caller_stream free to run ahead of the copy (a put
 * that overlaps the actor's compute: the caller only promises not to overwrite the sources until it
 * has observed completion with tsb_plan_poll / tsb_plan_wait). */
enum { TSB_LAUNCH_DEFAULT = 0, TSB_LAUNCH_NO_FENCE_OUT = 1 };
int tsb_plan_launch_flags(tsb_plan_t plan, void* caller_stream, uint32_t flags);
/* Completion of the last tsb_plan_launch: 1 = bytes are in destination HBM, 0 = still running
 * (the await point of `await asyncio.gather(*reads)`, direct_weight_sync.py:338-340). */
int tsb_plan_poll(tsb_plan_t plan, int* out_done);
int tsb_plan_wait(tsb_plan_t plan);
/* Device time of the last tsb_plan_launch (start event -> done event). */
int tsb_plan_elapsed_ms(tsb_plan_t plan, float* out_ms);
int tsb_plan_destroy(tsb_plan_t plan);
/* Host-only (no CUDA call): compile and copy the kernel tables out, for inspection and for the
 * CPU test-suite, which replays them against the oracle.  out_rects: records of 192 bytes,
 * out_tiles: pairs of uint32 {rect, tile_in_rect}.  tile_units == 0 selects the default. */
int tsb_plan_compile_host(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, uint32_t tile_units,
                          void* out_rects, uint64_t n_rect_cap, uint64_t* out_n_rects, void* out_tiles,
                          uint64_t n_tile_cap, uint64_t* out_n_tiles, tsb_plan_info_t* out_info);
/* One-shot (uncached store-path puts/gets): compile, upload the tables and launch on ONE stream;
 * table buffers come from a recycled pinned/device pool, so a warm call does no cudaMalloc/cudaFree. */
int tsb_copy_rects(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, void* stream);
/* Table-pool counters (tests / diagnostics). */
int tsb_pool_stats(uint64_t* out_blocks, uint64_t* out_allocs, uint64_t* out_reuses);

/* ------------------------------------------------------------------------------------------ */
/* block-scaled FP8 destinations (DeepSeek-V3 / vLLM weight_block_size=[128, 128] layout):      */
/* the pull quantises while it gathers                                                          */
/* ------------------------------------------------------------------------------------------ */

/* One block-scaled destination: `batch` independent [rows, cols] matrices.  Every 128x128 block
 * (anchored at (0, 0); edge blocks are partial) gets one scale:
 *   amax = max |x| over the block (NaN if any x is NaN); amax_c = max(amax, 1e-4f) (NaN stays NaN)
 *   dst[i, j] = e4m3fn(rn(x[i, j] * (448 / amax_c)))  with torch's .to(float8_e4m3fn) rounding
 *   scale_inv[i / 128, j / 128] = amax_c / 448
 * with correctly rounded f32 divisions and multiply, x widened exactly to f32.  With TSB_I8 rects dst is int8:
 *   scale = 127 / amax_c;  scale_inv = amax_c / 127
 *   dst[i, j] = int8(sat[-128, 127](rne_int(rn(x[i, j] * scale))))  with NaN -> 0
 * (a NaN group: scale_inv NaN, dst 0; an Inf group: scale 0, scale_inv Inf, dst 0).  The same holds for the
 * groups of tsb_sq_target_t. */
typedef struct tsb_bq_target {
  uint64_t dst;       /* float8_e4m3fn (or int8 for TSB_I8 rects), contiguous [batch, rows, cols] */
  uint64_t scale_inv; /* float32, contiguous [batch, ceil(rows/128), ceil(cols/128)] */
  uint64_t batch, rows, cols;
} tsb_bq_target_t;

/* Compile a block-scaled pull: `rects` are ordinary source -> destination rectangles with
 * src_dtype in {TSB_F32, TSB_BF16, TSB_F16}, dst_dtype == TSB_F8E4M3 (or TSB_I8 for every rect) and dst inside
 * one target.
 * Every element of every target must be written by exactly one rect (TSB_ERR_INVALID otherwise: a
 * block's scale needs all of it).  The result is a plan like any other: tsb_plan_launch[_flags],
 * _run, _poll, _wait, _elapsed_ms, _info and _destroy accept it.  flags: 0 or TSB_QUANT_UE8M0 (not with TSB_I8). */
int tsb_block_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets,
                              uint64_t n_targets, uint32_t flags, tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the kernel tables out.  out_blocks: records of 32 bytes
 *   {u64 dst, u64 scale_inv, u32 dst_pitch, u16 rows, u16 cols, u32 first_piece, u16 n_pieces, u16 src_dtype}
 * out_pieces: records of 32 bytes
 *   {u64 src, i64 src_row_stride_bytes, u16 row0, u16 col0, u16 rows, u16 cols, u32 vector, u32 pad}
 * (row0/col0 relative to the block; vector: 16-byte loads).  A NULL table only reports its count. */
int tsb_block_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_bq_target_t* targets,
                               uint64_t n_targets, uint32_t flags, void* out_blocks, uint64_t block_cap,
                               uint64_t* out_n_blocks, void* out_pieces, uint64_t piece_cap, uint64_t* out_n_pieces);

/* ------------------------------------------------------------------------------------------ */
/* per-channel / per-tensor scaled FP8 destinations (compressed-tensors FP8, fbgemm-fp8, vLLM  */
/* quantization="fp8"): the pull quantises while it gathers                                     */
/* ------------------------------------------------------------------------------------------ */

enum { TSB_SCALE_PER_CHANNEL = 1, TSB_SCALE_PER_TENSOR = 2 };

/* One scaled destination: `batch` independent [rows, cols] matrices.  A group is one row
 * (TSB_SCALE_PER_CHANNEL; scale_inv is float32 [batch, rows]) or one whole matrix
 * (TSB_SCALE_PER_TENSOR; scale_inv is float32 [batch]).  Per group:
 *   amax = max |x| over the group (NaN if any x is NaN); amax_c = max(amax, 1e-4f) (NaN stays NaN)
 *   dst = e4m3fn(rn(x * (448 / amax_c)))  with torch's .to(float8_e4m3fn) rounding;  scale_inv = amax_c / 448
 * with correctly rounded f32 divisions and multiply, x widened exactly to f32.  TSB_I8 rects quantise into int8 with
 * the formula of tsb_bq_target_t. */
typedef struct tsb_sq_target {
  uint64_t dst;       /* float8_e4m3fn (or int8 for TSB_I8 rects), contiguous [batch, rows, cols] */
  uint64_t scale_inv; /* float32, contiguous, one per group */
  uint64_t batch, rows, cols;
  uint32_t granularity; /* TSB_SCALE_PER_CHANNEL or TSB_SCALE_PER_TENSOR */
  uint32_t pad;         /* 0 */
} tsb_sq_target_t;

/* Compile a scaled pull: rects as for tsb_block_fp8_plan_create; every element of every target must
 * be written by exactly one rect, and every group read from one source dtype (TSB_ERR_INVALID
 * naming the target and group otherwise).  A per-channel row of at most 32 KiB of source bytes is
 * quantised from shared memory after one read; per-tensor groups and longer rows take two passes
 * (amax, then quantise), reading the source twice.  The result is a plan like any other.
 * flags: 0 or TSB_QUANT_UE8M0 (not with TSB_I8). */
int tsb_scaled_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets,
                               uint64_t n_targets, uint32_t flags, tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the kernel tables out.  A NULL table only reports its count.
 * out_bands (row-staged path, one CTA each): records of 40 bytes
 *   {u64 dst, u64 scale_inv_of_row0, u32 cols, u32 rows, u32 first_piece, u32 n_pieces, u32 src_dtype, u32 pad}
 * out_pieces: records of 40 bytes
 *   {u64 src, i64 src_row_stride_bytes, u32 row0, u32 col0, u32 rows, u32 cols, u32 vector, u32 pad}
 *   (row0/col0 relative to the band; vector: 16-byte loads)
 * out_tiles (two-pass path, one CTA per pass each): records of 56 bytes, sorted by group
 *   {u64 src, i64 src_row_stride_bytes, u64 dst, u64 scale_inv_or_0, u32 dst_pitch, u32 rows, u32 cols,
 *    u32 group, u32 src_dtype, u32 vector}
 *   (scale_inv_or_0: non-zero in exactly one tile per group, the one that writes its scale)
 * out_n_groups: the number of two-pass groups (amax words). */
int tsb_scaled_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_sq_target_t* targets,
                                uint64_t n_targets, uint32_t flags, void* out_bands, uint64_t band_cap,
                                uint64_t* out_n_bands, void* out_pieces, uint64_t piece_cap, uint64_t* out_n_pieces,
                                void* out_tiles, uint64_t tile_cap, uint64_t* out_n_tiles, uint64_t* out_n_groups);

/* ------------------------------------------------------------------------------------------ */
/* dequantising pulls: block-, channel- or tensor-scaled float8_e4m3fn (or int8) sources into   */
/* f32, bf16 or f16 destinations                                                                */
/* ------------------------------------------------------------------------------------------ */

enum { TSB_SCALE_PER_BLOCK = 3 };

/* One scaled source shard: `batch` contiguous [rows, cols] float8_e4m3fn (or int8) matrices whose first
 * element sits at (row0, col0) of the global tensor's last two dims.  Scales are anchored at the
 * global origin (checkpoint semantics), and the scale tensor holds exactly the groups the shard
 * touches:
 *   TSB_SCALE_PER_BLOCK    float32 [batch, ceil((row0+rows)/128) - row0/128, ceil((col0+cols)/128) - col0/128]
 *   TSB_SCALE_PER_CHANNEL  float32 [batch, rows]
 *   TSB_SCALE_PER_TENSOR   float32 [batch]
 * Element (b, i, j) of the shard becomes  dst = to_dst(f32(q[b, i, j]) * scale[b, g(i, j)])  with
 * g = ((row0+i)/128 - row0/128, (col0+j)/128 - col0/128) per block, i per channel and nothing per
 * tensor; f32(q) is exact, the multiply one correctly rounded f32 multiply (no flush to zero), and
 * to_dst the fused cast's f32 -> bf16 / f16 narrowing (identity for f32). */
typedef struct tsb_dq_source {
  uint64_t src;         /* float8_e4m3fn or int8 (the rects' src_dtype) as seen from the plan's device */
  uint64_t scale;       /* float32, contiguous, as seen from the plan's device */
  uint64_t batch, rows, cols;
  uint64_t row0, col0;  /* global offset of the shard in the last two dims (the block phase) */
  uint32_t granularity; /* TSB_SCALE_PER_BLOCK, TSB_SCALE_PER_CHANNEL or TSB_SCALE_PER_TENSOR */
  uint32_t pad;         /* 0 */
} tsb_dq_source_t;

/* Compile a dequantising pull: `rects` are ordinary source -> destination rectangles with src_dtype
 * == TSB_F8E4M3 or TSB_I8, dst_dtype in {TSB_F32, TSB_BF16, TSB_F16} and src inside one source (TSB_ERR_INVALID
 * naming the rect or source otherwise).  Every rect of one plan reads one source dtype (a mix of TSB_F8E4M3 and
 * TSB_I8 is TSB_ERR_INVALID); for TSB_I8, f32(q) is (float)(int8_t)q.  The tile table is the same for either.  Elements no rect reads are left alone.  The result is a plan
 * like any other.  flags: reserved, pass 0 (TSB_QUANT_UE8M0 is refused: a float32 scale dequantises the
 * same whatever its format). */
int tsb_dequant_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                uint64_t n_sources, uint32_t flags, tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the tile table out (one CTA per tile).  out_tiles: records
 * of 56 bytes
 *   {u64 src, u64 dst, u64 scale, i64 src_row_stride_bytes, i64 dst_row_stride_bytes, u32 rows, u32 cols,
 *    u16 scale_step_bytes, u8 dst_dtype, u8 vector, u32 pad}
 * (scale: the float32 scale of the tile's first row; scale_step_bytes: 4 per channel, else 0; vector:
 * 16-byte accesses on both sides).  A NULL table only reports its count. */
int tsb_dequant_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                 uint64_t n_sources, uint32_t flags, void* out_tiles, uint64_t tile_cap,
                                 uint64_t* out_n_tiles);

/* ------------------------------------------------------------------------------------------ */
/* requantising pulls: block-, channel- or tensor-scaled float8_e4m3fn sources into block-,     */
/* channel- or tensor-scaled float8_e4m3fn destinations                                         */
/* ------------------------------------------------------------------------------------------ */

/* Compile a requantising pull: `rects` are ordinary source -> destination rectangles with src_dtype ==
 * dst_dtype == TSB_F8E4M3, src inside one source and dst inside one target.  `sources` are as for
 * tsb_dequant_fp8_plan_create; `targets` as for tsb_scaled_fp8_plan_create, except that granularity may also
 * be TSB_SCALE_PER_BLOCK (scale_inv float32 [batch, ceil(rows/128), ceil(cols/128)], 128x128 blocks anchored
 * at (0, 0) as in tsb_block_fp8_plan_create).  Every element becomes
 *   x = f32(q) * scale[g_src]   (what tsb_dequant_fp8_plan_create writes into an f32 destination)
 * and is quantised with the target's formula as if x were an f32 source, so the result equals a dequantising
 * pull into f32 followed by a quantising pull from it, byte for byte.  A rect's source rows must be rows of
 * its source shard (TSB_ERR_INVALID naming the rect otherwise); every element of every target must be
 * written by exactly one rect (TSB_ERR_INVALID naming the target and group otherwise).  Block targets and
 * per-channel rows of at most 32 KiB read each source byte once; per-tensor groups and longer rows take two
 * passes.  The result is a plan like any other.  flags: 0 or TSB_QUANT_UE8M0 (the target's formula with
 * power-of-two scales). */
int tsb_requant_fp8_plan_create(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                uint64_t n_sources, const tsb_sq_target_t* targets, uint64_t n_targets, uint32_t flags,
                                tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the kernel tables out.  A NULL table only reports its count.
 * out_units (staged path, one CTA each: a 128x128 block, or a band of whole per-channel rows): records of 40 bytes
 *   {u64 dst, u64 scale_inv, u32 pitch, u32 rows, u32 cols, u32 first_piece, u32 n_pieces, u32 per_row}
 *   (scale_inv: the block's, or the band's first row's; per_row: 1 for bands, one scale per row)
 * out_pieces: records of 56 bytes
 *   {u64 src, i64 src_row_stride_bytes, u64 scale, u32 row0, u32 col0, u32 rows, u32 cols, u32 scale_step_bytes,
 *    u32 vector, u32 col_phase, u32 col_blocks}
 *   (scale: the float32 source scale of the piece's first element; scale_step_bytes: to the next row's, 0 unless
 *   the source is per channel; col_blocks: 1 for block sources, whose scale advances 4 bytes every 128 columns
 *   counted from col_phase; row0/col0 relative to the unit; vector: 16-byte loads)
 * out_tiles (two-pass path, one CTA per pass each): records of 64 bytes, sorted by group
 *   {u64 src, i64 src_row_stride_bytes, u64 scale, u64 dst, u64 scale_inv_or_0, u32 dst_pitch, u32 rows, u32 cols,
 *    u32 group, u32 scale_step_bytes, u32 vector}
 *   (scale_inv_or_0: non-zero in exactly one tile per group, the one that writes its scale)
 * out_n_groups: the number of two-pass groups (amax words). */
int tsb_requant_fp8_compile_host(int device, const tsb_rect_t* rects, uint64_t n, const tsb_dq_source_t* sources,
                                 uint64_t n_sources, const tsb_sq_target_t* targets, uint64_t n_targets, uint32_t flags,
                                 void* out_units, uint64_t unit_cap, uint64_t* out_n_units, void* out_pieces,
                                 uint64_t piece_cap, uint64_t* out_n_pieces, void* out_tiles, uint64_t tile_cap,
                                 uint64_t* out_n_tiles, uint64_t* out_n_groups);

/* ------------------------------------------------------------------------------------------ */
/* source-side quantisation: a publisher refreshes block-, channel- or tensor-scaled           */
/* float8_e4m3fn (or int8) staging from its live bf16/f16/f32 shards                            */
/* ------------------------------------------------------------------------------------------ */

/* One shard to quantise: `batch` contiguous [rows, cols] matrices of src_dtype at src, whose first element
 * sits at (row0, col0) of the global tensor's last two dims.  Groups are shard-local and anchored at the
 * global origin, exactly as a tsb_dq_source_t describes them: per block the intersection of a global
 * 128x128 block with the shard, per channel the shard's part of one row, per tensor the shard's [rows, cols]
 * matrix.  scale_inv has the shape of tsb_dq_source_t's scale.  Per group the formula of
 * tsb_bq_target_t / tsb_sq_target_t applies (amax_c = max(amax, 1e-4f), dst = e4m3fn(rn(x * 448 / amax_c)),
 * scale_inv = amax_c / 448; a NaN poisons its group). */
typedef struct tsb_source_quant_target {
  uint64_t src;         /* TSB_F32 / TSB_BF16 / TSB_F16, contiguous [batch, rows, cols], element-aligned */
  uint64_t dst;         /* float8_e4m3fn (int8 with tsb_source_quant_*_as(TSB_I8)), contiguous [batch, rows, cols] */
  uint64_t scale_inv;   /* float32, contiguous, one per group */
  uint64_t batch, rows, cols;
  uint64_t row0, col0;  /* global offset of the shard in the last two dims (the block phase) */
  uint32_t src_dtype;   /* TSB_F32, TSB_BF16 or TSB_F16 */
  uint32_t granularity; /* TSB_SCALE_PER_BLOCK, TSB_SCALE_PER_CHANNEL or TSB_SCALE_PER_TENSOR */
} tsb_source_quant_target_t;

/* Compile a source-side quantisation of `n` targets (TSB_ERR_INVALID naming the target otherwise).  Blocks and
 * per-channel rows of at most 32 KiB of source bytes are quantised from registers after one read, one CTA per
 * block or band of rows; per-tensor groups and longer rows take two passes (amax, then quantise).  The result is a plan like any other: tsb_plan_launch[_flags],
 * _run, _poll, _wait, _elapsed_ms, _info and _destroy accept it.  flags: 0 or TSB_QUANT_UE8M0. */
int tsb_source_quant_plan_create(int device, const tsb_source_quant_target_t* targets, uint64_t n, uint32_t flags,
                                 tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the kernel tables out.  A NULL table only reports its count.
 * out_units (one-read path: a block's part of the shard, or a band of whole per-channel rows; grouped by src_dtype,
 * bf16 then f16 then f32): records of 48 bytes
 *   {u64 src, u64 dst, u64 scale_inv, u32 src_pitch, u32 dst_pitch, u32 rows, u32 cols, u32 per_row,
 *    u16 src_dtype, u16 vec}
 *   (scale_inv: the block's, or the band's first row's; per_row: 1 for bands, one scale per row; pitches in
 *   bytes; vec: 16-byte loads)
 * out_tiles (two-pass path): the 56-byte tile records of tsb_scaled_fp8_compile_host, sorted by group
 * out_n_groups: the number of two-pass groups (amax words). */
int tsb_source_quant_compile_host(int device, const tsb_source_quant_target_t* targets, uint64_t n, uint32_t flags,
                                  void* out_units, uint64_t unit_cap, uint64_t* out_n_units, void* out_tiles,
                                  uint64_t tile_cap, uint64_t* out_n_tiles, uint64_t* out_n_groups);
/* The same two calls with the staging format named: dst_dtype TSB_F8E4M3 (exactly the calls above) or TSB_I8,
 * symmetric int8 with the formula of tsb_bq_target_t's TSB_I8 rects (amax_c = max(amax, 1e-4f), scale_inv =
 * amax_c / 127, dst = sat_s8(rne(rn(x * 127 / amax_c))), NaN -> 0; a NaN group gets a NaN scale, an Inf group an
 * Inf scale, both all zeros).  Any other dst_dtype, and TSB_I8 with TSB_QUANT_UE8M0, is TSB_ERR_INVALID.  The
 * tables do not depend on dst_dtype. */
int tsb_source_quant_plan_create_as(int device, const tsb_source_quant_target_t* targets, uint64_t n, uint32_t dst_dtype,
                                    uint32_t flags, tsb_plan_t* out);
int tsb_source_quant_compile_host_as(int device, const tsb_source_quant_target_t* targets, uint64_t n,
                                     uint32_t dst_dtype, uint32_t flags, void* out_units, uint64_t unit_cap,
                                     uint64_t* out_n_units, void* out_tiles, uint64_t tile_cap, uint64_t* out_n_tiles,
                                     uint64_t* out_n_groups);

/* ------------------------------------------------------------------------------------------ */
/* transposing pulls: input-major sources into output-major destinations                       */
/* ------------------------------------------------------------------------------------------ */

/* Compile a transposing pull: `rects` are ordinary tsb_rect_t with 2 <= ndim <= TSB_MAX_DIMS whose destination is
 * contiguous along dim ndim-1 (dst_stride == its element size) and whose source is contiguous along dim ndim-2
 * (src_stride == its element size); a dim of extent 1 is exempt from its rule.  The outer dims take any strides, and
 * src may be local or peer-mapped.  Element (o, i, j) becomes dst[o, i, j] = to_dst(src[o, i, j]) as for the copy
 * plan, but the mover reads 16-byte sectors along the source's dim ndim-2 and writes them along the destination's
 * dim ndim-1 (a 2-D transpose through shared memory).  Same-dtype moves of 1-, 2-, 4- and 8-byte elements and every
 * pair of tsb_cast_supported are accepted; any other pair is TSB_ERR_UNSUPPORTED, any other rect TSB_ERR_INVALID,
 * both naming "rect N".  The result is a plan like any other: tsb_plan_launch[_flags], _run, _poll, _wait,
 * _elapsed_ms, _info and _destroy accept it.  flags: reserved, pass 0. */
int tsb_transpose_plan_create(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, tsb_plan_t* out);
/* Host-only (no CUDA call): compile and copy the tile table out (grouped by dtype pair, rect order inside a group).
 * out_tiles: records of 48 bytes
 *   {u64 src, u64 dst, i64 src_stride_bytes, i64 dst_stride_bytes, u32 rows, u32 cols, u8 src_dtype, u8 dst_dtype,
 *    u8 vector, u8 pad, u32 pad}
 * (tile element (i, j), i < rows, j < cols, moves from src + i * src_elem + j * src_stride_bytes to
 * dst + i * dst_stride_bytes + j * dst_elem; tiles are at most 64 x 64 elements for 1- and 2-byte sources, 32 x 32
 * otherwise; vector bit 0: 16-byte source loads, bit 1: 16-byte destination stores, each set only where that side's
 * address and stride are 16-byte aligned).  A NULL table only reports its count. */
int tsb_transpose_compile_host(int device, const tsb_rect_t* rects, uint64_t n, uint32_t flags, void* out_tiles,
                               uint64_t tile_cap, uint64_t* out_n_tiles);

/* ------------------------------------------------------------------------------------------ */
/* streams and events (the await points of the reference's coroutines)                         */
/* ------------------------------------------------------------------------------------------ */

int tsb_stream_create(int device, void** out_stream);
int tsb_stream_destroy(void* stream);
int tsb_stream_sync(int device, void* stream); /* stream == NULL: the device's copy stream */
/* The library's per-device copy stream (what NULL means above). */
int tsb_copy_stream(int device, void** out_stream);

int tsb_event_create(int device, int timing, void** out_event);
int tsb_event_record(void* event, int device, void* stream);
int tsb_stream_wait_event(int device, void* stream, void* event);
/* 1 = complete, 0 = still running */
int tsb_event_query(void* event, int* out_done);
int tsb_event_sync(void* event);
int tsb_event_elapsed_ms(void* start, void* stop, float* out_ms);
int tsb_event_destroy(void* event);

/* ------------------------------------------------------------------------------------------ */
/* HBM arena: the storage volume's memory                                                      */
/*   reference: allocate_shared_tensor / SharedMemoryCache.allocate                            */
/*              transport/shared_memory.py:40-46,219-231 (host shm segments -> one HBM slab)    */
/* ------------------------------------------------------------------------------------------ */

typedef uint64_t tsb_arena_t;

typedef struct tsb_arena_stats {
  uint64_t capacity;
  uint64_t in_use;
  uint64_t high_water;
  uint64_t num_blocks;
  uint64_t base;      /* device address of the slab */
} tsb_arena_stats_t;

/* One cudaMalloc'd slab on `device`, exportable as a single region.  Blocks are carved
 * ring-buffer style (first fit from a rotating cursor, coalescing frees). */
int tsb_arena_create(int device, uint64_t capacity_bytes, tsb_arena_t* out);
int tsb_arena_alloc(tsb_arena_t arena, uint64_t nbytes, uint64_t align, void** out_ptr);
int tsb_arena_free(tsb_arena_t arena, void* ptr);
int tsb_arena_stats(tsb_arena_t arena, tsb_arena_stats_t* out);
int tsb_arena_destroy(tsb_arena_t arena);

/* ------------------------------------------------------------------------------------------ */
/* host staging (pinned memory + async copies) for CPU-resident callers                        */
/*   reference: pin_memory / cudaHostRegister         transport/shared_memory.py:55-96          */
/* ------------------------------------------------------------------------------------------ */

int tsb_host_alloc(uint64_t nbytes, void** out_ptr);
int tsb_host_free(void* ptr);
int tsb_host_register(void* ptr, uint64_t nbytes);
int tsb_host_unregister(void* ptr);
enum { TSB_H2D = 1, TSB_D2H = 2, TSB_D2D = 3 };
int tsb_memcpy_async(int device, void* dst, const void* src, uint64_t nbytes, int kind, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* host tier: POSIX shm segments + strided host mover, for CPU tensors and GPU-less volumes     */
/*   reference: allocate_shared_tensor / SharedMemoryCache   transport/shared_memory.py:40-46,210-260 */
/*              shm_tensor.copy_(t) / client_tensor.copy_(shm) transport/shared_memory.py:373-374,473-476 */
/*   These calls need no CUDA device.  GPU tensors never use them (no fallback: the tier is chosen */
/*   by tensor device / transport type).                                                          */
/* ------------------------------------------------------------------------------------------ */

/* Create (exclusive) / attach / detach / unlink a named segment ("/name").  create prefaults. */
int tsb_shm_create(const char* name, uint64_t nbytes, void** out_ptr);
int tsb_shm_attach(const char* name, uint64_t nbytes, void** out_ptr);
int tsb_shm_detach(void* ptr, uint64_t nbytes);
int tsb_shm_unlink(const char* name);
/* Same descriptors as tsb_copy_rects with HOST pointers and src_dtype == dst_dtype: strided byte
 * moves on `threads` host threads (byte-balanced split of the flattened row space). */
int tsb_host_copy_rects(const tsb_rect_t* rects, uint64_t n, uint32_t threads);

#ifdef __cplusplus
}
#endif
#endif /* TSTORE_B200_H */
