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

#define TSB_ABI_VERSION 2
#define TSB_MAX_DIMS 6

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
  TSB_U8 = 0,  /* also used for "opaque bytes": int8, bool, fp8 ... */
  TSB_U16 = 1, /* opaque 2-byte (int16) */
  TSB_U32 = 2, /* opaque 4-byte (int32) */
  TSB_U64 = 3, /* opaque 8-byte (int64, complex64) */
  TSB_F16 = 4,
  TSB_BF16 = 5,
  TSB_F32 = 6,
  TSB_F64 = 7,
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

/* Is (src_dtype -> dst_dtype) implemented?  Same dtype is always supported. */
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
