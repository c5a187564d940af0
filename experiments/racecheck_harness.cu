// experiments/racecheck_harness.cu -- torch-free driver for compute-sanitizer (racecheck / memcheck /
// synccheck) of the copy_rects kernel through the C-ABI.  Not part of the product library.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o experiments/racecheck_harness.bin \
//          experiments/racecheck_harness.cu -Iinclude -Ltorchstore_b200/lib -ltstore_b200 \
//          -Xlinker -rpath -Xlinker '$ORIGIN/../torchstore_b200/lib'
// Run:   compute-sanitizer --tool racecheck experiments/racecheck_harness.bin
//
// Workloads (each verified byte for byte on the host): narrow 1 KiB rows with an 8 KiB source pitch
// (the FSDP->TP hot case), wide rows, hundreds of tiny rects plus a large one, a strided
// destination; run twice -- copy warps only (TSB_LINK=0) and with every 16-byte rect routed through
// the link warp's TMA ring (TSB_LINK=2) -- and each plan is launched 3 times back to back so the
// self-resetting scheduler counters and the double-buffered claim slot are exercised across launches.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "tstore_b200.h"

#define CK(x)                                                                            \
  do {                                                                                   \
    cudaError_t e_ = (x);                                                                \
    if (e_ != cudaSuccess) {                                                             \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      exit(2);                                                                           \
    }                                                                                    \
  } while (0)
#define TSB(x)                                                                  \
  do {                                                                          \
    int s_ = (x);                                                               \
    if (s_ != TSB_OK) {                                                         \
      fprintf(stderr, "%s:%d %s -> %d: %s\n", __FILE__, __LINE__, #x, s_, tsb_last_error()); \
      exit(2);                                                                  \
    }                                                                           \
  } while (0)

struct Case {
  std::vector<tsb_rect_t> rects;
  // host-side description for verification: (src offset, dst offset, rows, row bytes, src pitch, dst pitch)
  struct Span { size_t so, dof, rows, row_bytes, sp, dp; };
  std::vector<Span> spans;
};

static void add_2d(Case& c, char* src, char* dst, size_t so, size_t dof, size_t rows, size_t row_bytes, size_t sp, size_t dp) {
  tsb_rect_t r;
  memset(&r, 0, sizeof(r));
  r.src = reinterpret_cast<uint64_t>(src + so);
  r.dst = reinterpret_cast<uint64_t>(dst + dof);
  r.ndim = 2;
  r.extent[0] = static_cast<int64_t>(rows);
  r.extent[1] = static_cast<int64_t>(row_bytes / 2);
  r.src_stride[0] = static_cast<int64_t>(sp);
  r.src_stride[1] = 2;
  r.dst_stride[0] = static_cast<int64_t>(dp);
  r.dst_stride[1] = 2;
  for (int i = 2; i < TSB_MAX_DIMS; ++i) r.extent[i] = 1;
  r.src_dtype = r.dst_dtype = TSB_U16;
  r.src_device = 0;
  c.rects.push_back(r);
  c.spans.push_back({so, dof, rows, row_bytes, sp, dp});
}

int main() {
  const size_t N = 96ull << 20;
  char *dsrc, *ddst;
  CK(cudaSetDevice(0));
  CK(cudaMalloc(&dsrc, N));
  CK(cudaMalloc(&ddst, N));
  std::vector<unsigned char> hsrc(N), hdst(N), expect(N);
  uint32_t x = 12345;
  for (size_t i = 0; i < N; ++i) {
    x = x * 1664525u + 1013904223u;
    hsrc[i] = static_cast<unsigned char>(x >> 24);
  }
  CK(cudaMemcpy(dsrc, hsrc.data(), N, cudaMemcpyHostToDevice));
  TSB(tsb_init());

  Case c;
  size_t so = 0, dof = 0;
  // 64 narrow-row rects: 512 rows x 1 KiB, source pitch 8 KiB, destination contiguous (wo at N=8)
  for (int i = 0; i < 8; ++i) {
    add_2d(c, dsrc, ddst, so + 1024 * i, dof, 512, 1024, 8192, 1024);
    dof += 512 * 1024;
  }
  so += 512 * 8192;
  // 3.5 KiB rows into a strided destination
  add_2d(c, dsrc, ddst, so, dof + 512, 256, 3584, 28672, 4096);
  so += 256 * 28672;
  dof += 256 * 4096;
  // one wide contiguous 24 MiB row
  add_2d(c, dsrc, ddst, so, dof, 1, 24u << 20, 24u << 20, 24u << 20);
  so += 24u << 20;
  dof += 24u << 20;
  // 300 tiny 1 KiB rects
  for (int i = 0; i < 300; ++i) {
    add_2d(c, dsrc, ddst, so, dof, 1, 1024, 1024, 1024);
    so += 2048;
    dof += 1024;
  }
  // misaligned rows (2-byte units: generic kernel path)
  add_2d(c, dsrc, ddst, so + 2, dof + 6, 100, 1002, 4096, 2048);

  int failures = 0;
  const char* modes[] = {"0", "2"};
  for (const char* mode : modes) {
    setenv("TSB_LINK", mode, 1);
    CK(cudaMemset(ddst, 0, N));
    memset(expect.data(), 0, N);
    for (const Case::Span& s : c.spans)
      for (size_t r = 0; r < s.rows; ++r) memcpy(&expect[s.dof + r * s.dp], &hsrc[s.so + r * s.sp], s.row_bytes);
    tsb_plan_t plan;
    TSB(tsb_plan_create(0, c.rects.data(), c.rects.size(), TSB_PLAN_DEFAULT, &plan));
    tsb_plan_info_t info;
    TSB(tsb_plan_info(plan, &info));
    for (int rep = 0; rep < 3; ++rep) {
      TSB(tsb_plan_launch(plan, nullptr));
      TSB(tsb_plan_wait(plan));
    }
    // one-shot path too (pooled tables, upload on the launch stream)
    TSB(tsb_copy_rects(0, c.rects.data(), c.rects.size(), TSB_PLAN_DEFAULT, nullptr));
    TSB(tsb_stream_sync(0, nullptr));
    CK(cudaMemcpy(hdst.data(), ddst, N, cudaMemcpyDeviceToHost));
    const bool ok = memcmp(hdst.data(), expect.data(), N) == 0;
    printf("TSB_LINK=%s: rects=%llu copy tiles=%llu link tiles=%llu grid=%u block=%u -> %s\n", mode,
           (unsigned long long)info.num_rects, (unsigned long long)info.num_tiles, (unsigned long long)info.num_link_tiles, info.grid,
           info.block, ok ? "bit-exact" : "MISMATCH");
    failures += !ok;
    TSB(tsb_plan_destroy(plan));
  }
  TSB(tsb_shutdown());
  return failures ? 1 : 0;
}
