// Host tier of libtstore_b200 (SURVEY.md section 8 row f4): POSIX shared-memory segments for CPU
// clients / GPU-less volumes and a threaded strided mover for host rectangles.
//
// It replaces, for CPU-resident tensors only,
//   allocate_shared_tensor / SharedMemoryCache.allocate   transport/shared_memory.py:40-46,219-231
//   SharedMemoryDescriptor.attach                          transport/shared_memory.py:166-197
//   shm_tensor.copy_(tensor) / client_tensor.copy_(shm)    transport/shared_memory.py:373-374,473-476
// GPU tensors never take this path: they live in HBM arenas and move with copy_rects (the
// selection is by tensor device and transport type in transport/__init__.py, not a fallback).
#include <fcntl.h>
#include <pthread.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <cstring>
#include <string>
#include <vector>

#include "tsb_internal.h"

namespace tsb {
namespace {

uint32_t host_dtype_size(uint32_t dt) {
  switch (dt) {
    case TSB_U8: case TSB_F8E4M3: case TSB_F8E5M2: return 1;
    case TSB_U16: case TSB_F16: case TSB_BF16: return 2;
    case TSB_U32: case TSB_F32: return 4;
    case TSB_U64: case TSB_F64: return 8;
    default: return 0;
  }
}

struct HostRect {
  const char* src;
  char* dst;
  int64_t ext[TSB_MAX_DIMS];
  int64_t ss[TSB_MAX_DIMS];
  int64_t ds[TSB_MAX_DIMS];
  uint32_t nd;          // outer dims (rows)
  uint64_t rows;
  uint64_t run_bytes;   // contiguous bytes per row
};

// normalise one tsb_rect_t: split off the innermost contiguous run, keep the outer dims as rows
int prepare(const tsb_rect_t& in, uint64_t index, HostRect* out) {
  const std::string where = "host rect " + std::to_string(index) + ": ";
  if (in.ndim < 1 || in.ndim > TSB_MAX_DIMS) return fail(TSB_ERR_INVALID, where + "bad ndim");
  const uint32_t es = host_dtype_size(in.src_dtype);
  if (!es) return fail(TSB_ERR_INVALID, where + "unknown dtype");
  if (in.src_dtype != in.dst_dtype)
    return fail(TSB_ERR_UNSUPPORTED, where + "the host tier moves bytes; dtype casts run on the GPU path");
  if (!in.src || !in.dst) return fail(TSB_ERR_INVALID, where + "NULL src/dst");
  HostRect r{};
  r.src = reinterpret_cast<const char*>(in.src);
  r.dst = reinterpret_cast<char*>(in.dst);
  struct D { int64_t e, ss, ds; };
  std::vector<D> dims;
  for (uint32_t i = 0; i < in.ndim; ++i) {
    if (in.extent[i] < 0) return fail(TSB_ERR_INVALID, where + "negative extent");
    if (in.extent[i] == 0) { r.rows = 0; *out = r; return TSB_OK; }
    if (in.extent[i] == 1) continue;
    dims.push_back({in.extent[i], in.src_stride[i], in.dst_stride[i]});
  }
  int64_t run = es;
  while (!dims.empty() && dims.back().ss == run && dims.back().ds == run) {
    run *= dims.back().e;
    dims.pop_back();
  }
  if (run == es && !dims.empty() && dims.back().ss != static_cast<int64_t>(es)) run = es;  // element-granular gather
  r.run_bytes = static_cast<uint64_t>(run);
  r.nd = static_cast<uint32_t>(dims.size());
  r.rows = 1;
  for (uint32_t i = 0; i < r.nd; ++i) {
    r.ext[i] = dims[i].e;
    r.ss[i] = dims[i].ss;
    r.ds[i] = dims[i].ds;
    r.rows *= static_cast<uint64_t>(dims[i].e);
  }
  *out = r;
  return TSB_OK;
}

void copy_rows(const HostRect& r, uint64_t row_begin, uint64_t row_end) {
  for (uint64_t row = row_begin; row < row_end; ++row) {
    uint64_t rem = row;
    int64_t so = 0, dof = 0;
    for (int d = static_cast<int>(r.nd) - 1; d >= 0; --d) {
      const uint64_t e = static_cast<uint64_t>(r.ext[d]);
      const uint64_t idx = rem % e;
      rem /= e;
      so += static_cast<int64_t>(idx) * r.ss[d];
      dof += static_cast<int64_t>(idx) * r.ds[d];
    }
    memcpy(r.dst + dof, r.src + so, r.run_bytes);
  }
}

struct Job {
  const std::vector<HostRect>* rects;
  uint64_t lo, hi;  // byte range of the flattened (rect, row) space
};

void* worker(void* arg) {
  Job* j = static_cast<Job*>(arg);
  uint64_t pos = 0;
  for (const HostRect& r : *j->rects) {
    const uint64_t bytes = r.rows * r.run_bytes;
    const uint64_t begin = pos, end = pos + bytes;
    pos = end;
    if (!bytes || end <= j->lo || begin >= j->hi) continue;
    uint64_t rb = j->lo > begin ? (j->lo - begin + r.run_bytes - 1) / r.run_bytes : 0;
    uint64_t re = j->hi < end ? (j->hi - begin + r.run_bytes - 1) / r.run_bytes : r.rows;
    if (re > r.rows) re = r.rows;
    if (rb < re) copy_rows(r, rb, re);
  }
  return nullptr;
}

}  // namespace
}  // namespace tsb

using namespace tsb;

extern "C" {

int tsb_shm_create(const char* name, uint64_t nbytes, void** out_ptr) {
  if (!name || !out_ptr || nbytes == 0) return fail(TSB_ERR_INVALID, "tsb_shm_create: bad argument");
  int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
  if (fd < 0) return fail(TSB_ERR_INVALID, std::string("shm_open(") + name + "): " + strerror(errno));
  if (ftruncate(fd, static_cast<off_t>(nbytes)) != 0) {
    const std::string msg = std::string("ftruncate: ") + strerror(errno);
    close(fd);
    shm_unlink(name);
    return fail(TSB_ERR_NOMEM, msg);
  }
  // MAP_POPULATE: fault the pages now, not inside the first timed copy (the reference prefaults by
  // zero-filling the new shm tensor, transport/shared_memory.py:40-46)
  void* p = mmap(nullptr, nbytes, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_POPULATE, fd, 0);
  close(fd);
  if (p == MAP_FAILED) {
    const std::string msg = std::string("mmap: ") + strerror(errno);
    shm_unlink(name);
    return fail(TSB_ERR_NOMEM, msg);
  }
  *out_ptr = p;
  return TSB_OK;
}

int tsb_shm_attach(const char* name, uint64_t nbytes, void** out_ptr) {
  if (!name || !out_ptr || nbytes == 0) return fail(TSB_ERR_INVALID, "tsb_shm_attach: bad argument");
  int fd = shm_open(name, O_RDWR, 0600);
  if (fd < 0) return fail(TSB_ERR_NOTFOUND, std::string("shm_open(") + name + "): " + strerror(errno));
  struct stat st;
  if (fstat(fd, &st) != 0 || static_cast<uint64_t>(st.st_size) < nbytes) {
    close(fd);
    return fail(TSB_ERR_INVALID, std::string("segment ") + name + " is smaller than the descriptor says");
  }
  void* p = mmap(nullptr, nbytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) return fail(TSB_ERR_NOMEM, std::string("mmap: ") + strerror(errno));
  *out_ptr = p;
  return TSB_OK;
}

int tsb_shm_detach(void* ptr, uint64_t nbytes) {
  if (!ptr) return TSB_OK;
  if (munmap(ptr, nbytes) != 0) return fail(TSB_ERR_INVALID, std::string("munmap: ") + strerror(errno));
  return TSB_OK;
}

int tsb_shm_unlink(const char* name) {
  if (!name) return fail(TSB_ERR_INVALID, "name is NULL");
  if (shm_unlink(name) != 0 && errno != ENOENT) return fail(TSB_ERR_INVALID, std::string("shm_unlink: ") + strerror(errno));
  return TSB_OK;
}

int tsb_host_copy_rects(const tsb_rect_t* rects, uint64_t n, uint32_t threads) {
  if (n && !rects) return fail(TSB_ERR_INVALID, "rects is NULL");
  std::vector<HostRect> prepared;
  prepared.reserve(n);
  uint64_t total = 0;
  for (uint64_t i = 0; i < n; ++i) {
    HostRect r;
    int st = prepare(rects[i], i, &r);
    if (st) return st;
    if (r.rows == 0) continue;
    prepared.push_back(r);
    total += r.rows * r.run_bytes;
  }
  if (threads == 0) threads = 1;
  if (threads > 256) threads = 256;
  if (threads == 1 || total < (4u << 20)) {
    Job j{&prepared, 0, total};
    worker(&j);
    return TSB_OK;
  }
  std::vector<pthread_t> th(threads);
  std::vector<Job> jobs(threads);
  const uint64_t share = total / threads;
  for (uint32_t t = 0; t < threads; ++t) {
    jobs[t] = Job{&prepared, share * t, t + 1 == threads ? total : share * (t + 1)};
    if (pthread_create(&th[t], nullptr, worker, &jobs[t]) != 0) {
      for (uint32_t k = 0; k < t; ++k) pthread_join(th[k], nullptr);
      return fail(TSB_ERR_NOMEM, "pthread_create failed");
    }
  }
  for (uint32_t t = 0; t < threads; ++t) pthread_join(th[t], nullptr);
  return TSB_OK;
}

}  // extern "C"
