// experiments/bulk_copy_probe.cu -- STANDALONE probe, not part of the product library.
//
// Question for round 2: does a TMA bulk pipeline (cp.async.bulk global->shared->global driven by one
// thread per CTA, mbarrier-signalled) move contiguous bytes faster than the product's LDG.128/STG.128
// path (a) inside one GPU's HBM and (b) when the source is a peer GPU over NVLink?
//
// Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o experiments/bulk_probe.bin experiments/bulk_copy_probe.cu
// Run:    experiments/bulk_probe.bin [peer]        (peer: source on GPU 0, kernel on GPU 1)
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#define CK(x)                                                                          \
  do {                                                                                 \
    cudaError_t e_ = (x);                                                              \
    if (e_ != cudaSuccess) {                                                           \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      exit(1);                                                                         \
    }                                                                                  \
  } while (0)

constexpr int kStages = 6;
constexpr uint32_t kChunk = 16384;  // bytes per bulk copy; 6 stages = 96 KiB smem -> 2 CTAs/SM

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// One thread per CTA drives the whole pipeline; chunk c of the buffer is handled by CTA (c % grid).
__global__ void __launch_bounds__(32, 2) bulk_copy_kernel(const char* __restrict__ src, char* __restrict__ dst, uint64_t nbytes) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t bars[kStages];
  if (threadIdx.x != 0) return;
  for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  const uint64_t nchunks = nbytes / kChunk;
  const uint64_t mine = (nchunks > blockIdx.x) ? (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  uint32_t phase_bits = 0;
  constexpr int kLag = kStages - 2;  // loads in flight; the stage being refilled was stored 2 commits ago
  for (uint64_t i = 0; i < mine + kLag; ++i) {
    if (i < mine) {
      const int s = static_cast<int>(i % kStages);
      if (i >= kStages) bulk_wait_read<1>();
      const uint64_t off = (blockIdx.x + i * gridDim.x) * static_cast<uint64_t>(kChunk);
      mbar_expect_tx(&bars[s], kChunk);
      bulk_g2s(smem + s * kChunk, src + off, kChunk, &bars[s]);
    }
    if (i >= kLag) {
      const uint64_t j = i - kLag;
      const int s = static_cast<int>(j % kStages);
      mbar_wait(&bars[s], (phase_bits >> s) & 1u);
      phase_bits ^= 1u << s;
      const uint64_t off = (blockIdx.x + j * gridDim.x) * static_cast<uint64_t>(kChunk);
      bulk_s2g(dst + off, smem + s * kChunk, kChunk);
      bulk_commit();
    }
  }
  bulk_wait_read<0>();
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Baseline: the product's data path in miniature.
__global__ void __launch_bounds__(256, 3) ldg_copy_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, uint64_t nvec) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x * 4;
  for (uint64_t i = blockIdx.x * blockDim.x * 4ull + threadIdx.x; i < nvec; i += stride) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (i + k * 256 < nvec)
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v[k].x), "=r"(v[k].y), "=r"(v[k].z), "=r"(v[k].w)
                     : "l"(src + i + k * 256));
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (i + k * 256 < nvec)
        asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + i + k * 256), "r"(v[k].x), "r"(v[k].y),
                     "r"(v[k].z), "r"(v[k].w)
                     : "memory");
  }
}

int main(int argc, char** argv) {
  const bool peer = argc > 1 && !strcmp(argv[1], "peer");
  const uint64_t nbytes = 4ull << 30;
  int exec_dev = peer ? 1 : 0;
  char *src, *dst;
  CK(cudaSetDevice(0));
  CK(cudaMalloc(&src, nbytes));
  CK(cudaMemset(src, 0x5a, nbytes));
  CK(cudaSetDevice(exec_dev));
  if (peer) CK(cudaDeviceEnablePeerAccess(0, 0));
  CK(cudaMalloc(&dst, nbytes));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, exec_dev));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const size_t smem = kStages * kChunk;
  CK(cudaFuncSetAttribute(bulk_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  for (int per_sm = 1; per_sm <= 2; ++per_sm) {
    float best = 1e9f;
    for (int it = 0; it < 6; ++it) {
      CK(cudaMemset(dst, 0, 1 << 20));
      CK(cudaEventRecord(e0));
      bulk_copy_kernel<<<sms * per_sm, 32, smem>>>(src, dst, nbytes);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaGetLastError());
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (it >= 2 && ms < best) best = ms;
    }
    printf("{\"kernel\": \"tma_bulk\", \"peer\": %d, \"ctas_per_sm\": %d, \"ms\": %.4f, \"payload_GBps\": %.1f}\n", peer, per_sm, best,
           nbytes / best / 1e6);
  }
  unsigned char probe[64];
  CK(cudaMemcpy(probe, dst + nbytes - 64, 64, cudaMemcpyDeviceToHost));
  for (int i = 0; i < 64; ++i)
    if (probe[i] != 0x5a) {
      fprintf(stderr, "tma_bulk copy produced wrong bytes\n");
      return 2;
    }
  for (int per_sm = 2; per_sm <= 4; ++per_sm) {
    float best = 1e9f;
    for (int it = 0; it < 6; ++it) {
      CK(cudaEventRecord(e0));
      ldg_copy_kernel<<<sms * per_sm, 256>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), nbytes / 16);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (it >= 2 && ms < best) best = ms;
    }
    printf("{\"kernel\": \"ldg128\", \"peer\": %d, \"ctas_per_sm\": %d, \"ms\": %.4f, \"payload_GBps\": %.1f}\n", peer, per_sm, best,
           nbytes / best / 1e6);
  }
  return 0;
}
