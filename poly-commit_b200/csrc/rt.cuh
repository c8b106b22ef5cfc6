// Thin runtime layer: kernel launch, device memory and stream helpers.
//
// Every kernel in this library is a functor ("body") invoked once per logical thread by one of the
// generic __global__ wrappers below.  When the sources are compiled by a host compiler with
// -DPCGPU_EMUL (tests/host_emul only -- a unit-test harness, never shipped, never loaded by the
// package) the same bodies run in a serial loop and "device" memory is host memory, which lets the
// limb schedules, digit recoding, bucket bookkeeping and scan logic be checked on a machine
// without a GPU.  The product build (nvcc, sm_90a) contains no host execution path.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <type_traits>

#ifndef PCGPU_EMUL
#include <cuda_runtime.h>
#endif

namespace pcgpu {
namespace rt {

enum : int {
  OK = 0,
  E_CUDA = -1,
  E_OOM = -2,
  E_BADARG = -3,
  E_LEN = -4,
  E_RANGE = -5,
  E_DEGREE = -6,
  E_HIDING = -7,
};

// number of kernels this library has launched in the process (bench.py reports it as gpu_launches)
inline std::atomic<uint64_t> &launch_counter() { static std::atomic<uint64_t> c{0}; return c; }

#ifdef PCGPU_EMUL
// ------------------------------------------------------------------ host emulation (tests only)
typedef void *stream_t;
inline int dev_malloc(void **p, size_t bytes) { *p = ::malloc(bytes ? bytes : 1); return *p ? OK : E_OOM; }
inline void dev_free(void *p) { ::free(p); }
inline int dev_memset(void *p, int v, size_t bytes, stream_t) { memset(p, v, bytes); return OK; }
inline int copy_h2d(void *d, const void *h, size_t bytes, stream_t) { memcpy(d, h, bytes); return OK; }
inline int copy_d2h(void *h, const void *d, size_t bytes, stream_t) { memcpy(h, d, bytes); return OK; }
inline int copy_d2d(void *d, const void *s, size_t bytes, stream_t) { memmove(d, s, bytes); return OK; }
inline int stream_sync(stream_t) { return OK; }
inline int last_error() { return OK; }
typedef int event_t;
inline int event_create(event_t *e) { *e = 0; return OK; }
inline void event_destroy(event_t) {}
inline int event_record(event_t, stream_t) { return OK; }
inline int stream_wait_event(stream_t, event_t) { return OK; }
inline int host_alloc_pinned(void **p, size_t bytes) { *p = ::malloc(bytes ? bytes : 1); return *p ? OK : E_OOM; }
inline void host_free_pinned(void *p) { ::free(p); }

template <int BLOCK, class Body>
inline int launch(const Body &body, size_t n, stream_t) {
  for (size_t i = 0; i < n; i++) body(i);
  return OK;
}
template <class T> inline T atomic_add(T *p, T v) { T o = *p; *p = o + v; return o; }
template <class T> inline T atomic_or(T *p, T v) { T o = *p; *p = o | v; return o; }
#define PCGPU_KERNEL_DEV inline
// Persistent bodies pull work from a global counter: next_task() returns this lane's next task index.
inline uint32_t next_task(uint32_t *counter) { return atomic_add(counter, 1u); }
template <int BLOCK, class Body>
inline int launch_persistent(const Body &body, stream_t) { body(0); return OK; }
// threads of one resident wave of `Body` (host emulation: a small number so multi-iteration paths are exercised)
template <int BLOCK, int MINB, class Body> inline int launch_occ(const Body &body, size_t n, stream_t s) { return launch<BLOCK>(body, n, s); }
template <int BLOCK, int MINB, class Body> inline int resident_threads_occ(size_t *out) { *out = 48; return OK; }
// Block-cooperative bodies: body(block_id, shared_memory).  Work inside the body is written as
// PCGPU_BLOCK_FOR loops separated by PCGPU_BLOCK_SYNC(); anything that must survive a sync lives in shared memory.
#define PCGPU_BLOCK_FOR(i, n) for (uint32_t i = 0; i < (uint32_t)(n); i++)
#define PCGPU_BLOCK_SYNC() do { } while (0)
// warp vote over a FULL warp (every lane must reach it): also the point where diverged lanes reconverge
#define PCGPU_WARP_ANY(x) (x)
template <int BLOCK, class Body>
inline int launch_blocks(const Body &body, size_t nblocks, size_t smem_bytes, stream_t) {
  uint32_t *smem = (uint32_t *)::malloc(smem_bytes ? smem_bytes : 16);
  if (!smem) return E_OOM;
  for (size_t b = 0; b < nblocks; b++) body(b, smem);
  ::free(smem);
  return OK;
}

template <int BLOCK, int MINB, class Body>
inline int launch_blocks_occ(const Body &body, size_t nblocks, size_t smem_bytes, stream_t s) { return launch_blocks<BLOCK>(body, nblocks, smem_bytes, s); }

#else
// ------------------------------------------------------------------ CUDA (the product)
typedef cudaStream_t stream_t;

inline int map_cuda(cudaError_t e) {
  if (e == cudaSuccess) return OK;
  if (e == cudaErrorMemoryAllocation) return E_OOM;
  return E_CUDA;
}
inline int dev_malloc(void **p, size_t bytes) { return map_cuda(cudaMalloc(p, bytes ? bytes : 1)); }
inline void dev_free(void *p) { if (p) cudaFree(p); }
inline int dev_memset(void *p, int v, size_t bytes, stream_t s) { return map_cuda(cudaMemsetAsync(p, v, bytes, s)); }
inline int copy_h2d(void *d, const void *h, size_t bytes, stream_t s) { return map_cuda(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s)); }
inline int copy_d2h(void *h, const void *d, size_t bytes, stream_t s) { return map_cuda(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s)); }
inline int copy_d2d(void *d, const void *s_, size_t bytes, stream_t s) { return map_cuda(cudaMemcpyAsync(d, s_, bytes, cudaMemcpyDeviceToDevice, s)); }
inline int stream_sync(stream_t s) { return map_cuda(cudaStreamSynchronize(s)); }
inline int last_error() { return map_cuda(cudaGetLastError()); }
typedef cudaEvent_t event_t;
inline int event_create(event_t *e) { return map_cuda(cudaEventCreateWithFlags(e, cudaEventDisableTiming)); }
inline void event_destroy(event_t e) { cudaEventDestroy(e); }
inline int event_record(event_t e, stream_t s) { return map_cuda(cudaEventRecord(e, s)); }
inline int stream_wait_event(stream_t s, event_t e) { return map_cuda(cudaStreamWaitEvent(s, e, 0)); }
inline int host_alloc_pinned(void **p, size_t bytes) { return map_cuda(cudaMallocHost(p, bytes ? bytes : 1)); }
inline void host_free_pinned(void *p) { if (p) cudaFreeHost(p); }

template <class Body, int BLOCK>
__global__ void __launch_bounds__(BLOCK) run_kernel(const Body body, size_t n) {
  size_t tid = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (tid < n) body(tid);
}

template <int BLOCK, class Body>
inline int launch(const Body &body, size_t n, stream_t s) {
  if (n == 0) return OK;
  size_t grid = (n + BLOCK - 1) / BLOCK;
  run_kernel<Body, BLOCK><<<(unsigned)grid, BLOCK, 0, s>>>(body, n);
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  return last_error();
}
// same, with a minimum number of resident blocks per SM (caps registers; for latency-bound bodies that want more warps)
template <class Body, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) run_kernel_occ(const Body body, size_t n) {
  size_t tid = (size_t)blockIdx.x * BLOCK + threadIdx.x;
  if (tid < n) body(tid);
}
template <int BLOCK, int MINB, class Body>
inline int launch_occ(const Body &body, size_t n, stream_t s) {
  if (n == 0) return OK;
  size_t grid = (n + BLOCK - 1) / BLOCK;
  run_kernel_occ<Body, BLOCK, MINB><<<(unsigned)grid, BLOCK, 0, s>>>(body, n);
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  return last_error();
}
template <int BLOCK, int MINB, class Body>
inline int resident_threads_occ(size_t *out) {
  static size_t cached = 0;
  if (!cached) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, run_kernel_occ<Body, BLOCK, MINB>, BLOCK, 0);
    if (e != cudaSuccess) return map_cuda(e);
    cached = (size_t)sms * (per_sm > 0 ? per_sm : 1) * BLOCK;
  }
  *out = cached;
  return OK;
}
#define PCGPU_BLOCK_FOR(i, n) for (uint32_t i = threadIdx.x; i < (uint32_t)(n); i += blockDim.x)
#define PCGPU_BLOCK_SYNC() __syncthreads()
#define PCGPU_WARP_ANY(x) __any_sync(0xffffffffu, (x))
template <class Body, int BLOCK>
__global__ void __launch_bounds__(BLOCK) run_block_kernel(const Body body) {
  extern __shared__ uint4 pcgpu_smem[];
  body((size_t)blockIdx.x, reinterpret_cast<uint32_t *>(pcgpu_smem));
}
template <int BLOCK, class Body>
inline int launch_blocks(const Body &body, size_t nblocks, size_t smem_bytes, stream_t s) {
  if (nblocks == 0) return OK;
  if (smem_bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(run_block_kernel<Body, BLOCK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e != cudaSuccess) return map_cuda(e);
  }
  run_block_kernel<Body, BLOCK><<<(unsigned)nblocks, BLOCK, smem_bytes, s>>>(body);
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  return last_error();
}
// same, with a minimum number of resident blocks per SM (caps the registers of register-heavy block-cooperative bodies)
template <class Body, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) run_block_kernel_occ(const Body body) {
  extern __shared__ uint4 pcgpu_smem[];
  body((size_t)blockIdx.x, reinterpret_cast<uint32_t *>(pcgpu_smem));
}
template <int BLOCK, int MINB, class Body>
inline int launch_blocks_occ(const Body &body, size_t nblocks, size_t smem_bytes, stream_t s) {
  if (nblocks == 0) return OK;
  if (smem_bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(run_block_kernel_occ<Body, BLOCK, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e != cudaSuccess) return map_cuda(e);
  }
  run_block_kernel_occ<Body, BLOCK, MINB><<<(unsigned)nblocks, BLOCK, smem_bytes, s>>>(body);
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  return last_error();
}
// Persistent kernels: one resident wave of threads (SM count x occupancy), each warp repeatedly claims 32
// consecutive tasks from a global counter -- no wave quantisation, no tail of half-empty blocks.
__device__ __forceinline__ uint32_t next_task(uint32_t *counter) {
  uint32_t lane = threadIdx.x & 31, base = 0;
  if (lane == 0) base = atomicAdd(counter, 32u);
  base = __shfl_sync(0xffffffffu, base, 0);
  return base + lane;
}
template <class Body, int BLOCK>
__global__ void __launch_bounds__(BLOCK) run_persistent_kernel(const Body body) {
  body((size_t)blockIdx.x * BLOCK + threadIdx.x);
}
template <int BLOCK, class Body>
inline int launch_persistent(const Body &body, stream_t s) {
  static int grid = 0;  // per kernel instantiation
  if (grid == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, run_persistent_kernel<Body, BLOCK>, BLOCK, 0);
    if (e != cudaSuccess) return map_cuda(e);
    grid = sms * (per_sm > 0 ? per_sm : 1);
  }
  run_persistent_kernel<Body, BLOCK><<<grid, BLOCK, 0, s>>>(body);
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  return last_error();
}
template <class T> __device__ __forceinline__ T atomic_add(T *p, T v) { return atomicAdd(p, v); }
template <class T> __device__ __forceinline__ T atomic_or(T *p, T v) { return atomicOr(p, v); }
#define PCGPU_KERNEL_DEV __device__ __forceinline__
#endif

// One device arena, re-used across calls and grown on demand, laid out afresh by every carve().
struct Arena {
  char *base = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return OK;
    if (base) dev_free(base);
    base = nullptr; cap = 0;
    int rc = dev_malloc((void **)&base, bytes);
    if (rc) return rc;
    cap = bytes;
    return OK;
  }
  // Lays the arena out as the buffers `list` names.  list(buf) calls buf(p, count) once per buffer, in layout order, with p a
  // T *& and count its elements; it runs twice, once to reserve the sum and once to point every p at its buffer.  Each buffer
  // takes whole 256-byte granules, at least one, so a zero-length buffer still gets a valid, distinct pointer.
  template <class List> int carve(const List &list) {
    size_t used = 0;
    list([&](auto *&p, size_t count) { used += padded(sizeof *p, count); });
    int rc = reserve(used);
    if (rc) return rc;
    used = 0;
    list([&](auto *&p, size_t count) {
      p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + used);
      used += padded(sizeof *p, count);
    });
    return OK;
  }
  static size_t padded(size_t elem, size_t count) { size_t b = elem * count; return ((b ? b : 1) + 255) & ~(size_t)255; }
  void release() { if (base) dev_free(base); base = nullptr; cap = 0; }
};

}  // namespace rt
}  // namespace pcgpu
