// Minimal launch / memory layer under the MSM engine.
//
// Replaces sxt/execution (coroutine futures + event-polling scheduler), sxt/memory (pmr device
// resources) and sxt/algorithm/iteration/for_each.h for this path with plain CUDA streams and the
// stream-ordered allocator: every kernel of the engine is an index-parallel body launched on one
// stream; there is no host-side scheduling.
//
// With -DB200_EMULATE (tests/emul only) the same bodies run as serial host loops so the whole
// pipeline can be exercised on a machine without a GPU. The product library is never built that
// way and has no CPU fallback.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <cctype>
#include <string>
#include <utility>
#include <vector>

#include "field.cuh"

#ifndef B200_EMULATE
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#endif

namespace b200 {

[[noreturn]] inline void die(const char* what, const char* file, int line) {
  std::fprintf(stderr, "blitzar_b200: fatal: %s (%s:%d)\n", what, file, line);
  std::abort();
}
#define B200_REQUIRE(cond, msg)                                                                    \
  do {                                                                                             \
    if (!(cond))                                                                                   \
      ::b200::die(msg, __FILE__, __LINE__);                                                        \
  } while (0)

// stderr log gated by BLITZAR_LOG_LEVEL (the reference's variable, sxt/base/log/setup.cc:28-55):
// unset / error / critical / off -> silent; warn; info (one line per entry point: shapes, window
// width, pieces, path taken); debug / trace (per stage).
inline int log_level() {
  static const int level = [] {
    const char* env = std::getenv("BLITZAR_LOG_LEVEL");
    if (!env)
      return 0;
    std::string s(env);
    for (auto& ch : s)
      ch = (char)std::tolower((unsigned char)ch);
    if (s == "warn")
      return 1;
    if (s == "info")
      return 2;
    if (s == "debug" || s == "trace")
      return 3;
    return 0;
  }();
  return level;
}
#define B200_LOG(level, ...)                                                                       \
  do {                                                                                             \
    if (::b200::log_level() >= (level)) {                                                          \
      std::fprintf(stderr, "[blitzar_b200] " __VA_ARGS__);                                         \
      std::fputc('\n', stderr);                                                                    \
    }                                                                                              \
  } while (0)

// NVTX range around a stage of the pipeline (visible in nsys / ncu --nvtx; free when no tool is
// attached). The reference brackets its benchmark loop with cudaProfilerStart/Stop only
// (benchmark/multi_commitment/benchmark.m.cc:205,221).
struct StageRange {
#ifndef B200_EMULATE
  explicit StageRange(const char* name) { nvtxRangePushA(name); }
  ~StageRange() { nvtxRangePop(); }
#else
  explicit StageRange(const char*) {}
#endif
  StageRange(const StageRange&) = delete;
  StageRange& operator=(const StageRange&) = delete;
};

#ifndef B200_EMULATE
#define B200_CUDA(call)                                                                            \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      ::b200::die(cudaGetErrorString(e_), __FILE__, __LINE__);                                     \
  } while (0)

typedef cudaStream_t stream_t;

// bodies may request a minimum number of resident blocks per SM (register cap) with kMinBlocks
template <class Body, class = void> struct MinBlocks {
  static constexpr int value = 1;
};
template <class Body> struct MinBlocks<Body, decltype((void)Body::kMinBlocks)> {
  static constexpr int value = Body::kMinBlocks;
};
template <class Body>
__global__ void __launch_bounds__(Body::kBlock, MinBlocks<Body>::value) k_run(Body body, u64 n) {
  u64 tid = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < n)
    body(tid);
}

struct LaunchCounter {
  static std::atomic<unsigned long long>& value() {
    static std::atomic<unsigned long long> v{0};
    return v;
  }
};

template <class Body> inline void launch(const Body& body, u64 n, stream_t s) {
  if (n == 0)
    return;
  u64 blocks = (n + Body::kBlock - 1) / Body::kBlock;
  B200_REQUIRE(blocks < (1ull << 31), "grid too large");
  k_run<Body><<<(unsigned)blocks, Body::kBlock, 0, s>>>(body, n);
  B200_CUDA(cudaGetLastError());
  ++LaunchCounter::value();
}
// Block-cooperative kernels: every thread of block b runs body.run(b, smem), with `smem_bytes` of
// dynamic shared memory. Above the 48 KB default the kernel's limit is raised first (per device: the
// attribute belongs to the calling thread's current device).
template <class Body> __global__ void __launch_bounds__(Body::kBlock) k_block(Body body) {
  extern __shared__ __align__(16) unsigned char smem[];
  body.run(blockIdx.x, smem);
}
template <class Body>
inline void launch_blocks(const Body& body, u64 blocks, size_t smem_bytes, stream_t s) {
  if (blocks == 0)
    return;
  B200_REQUIRE(blocks < (1ull << 31), "grid too large");
  static thread_local size_t raised = 48 * 1024;
  if (smem_bytes > raised) {
    B200_CUDA(cudaFuncSetAttribute(k_block<Body>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem_bytes));
    raised = smem_bytes;
  }
  k_block<Body><<<(unsigned)blocks, Body::kBlock, smem_bytes, s>>>(body);
  B200_CUDA(cudaGetLastError());
  ++LaunchCounter::value();
}
inline void* dev_alloc(size_t bytes, stream_t s) {
  void* p = nullptr;
  B200_CUDA(cudaMallocAsync(&p, bytes ? bytes : 16, s));
  return p;
}
inline void dev_free(void* p, stream_t s) {
  if (p)
    B200_CUDA(cudaFreeAsync(p, s));
}
inline void dev_zero(void* p, size_t bytes, stream_t s) { B200_CUDA(cudaMemsetAsync(p, 0, bytes, s)); }
inline void copy_h2d(void* d, const void* h, size_t bytes, stream_t s) {
  if (bytes)
    B200_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
}
inline void copy_d2h(void* h, const void* d, size_t bytes, stream_t s) {
  if (bytes)
    B200_CUDA(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s));
}
inline void copy_d2d(void* d, const void* s_, size_t bytes, stream_t s) {
  if (bytes)
    B200_CUDA(cudaMemcpyAsync(d, s_, bytes, cudaMemcpyDeviceToDevice, s));
}
inline void stream_sync(stream_t s) { B200_CUDA(cudaStreamSynchronize(s)); }
// everything enqueued on `later` from here on waits for what is on `earlier` now
inline void stream_follow(stream_t later, stream_t earlier) {
  static thread_local cudaEvent_t ring[64];
  static thread_local unsigned next = 0;
  cudaEvent_t& e = ring[next++ % 64];
  if (!e)
    B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  B200_CUDA(cudaEventRecord(e, earlier));
  B200_CUDA(cudaStreamWaitEvent(later, e, 0));
}

// a second stream of the calling thread (= of its device), for stages whose halves can overlap
inline stream_t aux_stream() {
  static thread_local cudaStream_t s = nullptr;
  if (!s)
    B200_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  return s;
}

// Small host->device parameter blocks (column descriptors, prefix tables). A pageable
// cudaMemcpyAsync synchronises the stream, which would stall the launch queue once per range; the
// blocks therefore go through a ring of pinned slots and are copied truly asynchronously. A slot is
// reused only after the copy that last read it has completed (per-slot event).
struct StagingRing {
  static constexpr size_t kSlotBytes = 65536, kSlots = 128;  // 64 KiB = ~1600 column descriptors
  unsigned char* base = nullptr;
  cudaEvent_t done[kSlots];
  size_t next = 0;
  static StagingRing& get() {
    static thread_local StagingRing r;  // one ring per host thread (= per device in multi-GPU mode)
    return r;
  }
  void* stage(stream_t s, const void* host, size_t bytes) {
    void* d = dev_alloc(bytes, s);
    if (bytes > kSlotBytes) {  // rare (thousands of columns): fall back to a synchronising copy
      copy_h2d(d, host, bytes, s);
      stream_sync(s);
      return d;
    }
    if (!base) {
      B200_CUDA(cudaHostAlloc((void**)&base, kSlotBytes * kSlots, cudaHostAllocDefault));
      for (auto& e : done) {
        B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      }
    }
    size_t slot = next++ % kSlots;
    B200_CUDA(cudaEventSynchronize(done[slot]));
    std::memcpy(base + slot * kSlotBytes, host, bytes);
    B200_CUDA(cudaMemcpyAsync(d, base + slot * kSlotBytes, bytes, cudaMemcpyHostToDevice, s));
    B200_CUDA(cudaEventRecord(done[slot], s));
    return d;
  }
};
inline void* stage_to_device(stream_t s, const void* host, size_t bytes) {
  return StagingRing::get().stage(s, host, bytes);
}

// Optional per-launch timing of the dominant kernel (bucket accumulation, level 1) with CUDA events
// on the launching stream — used by bench.py for the roofline line; off by default.
struct KernelTimer {
  bool enabled = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> spans;
  static KernelTimer& get() {
    static thread_local KernelTimer t;  // timings belong to the thread (device) that launched
    return t;
  }
  void begin(stream_t s) {
    if (!enabled)
      return;
    cudaEvent_t a, b;
    B200_CUDA(cudaEventCreate(&a));
    B200_CUDA(cudaEventCreate(&b));
    B200_CUDA(cudaEventRecord(a, s));
    spans.emplace_back(a, b);
  }
  void end(stream_t s) {
    if (!enabled)
      return;
    B200_CUDA(cudaEventRecord(spans.back().second, s));
  }
  // total milliseconds and number of timed launches since the last read
  void read(float* total_ms, unsigned* count) {
    float tot = 0;
    for (auto& sp : spans) {
      float ms = 0;
      B200_CUDA(cudaEventSynchronize(sp.second));
      B200_CUDA(cudaEventElapsedTime(&ms, sp.first, sp.second));
      tot += ms;
      B200_CUDA(cudaEventDestroy(sp.first));
      B200_CUDA(cudaEventDestroy(sp.second));
    }
    *total_ms = tot;
    *count = (unsigned)spans.size();
    spans.clear();
  }
};
// the host half of a __host__ __device__ body is never executed in the product build
template <class T> B200_HD T atomic_add(T* p, T v) {
#ifdef __CUDA_ARCH__
  return atomicAdd(p, v);
#else
  T old = *p;
  *p = old + v;
  return old;
#endif
}
#define B200_ATOMIC_ADD(ptr, v) ::b200::atomic_add((ptr), (v))
#else
// ---- emulation: serial host loops ---------------------------------------------------------------
typedef int stream_t;
struct LaunchCounter {
  static unsigned long long& value() {
    static unsigned long long v = 0;
    return v;
  }
};
template <class Body> inline void launch(const Body& body, u64 n, stream_t) {
  for (u64 t = 0; t < n; ++t)
    body(t);
  ++LaunchCounter::value();
}
inline void* dev_alloc(size_t bytes, stream_t) { return std::malloc(bytes ? bytes : 16); }
inline void dev_free(void* p, stream_t) { std::free(p); }
inline void dev_zero(void* p, size_t bytes, stream_t) { std::memset(p, 0, bytes); }
inline void copy_h2d(void* d, const void* h, size_t bytes, stream_t) { std::memcpy(d, h, bytes); }
inline void copy_d2h(void* h, const void* d, size_t bytes, stream_t) { std::memcpy(h, d, bytes); }
inline void copy_d2d(void* d, const void* s_, size_t bytes, stream_t) { std::memcpy(d, s_, bytes); }
inline void stream_sync(stream_t) {}
inline void stream_follow(stream_t, stream_t) {}
inline stream_t aux_stream() { return 0; }
inline void* stage_to_device(stream_t s, const void* host, size_t bytes) {
  void* d = dev_alloc(bytes, s);
  std::memcpy(d, host, bytes);
  return d;
}
struct KernelTimer {
  static KernelTimer& get() {
    static KernelTimer t;
    return t;
  }
  void begin(stream_t) {}
  void end(stream_t) {}
};
template <class T> inline T emul_atomic_add(T* p, T v) {
  T old = *p;
  *p = old + v;
  return old;
}
#define B200_ATOMIC_ADD(ptr, v) ::b200::emul_atomic_add((ptr), (v))
#endif

}  // namespace b200
