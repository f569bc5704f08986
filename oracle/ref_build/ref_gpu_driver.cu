// TEST / MEASUREMENT INFRASTRUCTURE — never linked into the product.
//
// Stand-in for the reference's GPU backend on the C2 path: its own bucket-method kernels
// (sxt/multiexp/bucket_method/accumulation_kernel.h:38, combination_kernel.h:40,81), compiled
// unmodified for sm_90a from the reference checkout, launched with the geometry of
// accumulation.h:54-95 and multiexponentiation.h:55-86 (one output, one device, whole range), then
// the host combine_buckets of combination.h:50-62. It covers the reference's KERNELS and copies
// only — not its coroutine scheduler, chunking or multi-device split, which nvcc cannot build
// (SURVEY §8c). Recipe: SURVEY.md Appendix B.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <vector>

#include "sxt/base/container/span.h"
#include "sxt/curve21/operation/add.h"
#include "sxt/curve21/operation/double.h"
#include "sxt/curve21/operation/neg.h"
#include "sxt/curve21/type/element_p3.h"
#include "sxt/multiexp/bucket_method/accumulation_kernel.h"
#include "sxt/multiexp/bucket_method/combination.h"
#include "sxt/multiexp/bucket_method/combination_kernel.h"

using namespace sxt;
using E = c21t::element_p3;

#define CK(x)                                                                                      \
  do {                                                                                             \
    cudaError_t e_ = (x);                                                                          \
    if (e_ != cudaSuccess) {                                                                       \
      std::fprintf(stderr, "ref_gpu: %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);  \
      return 1;                                                                                    \
    }                                                                                              \
  } while (0)

// 0 when the kernels have an image for the current device: a library built for another architecture
// loads, but its launches fail.
extern "C" int ref_gpu_probe() {
  cudaFuncAttributes a;
  return (int)cudaFuncGetAttributes(&a, mtxbk::bucket_accumulate<E>);
}

// generators: n x 160 B (host), scalars: n x 32 B (host), out: one element_p3 (160 B).
// times_ms[0] = whole call (H2D + kernels + D2H + host combine, wall clock of the GPU part by events),
// times_ms[1] = the three kernels only.
extern "C" int ref_gpu_bucket_msm(void* out, const void* generators, const uint8_t* scalars,
                                  unsigned n, float* times_ms) {
  constexpr unsigned kGroups = 32, kGroupSize = 255;
  const unsigned num_blocks = n < 192u ? n : 192u;
  E *d_gens, *d_partial, *d_sums, *d_reduced;
  uint8_t* d_scalars;
  cudaEvent_t e0, e1, e2, e3;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  CK(cudaEventCreate(&e2));
  CK(cudaEventCreate(&e3));
  CK(cudaMalloc(&d_gens, sizeof(E) * n));
  CK(cudaMalloc(&d_scalars, 32ull * n));
  CK(cudaMalloc(&d_partial, sizeof(E) * kGroupSize * kGroups * num_blocks));
  CK(cudaMalloc(&d_sums, sizeof(E) * kGroupSize * kGroups));
  CK(cudaMalloc(&d_reduced, sizeof(E) * kGroupSize));
  std::vector<E> reduced(kGroupSize);
  CK(cudaEventRecord(e0));
  CK(cudaMemcpyAsync(d_gens, generators, sizeof(E) * n, cudaMemcpyHostToDevice));
  CK(cudaMemcpyAsync(d_scalars, scalars, 32ull * n, cudaMemcpyHostToDevice));
  CK(cudaEventRecord(e1));
  mtxbk::bucket_accumulate<E><<<dim3(num_blocks, 1, 1), kGroups>>>(d_partial, d_gens, d_scalars, n);
  mtxbk::combine_partial_bucket_sums<E>
      <<<dim3(kGroupSize, 1, 1), kGroups>>>(d_sums, d_partial, num_blocks);
  mtxbk::combine_bucket_groups<kGroupSize, kGroups, E>
      <<<dim3((kGroupSize + 31) / 32, 1, 1), 32>>>(d_reduced, d_sums);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e2));
  CK(cudaMemcpyAsync(reduced.data(), d_reduced, sizeof(E) * kGroupSize, cudaMemcpyDeviceToHost));
  CK(cudaEventRecord(e3));
  CK(cudaDeviceSynchronize());
  E res;
  mtxbk::combine_buckets<E>(basct::span<E>{&res, 1}, basct::span<E>{reduced.data(), kGroupSize});
  *static_cast<E*>(out) = res;
  CK(cudaEventElapsedTime(&times_ms[0], e0, e3));
  CK(cudaEventElapsedTime(&times_ms[1], e1, e2));
  cudaFree(d_gens);
  cudaFree(d_scalars);
  cudaFree(d_partial);
  cudaFree(d_sums);
  cudaFree(d_reduced);
  return 0;
}
