// Micro-benchmark (GPU box only): single-warp latency (cycles per operation in a dependent chain)
// and full-chip throughput of the field / point primitives. Build:
//   nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr latency.cu -o latency
#include <cstdio>
#include <cuda_runtime.h>
#include "../../blitzar_b200/csrc/curve.cuh"
#include "rejected_experiments.cuh"
using namespace b200;

template <int OP> __global__ void k_lat(Fe<8>* io, long long* cycles, int iters) {
  typedef F25519 F;
  Fe<8> a = io[threadIdx.x & 3], b = io[4 + (threadIdx.x & 3)];
  Ed25519::Point P;
  P.X = a; P.Y = b; P.Z = io[1]; P.T = io[2];
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) F::mul(a, a, b);
    if (OP == 1) F::mul_lat(a, a, b);
    if (OP == 2) F::mul_ref(a, a, b);
    if (OP == 3) F::add(a, a, b);
    if (OP == 4) F::sub(a, a, b);
    if (OP == 5) Ed25519::dbl<SeqExec>(P, P);
    if (OP == 6) Ed25519::dbl<QuadExec>(P, P);
    if (OP == 7) Ed25519::add<SeqExec>(P, P, P);
    if (OP == 8) Ed25519::add<QuadExec>(P, P, P);
    if (OP == 9) Ed25519::dbl<QuadExecConv>(P, P);
    if (OP == 10) Ed25519::add<QuadExecConv>(P, P, P);
  }
  long long t1 = clock64();
  if (threadIdx.x == 0 && blockIdx.x == 0) cycles[0] = t1 - t0;
  io[8 + (threadIdx.x & 3)] = (OP >= 5) ? P.X : a;
}
template <int OP> __global__ void k_thr(Fe<8>* io, int iters) {
  typedef F25519 F;
  Fe<8> a = io[threadIdx.x & 3], b = io[4 + (threadIdx.x & 3)];
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) F::mul(a, a, b);
    if (OP == 1) F::mul_lat(a, a, b);
    if (OP == 2) F::mul_ref(a, a, b);
    if (OP == 3) rejected::mul_kara(a, a, b);
  }
  if (a.l[0] == 0x12345678u) io[8] = a;
}
__global__ void k_thr_fp64(Fe<8>* io, int iters) {
  Fe<8> a8, b8;
  F25519::canonical(a8, io[threadIdx.x & 3]);
  F25519::canonical(b8, io[4 + (threadIdx.x & 3)]);
  FeD a, b;
  F25519D::from_fe(a, a8);
  F25519D::from_fe(b, b8);
  long long ta[5], tb[5];
  for (int i = 0; i < 5; ++i) { ta[i] = a.l[i]; tb[i] = b.l[i]; }
  F25519D::carry(a, ta);
  F25519D::carry(b, tb);
  double db[5];
  for (int i = 0; i < 5; ++i) db[i] = F25519D::to_double(b.l[i]);
  for (int it = 0; it < iters; ++it) {
    double da[5];
    for (int i = 0; i < 5; ++i) da[i] = F25519D::to_double(a.l[i]);
    F25519D::mul(a, da, db);
  }
  if (a.l[0] == 0x12345678) io[8].l[0] = (u32)a.l[1];
}
__global__ void k_thr_accd(Fe<8>* io, int iters) {
  Ed25519::Gen g;
  F25519::canonical(g.YpX, io[0]); F25519::canonical(g.YmX, io[1]); F25519::canonical(g.Z2, io[2]); F25519::canonical(g.T2d, io[3]);
  rejected::AccD acc;
  rejected::accd_from_gen(acc, g, false);
  for (int it = 0; it < iters; ++it) rejected::accd_add_gen(acc, g, (it & 1) != 0);
  if (acc.X.l[0] == 0x12345678) io[8].l[0] = (u32)acc.Y.l[1];
}
__global__ void k_thr_addgen(Fe<8>* io, int iters) {
  Ed25519::Gen g;
  g.YpX = io[0]; g.YmX = io[1]; g.Z2 = io[2]; g.T2d = io[3];
  Ed25519::Point acc;
  Ed25519::gen_to_point(acc, g, false);
  for (int it = 0; it < iters; ++it) Ed25519::add_gen<SeqExec>(acc, acc, g, (it & 1) != 0);
  if (acc.X.l[0] == 0x12345678) io[8] = acc.Y;
}
static int g_sms = 0;
static double g_hz = 0;  // the device's maximum SM clock
template <class K> void thr_k(const char* name, K kern, Fe<8>* d, int threads, int blocks_per_sm) {
  const int iters = 1000, blocks = g_sms * blocks_per_sm;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  kern<<<blocks, threads>>>(d, iters);
  cudaEventRecord(e0);
  kern<<<blocks, threads>>>(d, iters);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double ops = (double)blocks * threads * iters;
  printf("throughput %-30s %d thr x %d blk/SM: %.2f G op/s (%.1f SM-cycles per warp-op)\n", name, threads, blocks_per_sm,
         ops / ms * 1e-6, g_hz * g_sms / (ops / 32 / (ms * 1e-3)));
}
template <int OP> void lat(const char* name, Fe<8>* d, long long* dc, int threads) {
  const int iters = 200;
  k_lat<OP><<<1, threads>>>(d, dc, iters);
  k_lat<OP><<<1, threads>>>(d, dc, iters);
  long long c; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
  printf("latency  %-28s %4d thr: %8.1f cycles/op\n", name, threads, (double)c / iters);
}
template <int OP> void thr(const char* name, Fe<8>* d) {
  const int iters = 2000, blocks = g_sms * 8, threads = 256;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  k_thr<OP><<<blocks, threads>>>(d, iters);
  cudaEventRecord(e0);
  k_thr<OP><<<blocks, threads>>>(d, iters);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double muls = (double)blocks * threads * iters;
  printf("throughput %-26s: %.2f G mul/s (%.1f SM-cycles per warp-mul)\n", name, muls / ms * 1e-6,
         g_hz * g_sms / (muls / 32 / (ms * 1e-3)));
}
int main() {
  int khz = 0;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  g_hz = khz * 1e3;
  Fe<8>* d; long long* dc;
  cudaMalloc(&d, 64 * sizeof(Fe<8>)); cudaMalloc(&dc, 8);
  Fe<8> h[16];
  for (int i = 0; i < 16; ++i) for (int k = 0; k < 8; ++k) h[i].l[k] = 0x9e3779b9u * (i * 8 + k + 1);
  cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
  lat<0>("F25519::mul (chains)", d, dc, 32);
  lat<1>("F25519::mul_lat (columns)", d, dc, 32);
  lat<2>("F25519::mul_ref (plain C)", d, dc, 32);
  lat<3>("F25519::add", d, dc, 32);
  lat<4>("F25519::sub", d, dc, 32);
  lat<5>("Ed25519::dbl seq", d, dc, 32);
  lat<6>("Ed25519::dbl quad", d, dc, 32);
  lat<7>("Ed25519::add seq", d, dc, 32);
  lat<8>("Ed25519::add quad", d, dc, 32);
  lat<9>("Ed25519::dbl quad fullmask", d, dc, 32);
  lat<10>("Ed25519::add quad fullmask", d, dc, 32);
  thr<0>("F25519::mul (chains)", d);
  thr<1>("F25519::mul_lat (columns)", d);
  thr<2>("F25519::mul_ref (plain C)", d);
  thr<3>("F25519::mul_kara (Karatsuba)", d);
  thr_k("F25519D::mul (fp64 pipe)", k_thr_fp64, d, 256, 8);
  thr_k("F25519D::mul (fp64 pipe)", k_thr_fp64, d, 128, 3);
  thr_k("accd_add_gen (fp64 point add)", k_thr_accd, d, 128, 3);
  thr_k("accd_add_gen (fp64 point add)", k_thr_accd, d, 128, 6);
  thr_k("add_gen (integer point add)", k_thr_addgen, d, 128, 3);
  thr_k("add_gen (integer point add)", k_thr_addgen, d, 128, 6);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
