// Micro-benchmark: issue rates of the pipes the field multiplier can use (per SM per clock).
//   nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a pipes.cu -o pipes
// Rates are per SM per clock at the SM clock sampled by nvidia-smi during the run (argv[1], MHz;
// default: the device's maximum clock).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
typedef unsigned long long u64;
typedef unsigned int u32;
template <int OP> __global__ void k(u64* out, int iters) {
  u64 a0 = threadIdx.x + 1, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, a4 = a0 * 11, a5 = a0 * 13, a6 = a0 * 17, a7 = a0 * 19;
  u32 m = (u32)(threadIdx.x * 2654435761u) | 1u;
  double d0 = a0, d1 = a1, d2 = a2, d3 = a3, d4 = a4, d5 = a5, d6 = a6, d7 = a7, dm = 1.0000001;
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) {  // IMAD.WIDE.U32: 64-bit acc += 32x32
      a0 += (u64)(u32)a1 * m; a1 += (u64)(u32)a2 * m; a2 += (u64)(u32)a3 * m; a3 += (u64)(u32)a4 * m;
      a4 += (u64)(u32)a5 * m; a5 += (u64)(u32)a6 * m; a6 += (u64)(u32)a7 * m; a7 += (u64)(u32)a0 * m;
    }
    if (OP == 1) {  // DFMA (round toward zero)
      d0 = __fma_rz(d0, dm, d1); d1 = __fma_rz(d1, dm, d2); d2 = __fma_rz(d2, dm, d3); d3 = __fma_rz(d3, dm, d4);
      d4 = __fma_rz(d4, dm, d5); d5 = __fma_rz(d5, dm, d6); d6 = __fma_rz(d6, dm, d7); d7 = __fma_rz(d7, dm, d0);
    }
    if (OP == 2) {  // 32-bit IMAD
      u32 x0 = (u32)a0, x1 = (u32)a1, x2 = (u32)a2, x3 = (u32)a3, x4 = (u32)a4, x5 = (u32)a5, x6 = (u32)a6, x7 = (u32)a7;
      x0 = x0 * m + x1; x1 = x1 * m + x2; x2 = x2 * m + x3; x3 = x3 * m + x4; x4 = x4 * m + x5; x5 = x5 * m + x6; x6 = x6 * m + x7; x7 = x7 * m + x0;
      a0 = x0; a1 = x1; a2 = x2; a3 = x3; a4 = x4; a5 = x5; a6 = x6; a7 = x7;
    }
    if (OP == 3) {  // 64-bit integer add (IADD3 + IADD3.X)
      a0 += a1; a1 += a2; a2 += a3; a3 += a4; a4 += a5; a5 += a6; a6 += a7; a7 += a0;
    }
    if (OP == 5) {  // IMAD.HI.U32
      u32 x0 = (u32)a0, x1 = (u32)a1, x2 = (u32)a2, x3 = (u32)a3, x4 = (u32)a4, x5 = (u32)a5, x6 = (u32)a6, x7 = (u32)a7;
      x0 = __umulhi(x0, m) + x1; x1 = __umulhi(x1, m) + x2; x2 = __umulhi(x2, m) + x3; x3 = __umulhi(x3, m) + x4;
      x4 = __umulhi(x4, m) + x5; x5 = __umulhi(x5, m) + x6; x6 = __umulhi(x6, m) + x7; x7 = __umulhi(x7, m) + x0;
      a0 = x0; a1 = x1; a2 = x2; a3 = x3; a4 = x4; a5 = x5; a6 = x6; a7 = x7;
    }
    if (OP == 6) {  // one 32x32 product accumulated into a 64-bit value WITHOUT IMAD.WIDE:
                    // mul.lo + mul.hi on the multiplier pipe, add.cc + addc on the ALU pipe
      u32 l[8] = {(u32)a0, (u32)a1, (u32)a2, (u32)a3, (u32)a4, (u32)a5, (u32)a6, (u32)a7};
      u32 h[8] = {(u32)(a0 >> 32), (u32)(a1 >> 32), (u32)(a2 >> 32), (u32)(a3 >> 32), (u32)(a4 >> 32), (u32)(a5 >> 32), (u32)(a6 >> 32), (u32)(a7 >> 32)};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        u32 x = l[(j + 1) & 7], pl, ph;
        asm volatile("mul.lo.u32 %0, %2, %3;\n\tmul.hi.u32 %1, %2, %3;" : "=r"(pl), "=r"(ph) : "r"(x), "r"(m));
        asm volatile("add.cc.u32 %0, %0, %2;\n\taddc.u32 %1, %1, %3;" : "+r"(l[j]), "+r"(h[j]) : "r"(pl), "r"(ph));
      }
      a0 = l[0] | ((u64)h[0] << 32); a1 = l[1] | ((u64)h[1] << 32); a2 = l[2] | ((u64)h[2] << 32); a3 = l[3] | ((u64)h[3] << 32);
      a4 = l[4] | ((u64)h[4] << 32); a5 = l[5] | ((u64)h[5] << 32); a6 = l[6] | ((u64)h[6] << 32); a7 = l[7] | ((u64)h[7] << 32);
    }
    if (OP == 4) {  // mixed: 8 DFMA + 8 IMAD.WIDE per iteration (do they overlap?)
      d0 = __fma_rz(d0, dm, d1); a0 += (u64)(u32)a1 * m; d1 = __fma_rz(d1, dm, d2); a1 += (u64)(u32)a2 * m;
      d2 = __fma_rz(d2, dm, d3); a2 += (u64)(u32)a3 * m; d3 = __fma_rz(d3, dm, d4); a3 += (u64)(u32)a4 * m;
      d4 = __fma_rz(d4, dm, d5); a4 += (u64)(u32)a5 * m; d5 = __fma_rz(d5, dm, d6); a5 += (u64)(u32)a6 * m;
      d6 = __fma_rz(d6, dm, d7); a6 += (u64)(u32)a7 * m; d7 = __fma_rz(d7, dm, d0); a7 += (u64)(u32)a0 * m;
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 + (u64)(d0 + d1 + d2 + d3 + d4 + d5 + d6 + d7);
}
static int g_sms = 0;
static double g_hz = 0;
template <int OP> void run(const char* name, u64* d, double ops_per_iter) {
  const int iters = 4000, blocks = g_sms * 8, threads = 256;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  k<OP><<<blocks, threads>>>(d, iters);
  cudaEventRecord(e0);
  k<OP><<<blocks, threads>>>(d, iters);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double ops = (double)blocks * threads * iters * ops_per_iter;
  printf("%-34s %8.1f Gop/s  = %5.1f lane-ops/clk/SM at %.3f GHz\n", name, ops / ms * 1e-6,
         ops / (ms * 1e-3) / g_sms / g_hz, g_hz * 1e-9);
}
int main(int argc, char** argv) {
  int khz = 0;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  g_hz = argc > 1 ? std::atof(argv[1]) * 1e6 : khz * 1e3;
  printf("%d SMs\n", g_sms);
  u64* d; cudaMalloc(&d, (size_t)g_sms * 8 * 256 * 8);
  run<0>("IMAD.WIDE.U32 (64 += 32x32)", d, 8);
  run<1>("DFMA.RZ", d, 8);
  run<2>("IMAD (32-bit)", d, 8);
  run<3>("64-bit integer add", d, 8);
  run<4>("8 DFMA + 8 IMAD.WIDE interleaved", d, 16);
  run<5>("IMAD.HI.U32", d, 8);
  run<6>("product via mul.lo+mul.hi+add.cc+addc", d, 8);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
}
