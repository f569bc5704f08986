// Micro-benchmark: issue rates of integer-pipe forms a multiplier-free curve25519 fold would use
// (IADD3, LEA / LEA.HI.X, SHF.L.W), and whether funnel shifts overlap IMAD.WIDE (companion of
// pipes.cu). ptxas may move plain adds and moves onto the multiplier pipe (IMAD.IADD, IMAD.MOV):
// check the SASS of a form before reading its rate as the integer pipe's.
//   nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a alu_pipes.cu -o alu_pipes
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
  u32 x[8] = {m, m ^ 1u, m ^ 2u, m ^ 3u, m ^ 4u, m ^ 5u, m ^ 6u, m ^ 7u};
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) {  // IMAD.WIDE.U32: 64-bit acc += 32x32
      a0 += (u64)(u32)a1 * m; a1 += (u64)(u32)a2 * m; a2 += (u64)(u32)a3 * m; a3 += (u64)(u32)a4 * m;
      a4 += (u64)(u32)a5 * m; a5 += (u64)(u32)a6 * m; a6 += (u64)(u32)a7 * m; a7 += (u64)(u32)a0 * m;
    }
    if (OP == 7) {  // 3-input 32-bit add (IADD3)
      u32 x0 = (u32)a0, x1 = (u32)a1, x2 = (u32)a2, x3 = (u32)a3, x4 = (u32)a4, x5 = (u32)a5, x6 = (u32)a6, x7 = (u32)a7;
      x0 += x1 + m; x1 += x2 + m; x2 += x3 + m; x3 += x4 + m; x4 += x5 + m; x5 += x6 + m; x6 += x7 + m; x7 += x0 + m;
      a0 = x0; a1 = x1; a2 = x2; a3 = x3; a4 = x4; a5 = x5; a6 = x6; a7 = x7;
    }
    if (OP == 8) {  // 64-bit a += b << 3 (LEA + LEA.HI.X): 8 64-bit ops = 16 instructions
      a0 += a1 << 3; a1 += a2 << 3; a2 += a3 << 3; a3 += a4 << 3; a4 += a5 << 3; a5 += a6 << 3; a6 += a7 << 3; a7 += a0 << 3;
    }
    if (OP == 9) {  // funnel shift (SHF.L.W)
      u32 x0 = (u32)a0, x1 = (u32)a1, x2 = (u32)a2, x3 = (u32)a3, x4 = (u32)a4, x5 = (u32)a5, x6 = (u32)a6, x7 = (u32)a7;
      x0 = __funnelshift_l(x1, x0, 5); x1 = __funnelshift_l(x2, x1, 5); x2 = __funnelshift_l(x3, x2, 5); x3 = __funnelshift_l(x4, x3, 5);
      x4 = __funnelshift_l(x5, x4, 5); x5 = __funnelshift_l(x6, x5, 5); x6 = __funnelshift_l(x7, x6, 5); x7 = __funnelshift_l(x0, x7, 5);
      a0 = x0; a1 = x1; a2 = x2; a3 = x3; a4 = x4; a5 = x5; a6 = x6; a7 = x7;
    }
    if (OP == 10) {  // mixed: 8 IMAD.WIDE + 8 SHF.L.W per iteration. A funnel shift of two registers has no
                     // multiplier-pipe form, so the shifts stay on the integer pipe; the rate printed is
                     // that of the IMAD.WIDEs (equal to the IMAD.WIDE-only rate = the shifts hide)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        u64& p = j == 0 ? a0 : j == 1 ? a1 : j == 2 ? a2 : j == 3 ? a3 : j == 4 ? a4 : j == 5 ? a5 : j == 6 ? a6 : a7;
        u64& q = j == 0 ? a1 : j == 1 ? a2 : j == 2 ? a3 : j == 3 ? a4 : j == 4 ? a5 : j == 5 ? a6 : j == 6 ? a7 : a0;
        p += (u64)(u32)q * m;
        x[j] = __funnelshift_l(x[(j + 1) & 7], x[j], 5);
      }
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 + (x[0] ^ x[1] ^ x[2] ^ x[3] ^ x[4] ^ x[5] ^ x[6] ^ x[7]);
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
  run<7>("IADD3 (32-bit, 3 inputs)", d, 8);
  run<8>("LEA + LEA.HI.X (64 += 64 << 3)", d, 16);
  run<9>("SHF.L.W (funnel shift)", d, 8);
  run<10>("IMAD.WIDE with 8 SHF.L.W alongside", d, 8);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
}
