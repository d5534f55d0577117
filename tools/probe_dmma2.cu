// DMMA latency / occupancy probe: throughput of fp64 mma chains vs warps per SM and chains per warp, for the
// shapes m8n8k4 (DMMA.8x8x4), m16n8k4 (DMMA.16x8x4) and m16n8k8 (DMMA.16x8x8).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe_dmma2.bin tools/probe_dmma2.cu
#include <cstdio>
#include <cuda_runtime.h>
enum Shape { k884 = 0, k1684 = 1, k1688 = 2 };
template <int S>
__device__ __forceinline__ void mma(double (&c)[4], double a, double b) {
  if constexpr (S == k884)
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
  else if constexpr (S == k1684)
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(a), "d"(b));
  else
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b));
}
template <int S, int CH>
__global__ void k(double* out, int iters) {
  double a = threadIdx.x * 1e-9, b = 1.0 + threadIdx.x * 1e-9, c[CH][4];
  for (int u = 0; u < CH; ++u) c[u][0] = c[u][1] = c[u][2] = c[u][3] = 0.0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int u = 0; u < CH; ++u) mma<S>(c[u], a, b);
  }
  double s = 0;
  for (int u = 0; u < CH; ++u) s += c[u][0] + c[u][1] + c[u][2] + c[u][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int S, int CH>
static void run(double* out, int sm, int wps) {
  const int iters = 4000;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    cudaEventRecord(e0); k<S, CH><<<sm, wps * 32>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    if (cudaGetLastError() != cudaSuccess) {  // too many registers for this many warps in one CTA
      printf("%-8s warps/SM %2d chains %d: not launchable (registers)\n",
             S == k884 ? "m8n8k4" : S == k1684 ? "m16n8k4" : "m16n8k8", wps, CH);
      cudaEventDestroy(e0); cudaEventDestroy(e1);
      return;
    }
    float ms; cudaEventElapsedTime(&ms, e0, e1); if (r && ms < best) best = ms;
  }
  const double n = (double)iters * 8 * CH * wps * sm;  // DMMA warp-instructions
  const double flop = S == k884 ? 512 : S == k1684 ? 1024 : 2048;  // 2 * m * n * k
  int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  printf("%-8s warps/SM %2d chains %d: %6.2f TFLOP/s   %.1f clk per DMMA per SMSP-warp-chain\n",
         S == k884 ? "m8n8k4" : S == k1684 ? "m16n8k4" : "m16n8k8", wps, CH, n * flop / (best * 1e-3) / 1e12,
         best * 1e-3 * clk * 1e3 / ((double)iters * 8));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
}
template <int S>
static void sweep(double* out, int sm) {
  for (int wps : {4, 8, 16, 24, 32}) { run<S, 1>(out, sm, wps); run<S, 2>(out, sm, wps); run<S, 4>(out, sm, wps); run<S, 8>(out, sm, wps); }
}
int main() {
  int sm = 0; cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
  double* out; cudaMalloc(&out, (size_t)sm * 1024 * 8);
  sweep<k884>(out, sm);
  sweep<k1684>(out, sm);
  sweep<k1688>(out, sm);
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  cudaFree(out);
}
