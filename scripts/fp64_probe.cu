// Measures the sustained fp64 rates of this GPU: scalar DFMA and mma.sync.m8n8k4.f64 (DMMA).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/fp64_probe scripts/fp64_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void dfma_kernel(double* out, int iters, double a, double b) {
  double acc[8];
  for (int i = 0; i < 8; ++i) acc[i] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = fma(acc[i], a, b);
  }
  double s = 0;
  for (int i = 0; i < 8; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void ffma_kernel(float* out, int iters, float a, float b) {
  float acc[8];
  for (int i = 0; i < 8; ++i) acc[i] = threadIdx.x * 1e-3f + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = fmaf(acc[i], a, b);
  }
  float s = 0;
  for (int i = 0; i < 8; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void dmma_kernel(double* out, int iters, double a, double b) {
  double c[4][2];
  for (int i = 0; i < 4; ++i) c[i][0] = c[i][1] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double s = 0;
  for (int i = 0; i < 4; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  double* out; cudaMalloc(&out, 148 * 8 * 256 * 8);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 20000, grid = 148 * 8, block = 256;
  float ms;
  for (int rep = 0; rep < 2; ++rep) {
    cudaEventRecord(e0); dfma_kernel<<<grid, block>>>(out, iters, 0.999, 1e-3); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    double n = (double)grid * block * iters * 8;
    printf("DFMA: %.3f ms  %.2f T DFMA/s  = %.1f DFMA/clk/SM at 1.9 GHz\n", ms, n / ms / 1e9, n / (ms * 1e-3) / 148 / 1.9e9);
    cudaEventRecord(e0); ffma_kernel<<<grid, block>>>((float*)out, iters, 0.999f, 1e-3f); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    printf("FFMA: %.3f ms  %.2f T FFMA/s  = %.1f FFMA/clk/SM\n", ms, n / ms / 1e9, n / (ms * 1e-3) / 148 / 1.9e9);
    cudaEventRecord(e0); dmma_kernel<<<grid, block>>>(out, iters / 4, 0.999, 1e-3); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    double nm = (double)grid * (block / 32) * (iters / 4) * 4 * 256;   // 8x8x4 MACs per warp-level mma
    printf("DMMA: %.3f ms  %.2f T MAC/s  = %.1f MAC/clk/SM\n", ms, nm / ms / 1e9, nm / (ms * 1e-3) / 148 / 1.9e9);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
