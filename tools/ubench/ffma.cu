// ffma.cu -- FP32 SIMT peak of the device as a kernel can reach it: 8 independent FFMA chains per thread, 1024 threads
// per SM x 4 resident blocks, no memory traffic: what the FP32 pipe of the GMM kernel's roofline_scoring can reach on this
// device, against the data-sheet figure bench.py divides by.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ffma ffma.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void __launch_bounds__(256) k(float *out, int iters, float a, float b) {
  float x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int u = 0; u < 16; u++) {
      x0 = fmaf(x0, a, b); x1 = fmaf(x1, a, b); x2 = fmaf(x2, a, b); x3 = fmaf(x3, a, b);
      x4 = fmaf(x4, a, b); x5 = fmaf(x5, a, b); x6 = fmaf(x6, a, b); x7 = fmaf(x7, a, b);
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
}

int main() {
  int sms = 0, khz = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0); cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const int blocks = sms * 8, iters = 4096;
  float *o; cudaMalloc(&o, sizeof(float) * blocks * 256);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  double best1 = 0;
  for (int rep = 0; rep < 5; rep++) {
    cudaEventRecord(e0); k<<<blocks, 256>>>(o, iters, 0.999f, 0.001f); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double tf = 2.0 * 8 * 16 * (double)iters * blocks * 256 / (ms * 1e-3) / 1e12; if (tf > best1) best1 = tf;
  }
  printf("{\"ffma_tflops\": %.2f, \"sms\": %d, \"clock_mhz\": %d, \"how\": \"tools/ubench/ffma.cu: 8 independent FFMA chains per thread, %d blocks x 256 threads, best of 5, CUDA events\"}\n",
         best1, sms, khz / 1000, blocks);
  return cudaGetLastError() != cudaSuccess;
}
