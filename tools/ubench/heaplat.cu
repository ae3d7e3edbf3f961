// heaplat.cu -- micro-benchmark: what does one level of the single-thread heap sift cost on sm_90a?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o heaplat heaplat.cu ; run on an H100.
// Each variant walks root->leaf paths of a 4096-entry (id,score) heap in shared memory, ITER times, and
// reports cycles per level (clock64 around the loop, thread 0 of a 256-thread block, others at a barrier).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define N 4096
#define LEVELS 10
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void lds_pair(unsigned a, unsigned &x0, unsigned &x1, unsigned &y0, unsigned &y1) {
  asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(a) : "memory");
}
__device__ __forceinline__ void lds_pair_nv(unsigned a, unsigned &x0, unsigned &x1, unsigned &y0, unsigned &y1) {
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(a) : "memory");
}
__device__ __forceinline__ void lds_one(unsigned a, unsigned &x0) {
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x0) : "r"(a) : "memory");
}
__device__ __forceinline__ void sts_one(unsigned a, unsigned x0, unsigned x1) {
  asm volatile("st.shared.v2.u32 [%0], {%1,%2};" :: "r"(a), "r"(x0), "r"(x1) : "memory");
}

template <int V>
__global__ void __launch_bounds__(256, 4) k(const float *init, long long *out, int iters) {
  __shared__ __align__(16) unsigned long long A[N + 8];
  for (int i = threadIdx.x; i < N + 8; i += blockDim.x) A[i] = ((unsigned long long)i << 32) | __float_as_uint(init[i % N]);
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned hb = smem_u32(A);
    unsigned acc = 0;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
      unsigned cur = hb + 16u, slot = hb + 8u;
      unsigned x0, x1, y0, y1;
      if (V == 0) {            // pure pointer chase through LDS.32 (address from data)
        unsigned a = hb + 8u;
        for (int l = 0; l < LEVELS; l++) { unsigned v; lds_one(a, v); a = hb + ((v & 0xfffu) << 3); }
        acc += a;
      } else if (V == 1) {     // LDS.128 -> FSETP -> select address -> LDS.128
        lds_pair_nv(cur, x0, x1, y0, y1);
        for (int l = 0; l < LEVELS; l++) {
          const unsigned u = (cur << 1) - hb;
          const bool r = __uint_as_float(x0) < __uint_as_float(y0);
          cur = r ? u + 16u : u;
          lds_pair_nv(cur, x0, x1, y0, y1);
        }
        acc += x1;
      } else if (V == 2) {     // + STS.64 of the chosen child to the parent slot
        lds_pair_nv(cur, x0, x1, y0, y1);
        for (int l = 0; l < LEVELS; l++) {
          const unsigned u = (cur << 1) - hb;
          const bool r = __uint_as_float(x0) < __uint_as_float(y0);
          const unsigned nc = r ? u + 16u : u;
          const unsigned c0 = r ? y0 : x0, c1 = r ? y1 : x1;
          sts_one(slot, c0, c1);
          slot = cur + (r ? 8u : 0u);
          cur = nc;
          lds_pair_nv(cur, x0, x1, y0, y1);
        }
        acc += x1;
      } else if (V == 3) {     // + stop test (never taken) after the speculative volatile load
        const float sv = -1e30f;
        lds_pair(cur, x0, x1, y0, y1);
        for (int l = 0; l < LEVELS; l++) {
          const unsigned u = (cur << 1) - hb;
          const bool r = __uint_as_float(x0) < __uint_as_float(y0);
          const unsigned nc = r ? u + 16u : u;
          unsigned n0, n1, n2, n3;
          lds_pair(nc, n0, n1, n2, n3);
          const unsigned c0 = r ? y0 : x0, c1 = r ? y1 : x1;
          if (sv >= __uint_as_float(c0)) break;
          sts_one(slot, c0, c1);
          slot = cur + (r ? 8u : 0u);
          cur = nc; x0 = n0; x1 = n1; y0 = n2; y1 = n3;
        }
        acc += x1;
      } else if (V == 4) {     // two independent chains interleaved in one thread (ILP 2)
        unsigned curb = hb + 16u, z0, z1, w0, w1;
        lds_pair_nv(cur, x0, x1, y0, y1);
        lds_pair_nv(curb, z0, z1, w0, w1);
        for (int l = 0; l < LEVELS; l++) {
          const unsigned u = (cur << 1) - hb, ub = (curb << 1) - hb;
          const bool r = __uint_as_float(x0) < __uint_as_float(y0);
          const bool rb = __uint_as_float(z0) > __uint_as_float(w0);
          cur = r ? u + 16u : u; curb = rb ? ub + 16u : ub;
          lds_pair_nv(cur, x0, x1, y0, y1);
          lds_pair_nv(curb, z0, z1, w0, w1);
        }
        acc += x1 + z1;
      } else if (V == 5) {     // dependent ALU chain only (no memory): fsetp -> sel, LEVELS times
        unsigned a = cur; float f = init[0];
        for (int l = 0; l < LEVELS; l++) {
          const bool r = __uint_as_float(a) < f;
          a = r ? (a << 1) + 16u : (a << 1) - 3u;
        }
        acc += a;
      }
    }
    long long t1 = clock64();
    out[blockIdx.x * 2] = t1 - t0;
    out[blockIdx.x * 2 + 1] = acc;
  }
  __syncthreads();
}

int main() {
  float *h = (float *)malloc(N * 4);
  srand(1);
  // a valid max-heap by construction: value decreases with depth
  for (int i = 0; i < N; i++) { int d = 0, j = i; while (j > 1) { j >>= 1; d++; } h[i] = -1000.0f * d - (rand() % 997); }
  float *d; long long *o, ho[2 * 592];
  cudaMalloc(&d, N * 4); cudaMemcpy(d, h, N * 4, cudaMemcpyHostToDevice);
  cudaMalloc(&o, sizeof(ho));
  const int iters = 2000;
  for (int blocks : {1, 132, 528}) {
    for (int v = 0; v < 6; v++) {
      for (int rep = 0; rep < 2; rep++) {
        switch (v) {
          case 0: k<0><<<blocks, 256>>>(d, o, iters); break;
          case 1: k<1><<<blocks, 256>>>(d, o, iters); break;
          case 2: k<2><<<blocks, 256>>>(d, o, iters); break;
          case 3: k<3><<<blocks, 256>>>(d, o, iters); break;
          case 4: k<4><<<blocks, 256>>>(d, o, iters); break;
          case 5: k<5><<<blocks, 256>>>(d, o, iters); break;
        }
        cudaDeviceSynchronize();
      }
      cudaMemcpy(ho, o, sizeof(long long) * 2 * blocks, cudaMemcpyDeviceToHost);
      double s = 0; for (int b = 0; b < blocks; b++) s += (double)ho[2 * b];
      printf("blocks %3d variant %d: %.1f cycles/level%s\n", blocks, v, s / blocks / iters / LEVELS, v == 4 ? " (two chains)" : "");
    }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { printf("CUDA error %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}
