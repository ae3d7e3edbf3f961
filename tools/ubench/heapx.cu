// heapx.cu -- micro-benchmark of the beam-cut extraction replay on a realistic heap (n=2400 random scores,
// 800 extractions, loser cut at the 800th largest).  Variants isolate what a level / an extraction costs.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o heapx heapx.cu
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>
#include "../../julius_b200/csrc/heap_pipe.cuh"

#define MAXT 3328
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void lds_pair_spec(unsigned a, unsigned &x0, unsigned &x1, unsigned &y0, unsigned &y1) {
  asm volatile("ld.volatile.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(a) : "memory");
}
__device__ __forceinline__ void lds_pair(unsigned a, unsigned &x0, unsigned &x1, unsigned &y0, unsigned &y1) {
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(y0), "=r"(y1) : "r"(a) : "memory");
}
__device__ __forceinline__ void lds_one(unsigned a, unsigned &x0, unsigned &x1) {
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(x0), "=r"(x1) : "r"(a) : "memory");
}
__device__ __forceinline__ void sts_one(unsigned a, unsigned x0, unsigned x1) {
  asm volatile("st.shared.v2.u32 [%0], {%1,%2};" :: "r"(a), "r"(x0), "r"(x1) : "memory");
}
__device__ __forceinline__ unsigned heap_pick(unsigned x0, unsigned y0, unsigned a_left, unsigned a_right, bool &right) {
  unsigned r, pr;
  asm("{ .reg .pred p; setp.lt.f32 p, %4, %5; selp.u32 %0, %2, %3, p; selp.u32 %1, 1, 0, p; }"
      : "=r"(r), "=r"(pr) : "r"(a_right), "r"(a_left), "f"(__uint_as_float(x0)), "f"(__uint_as_float(y0)));
  right = (pr != 0u);
  return r;
}

// V: 18 = the pipelined warp replay of heap_pipe.cuh (what beam.cu ships);
// single-thread variants: 0 = round 1's loop; 1 = outv in shared memory; 2 = no loser-cut test; 3 = non-volatile (sinkable) load;
//    4 = one level per loop trip (no ping-pong unroll); 5 = plain load whose result is also consumed on the
//    exit path (ptxas must issue it ahead of the stop test); 6 = 5 + both grandchild pairs requested one level
//    ahead (two-level speculation)
#define LEVEL(X0, X1, Y0, Y1, N0, N1, N2, N3)                                                        \
  {                                                                                                  \
    const unsigned u = (cur << 1) - hb;                                                              \
    bool right;                                                                                      \
    const unsigned ncur = heap_pick(X0, Y0, min(u, capa), min(u + 16u, capa), right);                \
    if (V == 3 || V >= 5) lds_pair(ncur, N0, N1, N2, N3); else lds_pair_spec(ncur, N0, N1, N2, N3);  \
    if (V >= 5) sink = N0;                                                                           \
    const unsigned c_lo = right ? Y0 : X0, c_hi = right ? Y1 : X1;                                   \
    levels++;                                                                                        \
    if (sv >= __uint_as_float(c_lo) || (V != 2 && __uint_as_float(c_lo) < lose_below)) break;        \
    sts_one(slot, c_lo, c_hi);                                                                       \
    slot = cur + (right ? 8u : 0u);                                                                  \
    cur = ncur;                                                                                      \
  }

// two tree levels per round trip: the pairs below BOTH children are requested together with the children
template <int V>
__device__ __forceinline__ void extract2(unsigned long long *A, int n, int extract, float lose_below, unsigned long long *outv,
                                         unsigned &levels_out, unsigned &sink_out) {
  unsigned levels = 0, sinkacc = 0;
  const unsigned hb = smem_u32(A);
  const unsigned capa = hb + (((unsigned)(MAXT >> 1) + 1u) << 4);
  unsigned mslot = hb + ((unsigned)n << 3);
  for (int x = 0; x < extract; x++) {
    unsigned s_lo, s_hi, r_lo, r_hi;
    unsigned p0, p1, p2, p3, l0, l1, l2, l3, r0, r1, r2, r3;     // children pair, left child's pair, right child's pair
    lds_one(mslot, s_lo, s_hi);
    sts_one(mslot, 0xff800000u, 0u);
    lds_one(hb + 8u, r_lo, r_hi);
    lds_pair(hb + 16u, p0, p1, p2, p3);
    lds_pair(hb + 32u, l0, l1, l2, l3);
    lds_pair(hb + 48u, r0, r1, r2, r3);
    mslot -= 8u;
    outv[x] = ((unsigned long long)r_hi << 32) | r_lo;
    const float sv = __uint_as_float(s_lo);
    unsigned slot = hb + 8u, cur = hb + 16u;
    while (true) {
      // level A
      const bool ra = __uint_as_float(p0) < __uint_as_float(p2);
      const unsigned ca_lo = ra ? p2 : p0, ca_hi = ra ? p3 : p1;
      const unsigned g0 = ra ? r0 : l0, g1 = ra ? r1 : l1, g2 = ra ? r2 : l2, g3 = ra ? r3 : l3;
      const unsigned ua = (cur << 1) - hb;
      const unsigned cura = ra ? ua + 16u : ua;                 // pair of the chosen child (what g* holds); may exceed the array
      // level B
      const bool rb = __uint_as_float(g0) < __uint_as_float(g2);
      const unsigned ub = (cura << 1) - hb;
      const unsigned curb = min(rb ? ub + 16u : ub, capa);
      const unsigned uc = (curb << 1) - hb;
      lds_pair(curb, p0, p1, p2, p3);                           // speculative: next round's three pairs
      lds_pair(min(uc, capa), l0, l1, l2, l3);
      lds_pair(min(uc + 16u, capa), r0, r1, r2, r3);
      sinkacc += p0 ^ l0 ^ r0;
      levels++;
      if (sv >= __uint_as_float(ca_lo) || __uint_as_float(ca_lo) < lose_below) break;
      sts_one(slot, ca_lo, ca_hi);
      slot = cur + (ra ? 8u : 0u);
      const unsigned cb_lo = rb ? g2 : g0, cb_hi = rb ? g3 : g1;
      levels++;
      if (sv >= __uint_as_float(cb_lo) || __uint_as_float(cb_lo) < lose_below) break;
      sts_one(slot, cb_lo, cb_hi);
      slot = min(cura, capa) + (rb ? 8u : 0u);
      cur = curb;
    }
    sts_one(slot, s_lo, s_hi);
  }
  levels_out = levels; sink_out = sinkacc;
}

// variant 7: no address clamp while the speculative address cannot leave the array (the first SAFE levels)
#define LEVEL_NC(X0, X1, Y0, Y1, N0, N1, N2, N3)                                                     \
  {                                                                                                  \
    const unsigned u = (cur << 1) - hb;                                                              \
    bool right;                                                                                      \
    const unsigned ncur = heap_pick(X0, Y0, u, u + 16u, right);                                      \
    lds_pair(ncur, N0, N1, N2, N3);                                                                  \
    sink = N0;                                                                                       \
    const unsigned c_lo = right ? Y0 : X0, c_hi = right ? Y1 : X1;                                   \
    levels++;                                                                                        \
    if (sv >= __uint_as_float(c_lo) || __uint_as_float(c_lo) < lose_below) goto done;                \
    sts_one(slot, c_lo, c_hi);                                                                       \
    slot = cur + (right ? 8u : 0u);                                                                  \
    cur = ncur;                                                                                      \
  }
#define LEVEL_C(X0, X1, Y0, Y1, N0, N1, N2, N3)                                                      \
  {                                                                                                  \
    const unsigned u = (cur << 1) - hb;                                                              \
    bool right;                                                                                      \
    const unsigned ncur = heap_pick(X0, Y0, min(u, capa), min(u + 16u, capa), right);                \
    lds_pair(ncur, N0, N1, N2, N3);                                                                  \
    sink = N0;                                                                                       \
    const unsigned c_lo = right ? Y0 : X0, c_hi = right ? Y1 : X1;                                   \
    levels++;                                                                                        \
    if (sv >= __uint_as_float(c_lo) || __uint_as_float(c_lo) < lose_below) goto done;                \
    sts_one(slot, c_lo, c_hi);                                                                       \
    slot = cur + (right ? 8u : 0u);                                                                  \
    cur = ncur;                                                                                      \
  }
__device__ __forceinline__ void extract7(unsigned long long *A, int n, int extract, float lose_below, unsigned long long *outv,
                                         unsigned &levels_out, unsigned &sink_out) {
  unsigned levels = 0, sinkacc = 0, sink = 0;
  const unsigned hb = smem_u32(A);
  const unsigned capa = hb + (((unsigned)(MAXT >> 1) + 1u) << 4);
  unsigned mslot = hb + ((unsigned)n << 3);
  int safe = 0; while ((4 << (safe + 1)) <= MAXT) safe++;       // levels whose grandchild pair index stays below MAXT/2
  safe &= ~1;
  for (int x = 0; x < extract; x++) {
    unsigned s_lo, s_hi, r_lo, r_hi, x0, x1, y0, y1, z0, z1, w0, w1;
    lds_one(mslot, s_lo, s_hi);
    sts_one(mslot, 0xff800000u, 0u);
    lds_one(hb + 8u, r_lo, r_hi);
    lds_pair(hb + 16u, x0, x1, y0, y1);
    mslot -= 8u;
    outv[x] = ((unsigned long long)r_hi << 32) | r_lo;
    const float sv = __uint_as_float(s_lo);
    unsigned slot = hb + 8u, cur = hb + 16u;
    for (int lv = 0; lv < safe; lv += 2) {
      LEVEL_NC(x0, x1, y0, y1, z0, z1, w0, w1)
      LEVEL_NC(z0, z1, w0, w1, x0, x1, y0, y1)
    }
    while (true) {
      LEVEL_C(x0, x1, y0, y1, z0, z1, w0, w1)
      LEVEL_C(z0, z1, w0, w1, x0, x1, y0, y1)
    }
  done:
    sts_one(slot, s_lo, s_hi);
    sinkacc += sink;
  }
  levels_out = levels; sink_out = sinkacc;
}

// variant 8: the top four levels of the heap (slots 1..15) live in REGISTERS of the extracting thread.  A sift through
// them is a compile-time decision tree (sift_reg<P> knows its slot P, so every register index is static); only below
// slot 15 does the shared-memory loop of variant 5 take over.  Saves the LDS round trip on the first four levels.
struct SiftState { unsigned slot, cur; bool done; };

template <int P>
__device__ __forceinline__ void sift_reg(unsigned (&rv)[16], unsigned (&ri)[16], const unsigned s_lo, const unsigned s_hi, const float sv,
                                         const float lose_below, const unsigned hb, unsigned &levels, SiftState &st) {
  if constexpr (P >= 8) {
    // children of P are the shared-memory slots 2P, 2P+1: one level by hand (its store target is a register)
    unsigned x0, x1, y0, y1;
    lds_pair(hb + (unsigned)P * 16u, x0, x1, y0, y1);
    const bool right = __uint_as_float(x0) < __uint_as_float(y0);
    const unsigned c_lo = right ? y0 : x0, c_hi = right ? y1 : x1;
    levels++;
    if (sv >= __uint_as_float(c_lo) || __uint_as_float(c_lo) < lose_below) { rv[P] = s_lo; ri[P] = s_hi; st.done = true; return; }
    rv[P] = c_lo; ri[P] = c_hi;
    st.slot = hb + (unsigned)(2 * P) * 8u + (right ? 8u : 0u);        // the chosen child's slot
    st.cur = hb + ((unsigned)(2 * P) + (right ? 1u : 0u)) * 16u;      // the pair below it
    st.done = false;
  } else {
    levels++;
    if (__uint_as_float(rv[2 * P]) < __uint_as_float(rv[2 * P + 1])) {
      if (sv >= __uint_as_float(rv[2 * P + 1]) || __uint_as_float(rv[2 * P + 1]) < lose_below) { rv[P] = s_lo; ri[P] = s_hi; st.done = true; return; }
      rv[P] = rv[2 * P + 1]; ri[P] = ri[2 * P + 1];
      sift_reg<2 * P + 1>(rv, ri, s_lo, s_hi, sv, lose_below, hb, levels, st);
    } else {
      if (sv >= __uint_as_float(rv[2 * P]) || __uint_as_float(rv[2 * P]) < lose_below) { rv[P] = s_lo; ri[P] = s_hi; st.done = true; return; }
      rv[P] = rv[2 * P]; ri[P] = ri[2 * P];
      sift_reg<2 * P>(rv, ri, s_lo, s_hi, sv, lose_below, hb, levels, st);
    }
  }
}

__device__ __forceinline__ void extract8(unsigned long long *A, int n, int extract, float lose_below, unsigned long long *outv,
                                         unsigned &levels_out, unsigned &sink_out) {
  unsigned levels = 0, sinkacc = 0, sink = 0;
  const unsigned hb = smem_u32(A);
  const unsigned capa = hb + (((unsigned)(MAXT >> 1) + 1u) << 4);
  unsigned mslot = hb + ((unsigned)n << 3);
  unsigned rv[16], ri[16];
#pragma unroll
  for (int i = 1; i < 16; i++) { rv[i] = (unsigned)A[i]; ri[i] = (unsigned)(A[i] >> 32); }
  for (int x = 0; x < extract; x++) {
    unsigned s_lo, s_hi;
    lds_one(mslot, s_lo, s_hi);
    sts_one(mslot, 0xff800000u, 0u);
    mslot -= 8u;
    outv[x] = ((unsigned long long)ri[1] << 32) | rv[1];
    const float sv = __uint_as_float(s_lo);
    SiftState st;
    sift_reg<1>(rv, ri, s_lo, s_hi, sv, lose_below, hb, levels, st);
    if (!st.done) {
      unsigned slot = st.slot, cur = st.cur;
      unsigned x0, x1, y0, y1, z0, z1, w0, w1;
      lds_pair(cur, x0, x1, y0, y1);
      while (true) {
        LEVEL_C(x0, x1, y0, y1, z0, z1, w0, w1)
        LEVEL_C(z0, z1, w0, w1, x0, x1, y0, y1)
      }
    done:
      sts_one(slot, s_lo, s_hi);
      sinkacc += sink;
    }
  }
  levels_out = levels; sink_out = sinkacc;
}

template <int V>
__global__ void __launch_bounds__(256, 4) k(const unsigned long long *init, int n, int extract_in, float lose_below,
                                            unsigned long long *outg, long long *res) {
  __shared__ __align__(16) unsigned long long A[MAXT + 4];
  __shared__ unsigned long long outs[1024];
  for (int i = threadIdx.x; i < MAXT + 4; i += blockDim.x) A[i] = (i >= 1 && i <= n) ? init[i] : 0xff800000ull;
  __syncthreads();
  int extract = extract_in;
  if (V == 18) {
    if (threadIdx.x < 32) {
      unsigned ticks, stalls;
      long long t0 = clock64();
      jb200::heap_extract_pipe_warp6<true>(A, n, extract, lose_below, outs, MAXT, threadIdx.x, ticks, stalls);
      long long t1 = clock64();
      if (threadIdx.x == 0) { res[blockIdx.x * 2] = t1 - t0; res[blockIdx.x * 2 + 1] = ticks; }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < extract_in; i += blockDim.x) outg[(size_t)blockIdx.x * 1024 + i] = outs[i];
    return;
  }
  if (threadIdx.x == 0) {
    unsigned long long *outv = (V == 1) ? outs : outg + (size_t)blockIdx.x * 1024;
    unsigned levels = 0, sink = 0, sinkacc = 0;
    const unsigned hb = smem_u32(A);
    const unsigned capa = hb + (((unsigned)(MAXT >> 1) + 1u) << 4);
    unsigned mslot = hb + ((unsigned)n << 3);
    long long t0 = clock64();
    if (V == 6) { extract2<V>(A, n, extract, lose_below, outv, levels, sinkacc); extract = 0; }
    if (V == 7) { extract7(A, n, extract, lose_below, outv, levels, sinkacc); extract = 0; }
    if (V == 8) { extract8(A, n, extract, lose_below, outv, levels, sinkacc); extract = 0; }
    for (int x = 0; x < extract; x++) {
      unsigned s_lo, s_hi, r_lo, r_hi, x0, x1, y0, y1, z0, z1, w0, w1;
      lds_one(mslot, s_lo, s_hi);
      sts_one(mslot, 0xff800000u, 0u);
      lds_one(hb + 8u, r_lo, r_hi);
      lds_pair(hb + 16u, x0, x1, y0, y1);
      mslot -= 8u;
      outv[x] = ((unsigned long long)r_hi << 32) | r_lo;
      const float sv = __uint_as_float(s_lo);
      unsigned slot = hb + 8u, cur = hb + 16u;
      if (V == 4) {
        while (true) {
          LEVEL(x0, x1, y0, y1, z0, z1, w0, w1)
          x0 = z0; x1 = z1; y0 = w0; y1 = w1;
        }
      } else {
        while (true) {
          LEVEL(x0, x1, y0, y1, z0, z1, w0, w1)
          LEVEL(z0, z1, w0, w1, x0, x1, y0, y1)
        }
      }
      sts_one(slot, s_lo, s_hi);
      sinkacc += sink;
    }
    long long t1 = clock64();
    if (V >= 5) outv[1000] = sinkacc;
    res[blockIdx.x * 2] = t1 - t0;
    res[blockIdx.x * 2 + 1] = levels;
  }
  __syncthreads();
  if (blockIdx.x == 0 && V == 1) for (int i = threadIdx.x; i < extract_in; i += blockDim.x) outg[i] = outs[i];
}

// floor of a tick: 16 lanes walk down the heap (read-only) picking the larger child, restarting at the root from a leaf.
// MODE 0: load + compare + address select only; MODE 1: plus one predicated 8-byte store per level (to a scratch copy of
// the slot); MODE 2: MODE 1 plus __syncwarp per level.
template <int MODE>
__global__ void __launch_bounds__(256, 4) kfloor(const unsigned long long *init, int n, int nticks, long long *res) {
  __shared__ __align__(16) unsigned long long A[MAXT + 4];
  __shared__ __align__(16) unsigned long long scratch[64];
  for (int i = threadIdx.x; i < MAXT + 4; i += blockDim.x) A[i] = (i >= 1 && i <= n) ? init[i] : 0xff800000ull;
  __syncthreads();
  if (threadIdx.x < 32) {
    const unsigned hb = jb200::hp_smem_u32(A), sb = jb200::hp_smem_u32(scratch);
    const unsigned capa = hb + (((unsigned)(MAXT >> 1) + 1u) << 4);
    unsigned cur = (threadIdx.x < 16) ? hb + 16u : capa;
    unsigned acc = 0;
    long long t0 = clock64();
    for (int t = 0; t < nticks; t++) {
      unsigned x0, x1, y0, y1;
      lds_pair(cur, x0, x1, y0, y1);
      const bool right = __uint_as_float(x0) < __uint_as_float(y0);
      const unsigned base2 = (cur << 1) - hb;
      unsigned ncur = min(base2 + (right ? 16u : 0u), capa);
      if (MODE >= 1) jb200::hp_sts_one_if(threadIdx.x < 16, sb + (threadIdx.x << 3), right ? y0 : x0, right ? y1 : x1);
      acc += right ? y1 : x1;
      cur = (ncur == capa && threadIdx.x < 16) ? hb + 16u : ncur;
      if (MODE >= 2) __syncwarp();
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) { res[blockIdx.x * 2] = t1 - t0; res[blockIdx.x * 2 + 1] = acc; }
  }
}

int main() {
  const int n = 2400, extract = 800;
  std::vector<unsigned long long> h(MAXT + 4, 0);
  std::vector<float> sc(n + 1);
  srand(7);
  for (int i = 1; i <= n; i++) sc[i] = -30000.0f - (float)(rand() % 200000) / 512.0f;     // coarse grid => ties
  // host max-heap build (same sift-down as the reference) so that the device starts from a valid heap
  auto val = [&](int i) { return sc[i]; };
  std::vector<int> idx(n + 1); for (int i = 1; i <= n; i++) idx[i] = i;
  for (int root = n / 2; root >= 1; root--) {
    int s = idx[root]; int parent = root, child;
    while ((child = parent * 2) <= n) {
      if (child < n && val(idx[child]) < val(idx[child + 1])) child++;
      if (val(s) >= val(idx[child])) break;
      idx[parent] = idx[child]; parent = child;
    }
    idx[parent] = s;
  }
  for (int i = 1; i <= n; i++) { unsigned b; float f = sc[idx[i]]; memcpy(&b, &f, 4); h[i] = ((unsigned long long)idx[i] << 32) | b; }
  std::vector<float> sorted(sc.begin() + 1, sc.end()); std::sort(sorted.begin(), sorted.end(), std::greater<float>());
  const float lose_below = sorted[extract - 1] - 0.5f;
  // host reference extraction order
  std::vector<int> ref;
  { std::vector<int> a(idx); int m = n;
    for (int x = 0; x < extract; x++) { int s = a[m]; ref.push_back(a[1]); a[m] = a[1]; m--; int parent = 1, child;
      while ((child = parent * 2) <= m) { if (child < m && val(a[child]) < val(a[child + 1])) child++; if (val(s) >= val(a[child])) break; a[parent] = a[child]; parent = child; }
      a[parent] = s; } }
  constexpr int WAVE = 4 * 132;   // one resident wave of beam blocks on an H100: 4 per SM
  unsigned long long *d, *o; long long *r, hr[2 * WAVE];
  cudaMalloc(&d, sizeof(unsigned long long) * (MAXT + 4)); cudaMemcpy(d, h.data(), sizeof(unsigned long long) * (MAXT + 4), cudaMemcpyHostToDevice);
  cudaMalloc(&o, sizeof(unsigned long long) * 1024 * WAVE); cudaMalloc(&r, sizeof(hr));
  std::vector<unsigned long long> ho(1024);
  for (int blocks : {1, WAVE}) for (int mode = 0; mode < 3; mode++) {
    const int nt = 4000;
    for (int rep = 0; rep < 2; rep++) {
      if (mode == 0) kfloor<0><<<blocks, 256>>>(d, n, nt, r); else if (mode == 1) kfloor<1><<<blocks, 256>>>(d, n, nt, r); else kfloor<2><<<blocks, 256>>>(d, n, nt, r);
      cudaDeviceSynchronize();
    }
    cudaMemcpy(hr, r, sizeof(long long) * 2 * blocks, cudaMemcpyDeviceToHost);
    double sfl = 0; for (int b = 0; b < blocks; b++) sfl += (double)hr[2 * b];
    printf("blocks %3d tick floor mode %d: %.1f cycles/tick\n", blocks, mode, sfl / blocks / nt);
  }
  for (int blocks : {1, WAVE}) {
    for (int v : {5, 18}) {
      for (int rep = 0; rep < 2; rep++) {
        switch (v) {
          case 0: k<0><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 1: k<1><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 2: k<2><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 3: k<3><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 4: k<4><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 5: k<5><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 6: k<6><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 7: k<7><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 8: k<8><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
          case 18: k<18><<<blocks, 256>>>(d, n, extract, lose_below, o, r); break;
        }
        cudaDeviceSynchronize();
      }
      cudaMemcpy(hr, r, sizeof(long long) * 2 * blocks, cudaMemcpyDeviceToHost);
      cudaMemcpy(ho.data(), o, sizeof(unsigned long long) * 1024, cudaMemcpyDeviceToHost);
      int bad = 0; for (int x = 0; x < extract; x++) if ((int)(ho[x] >> 32) != ref[x]) bad++;
      double s = 0, l = 0; for (int b = 0; b < blocks; b++) { s += (double)hr[2 * b]; l += (double)hr[2 * b + 1]; }
      printf("blocks %3d variant %d: %.0f cycles/extraction, %.2f levels(ticks)/extraction, %.1f cycles/level(tick), order mismatches %d\n",
             blocks, v, s / blocks / extract, l / blocks / extract, s / l, bad);
    }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { printf("CUDA error %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}
