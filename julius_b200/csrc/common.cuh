// common.cuh -- shared helpers for libjb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <atomic>
#include <vector>
#include "julius_b200.h"

namespace jb200 {

void set_error(const char *fmt, ...);
extern std::atomic<int64_t> g_launches;

// ---- addlog_array (addlog.c:28-57,102-123): table-driven log-add, used by K1 and K2 ---------------
static constexpr int ADDLOG_TABLE_N = 500000;
// the 500 000-entry log(1 + exp(-x)) table, built with the same libm calls as addlog.c:39-57
void build_addlog_table(std::vector<float> &tbl);
// one step of the walk, addlog.c:112-120: y is the running sum, x the next term.  The drop test compares the float
// difference with the double LOG_ADDMIN; against LOG_ADDMIN rounded up to a float it is the same test.
__device__ __forceinline__ float addlog_step_exact(float y, float x, const float *__restrict__ tbl) {
  if (x > y) { float t = x; x = y; y = t; }
  float tmp = __fsub_rn(x, y);
  if (tmp < __double2float_ru(JB200_LOG_ADDMIN)) return y;
  unsigned int idx = (unsigned int)__dadd_rn(__dmul_rn((double)(-tmp), 33333.3333), 0.5);
  return __fadd_rn(y, __ldg(tbl + idx));
}

// ---- outprob_cd (outprob.c:286-400): a pseudo-phone set's score from the frame's state-score row -------------------
// The cd-set kernel fills the set columns with it and the beam kernels evaluate it on demand.  Plain + and / only: the
// sums have no product to contract, and the beam kernels' machine code depends on the form.
static constexpr int NBEST_MAX = 16;   // largest N of a best-N list: -iwcd1 best N, and -tmix N of the pruned K1 variants
// a model's cd sets on the device: set c holds the states states[off[c] .. off[c+1]), combined by method (JB200_IWCD_*)
struct CdSets { const int *off; const int *states; int method, nbest; };
static __device__ float outprob_cd(const CdSets &cd, const float *__restrict__ row, int c) {
  const int b0 = __ldg(cd.off + c), n_in = __ldg(cd.off + c + 1) - b0;
  if (cd.method == JB200_IWCD_AVG) {
    float sum = 0.0f; int j = 0;
    for (int i = 0; i < n_in; i++) { float v = __ldg(row + __ldg(cd.states + b0 + i)); if (v > JB200_LOG_ZERO) { sum += v; j++; } }
    return sum / (float)j;
  } else if (cd.method == JB200_IWCD_MAX) {
    float mx = JB200_LOG_ZERO;
    for (int i = 0; i < n_in; i++) { float v = __ldg(row + __ldg(cd.states + b0 + i)); if (mx < v) mx = v; }
    return mx;
  }
  const int maxn = cd.nbest;
  if (maxn <= 3) {
    // the kept list is the sorted multiset of the maxn largest valid scores, and the result adds it up from the
    // largest down (outprob.c:313-318): three registers instead of an indexed array in local memory
    float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY; int n = 0;
    for (int i = 0; i < n_in; i++) {
      const float v = __ldg(row + __ldg(cd.states + b0 + i));
      if (v <= JB200_LOG_ZERO) continue;
      n++;
      if (v > m0) { m2 = m1; m1 = m0; m0 = v; }
      else if (v > m1) { m2 = m1; m1 = v; }
      else if (v > m2) m2 = v;
    }
    n = min(n, maxn);
    float prob = 0.0f;
    if (n > 0) prob += m0;
    if (n > 1) prob += m1;
    if (n > 2) prob += m2;
    return prob / (float)n;
  }
  float mp[NBEST_MAX + 1]; int n = 0;
  for (int i = 0; i < n_in; i++) {
    float prob = __ldg(row + __ldg(cd.states + b0 + i));
    if (prob <= JB200_LOG_ZERO) continue;
    if (n == 0 || prob <= mp[n - 1]) {
      if (n == maxn) continue;
      mp[n] = prob; n++;
    } else {
      for (int k = 0; k < n; k++) {
        if (prob > mp[k]) {
          int cnt = n - k - ((n == maxn) ? 1 : 0);
          for (int q = k + cnt; q > k; q--) mp[q] = mp[q - 1];
          mp[k] = prob;
          break;
        }
      }
      if (n < maxn) n++;
    }
  }
  float prob = 0.0f;
  for (int i = 0; i < n; i++) prob += mp[i];
  return prob / (float)n;
}

// ---- DNN input splicing (wav2mfcc.c:160-183, splice_mfcc realtime-1stpass.c:445-460) -------------------------------
// A DNN with context_len ctx > 1 takes frames fl = in_dim / ctx wide; network input row r is the concatenation of ctx
// consecutive frames of a window.  A segment is an utterance of a batch or a stream's feed: its rows start at row0, and
// its window is n_carry frames carried over from earlier feeds (carry[carry0 ..]) followed by its new frames
// (in[frame0 ..]), n_win frames in all.  Row r of the segment reads window frames k = r - row0 .. r - row0 + ctx - 1.
// A table of nseg segments ends with a sentinel whose row0 is the total row count.
struct SpliceSeg { int row0, frame0, carry0, n_carry, n_win; };
struct SpliceMap {
  const SpliceSeg *seg = nullptr;   // device, nseg + 1 entries; nseg == 0: row r is the window in[r .. r + ctx - 1]
  int nseg = 0;
  const float *carry = nullptr;     // device [.][fl]
};
// frame k of segment s's window
__device__ __forceinline__ const float *splice_frame(const SpliceSeg &s, int k, const float *in, const float *carry, int fl) {
  return (k < s.n_carry) ? carry + (size_t)(s.carry0 + k) * fl : in + (size_t)(s.frame0 + k - s.n_carry) * fl;
}

#define JB_CUDA(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      jb200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return JB200_ERR_CUDA;                                                       \
    }                                                                              \
  } while (0)

// passes on a failed JB200_* return code
#define JB_RC(expr)                                                                \
  do {                                                                             \
    const int _rc = (expr);                                                        \
    if (_rc != JB200_OK) return _rc;                                               \
  } while (0)

#define JB_LAUNCH_CHECK()                                                          \
  do {                                                                             \
    jb200::g_launches.fetch_add(1, std::memory_order_relaxed);                     \
    cudaError_t _e = cudaGetLastError();                                           \
    if (_e != cudaSuccess) {                                                       \
      jb200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return JB200_ERR_CUDA;                                                       \
    }                                                                              \
  } while (0)

// ---- mbarrier + 1-D bulk (TMA) copy, global -> shared::cta -------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// bytes must be a multiple of 16; src/dst 16-byte aligned.  SASS: UBLKCP.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

}  // namespace jb200
