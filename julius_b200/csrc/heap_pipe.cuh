// heap_pipe.cuh -- pipelined replay of the extraction loop of sort_token_upward / sort_token_downward
// (libjulius/src/beam.c:1370-1384, :1436-1450) by ONE WARP.  Included by beam.cu and by tools/ubench/heapx.cu.
//
// The reference extracts the beam survivors one by one:  s = A[m]; A[m] = A[1]; m--; sift s down from the root.
// The output order of these extractions decides the next frame's visiting order and exact ties are routine, so
// the loop has to be replayed comparison for comparison.  A single thread needs one shared-memory round trip per
// tree level (~50 cycles) and ~10 levels per extraction.  Here up to NL extractions are in flight, one per lane,
// in lock-step "ticks":
//   * an extraction in flight moves its hole down exactly one level per tick:  read the children pair of the hole,
//     pick the larger (smaller) child, stop test, write the hole, move;
//   * a new extraction starts at the earliest two ticks after its predecessor, so that it reads level L+1 one tick
//     after the predecessor wrote it and never touches a level the predecessor touches in the same tick;
//   * what an extraction writes into the root is the next extraction's output (nobody re-reads the root);
//   * freed tail slots and everything up to the last child slot hold sentinels (heap_pad_sentinels), so the two
//     bounds tests of the reference loop fall out of the value comparisons, and the extracted roots go to `outv`
//     (the tail slots still belong to the larger heaps of older extractions in flight);
//   * the only other coupling is the tail slot an extraction takes its s from (and retires):  an older extraction
//     whose hole sits on an ancestor of that slot, or on the slot, may still compare against its content or end its
//     own sift there.  The new extraction waits until no hole in flight is on that root path (decided on the holes
//     as they are after the tick's move).  With the loser cut of a max-heap select (a sift stops at a child below
//     `lose_below`, a lower bound of the smallest score that can be extracted) a tail slot holding a loser is never read
//     for a decision that matters and never becomes a hole, and a loser stays a loser, so those starts -- 97 % of them
//     on the 20k-word workload -- need no check at all.
// tools/beamcut.cpp runs exactly this schedule on the CPU against the plain loop (tests/test_beamcut.py).
// 1608 ticks for 800 extractions out of ~2430 on the 20k-word workload (tools/beamcut.cpp on a real decode).
#pragma once
#include <cuda_runtime.h>

namespace jb200 {

// volatile: keeps the window address in a register (ptxas otherwise re-derives it from SR_CgaCtaId inside the tick loop)
__device__ __forceinline__ unsigned hp_smem_u32(const void *p) {
  unsigned r;
  asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void hp_lds_one(unsigned addr, unsigned &x0, unsigned &x1) {
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(x0), "=r"(x1) : "r"(addr) : "memory");
}

// ---- predicated stores / loads: a lane that has nothing to do skips the access without leaving the warp's common path
__device__ __forceinline__ void hp_sts_one_if(bool p, unsigned addr, unsigned x0, unsigned x1) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %3, 0; @q st.shared.v2.u32 [%0], {%1,%2}; }"
               :: "r"(addr), "r"(x0), "r"(x1), "r"((unsigned)p) : "memory");
}
__device__ __forceinline__ void hp_lds_one_if(bool p, unsigned addr, unsigned &x0, unsigned &x1) {
  asm volatile("{ .reg .pred q; setp.ne.u32 q, %3, 0; @q ld.shared.v2.u32 {%0,%1}, [%2]; }"
               : "+r"(x0), "+r"(x1) : "r"(addr), "r"((unsigned)p) : "memory");
}

// ---- the loop, written for the issue slots of one warp:
//   * no lane ever leaves the warp's common path: stores and the starting lane's accesses are predicated, every decision
//     is a select (an `if (act) ...` region makes the warp diverge and reconverge in every tick: 257 vs 107 cycles/tick);
//   * the extracted roots go to SHARED memory (`outs`, 8-byte entries; a global store in the tick costs ~40 cycles per
//     extraction);
//   * both possible next pair addresses exist before the child comparison resolves and the stop test is one comparison,
//     so the loop-carried chains are
//     LDS.128 -> FSETP -> SEL -> VIMNMX -> LDS.128     (address)
//     LDS.128 -> FMNMX -> FSETP -> SEL -> STS          (hole)
// An idle lane sits on the sentinel pair `capa`; its "next pair" clamps back to capa by itself (2*capa - hb > capa).
//
// The stop test of a max-heap level, "s >= c || c < lose_below" (c = the larger child), is ONE comparison against
// thr = max(s, nextdown(lose_below)):  if s >= lose_below then c < lose_below implies c <= s, so the test is c <= s;
// otherwise c <= s implies c < lose_below, so the test is c < lose_below, i.e. c <= nextdown(lose_below).
// (Scores are finite or the -inf sentinel, never NaN.)  Min-heap: "s <= c" (c = the smaller child), no cut.
//
// ---- the step in PTX.  One warp issues about one instruction every two cycles however little they depend on each other,
// so once the shared-memory round trip is covered (~64 cycles with the compare and the address select: "tick floor" in
// tools/ubench/heapx.cu) a tick costs its instruction count.  The step below is 24 instructions; the address arithmetic
// that does not need the loaded pair is issued in the load's shadow.  act: 0/1.
template <bool MAXHEAP>
__device__ __forceinline__ void hp_step(unsigned &cur, unsigned &slot, unsigned &act, const unsigned s_lo, const unsigned s_hi,
                                        const float lose_dn, const unsigned out_w, const unsigned nhb, const unsigned capa,
                                        const unsigned root) {
#define HP_STEP_HEAD                                                                                                     \
      "{\n\t"                                                                                                            \
      ".reg .pred pa, pr, ps, pq, pg;\n\t"                                                                               \
      ".reg .b32 x0, x1, y0, y1, clo, chi, plo, phi, b2, b2r, sr;\n\t"                                                   \
      ".reg .f32 fx, fy, fs, cv, thr;\n\t"                                                                               \
      "setp.ne.u32 pa, %2, 0;\n\t"                                                                                       \
      "ld.shared.v4.u32 {x0, x1, y0, y1}, [%0];\n\t"                                                                     \
      "mad.lo.u32 b2, %0, 2, %7;\n\t"             /* 2*cur - hb: the pair below the LEFT child */                        \
      "add.u32 b2r, b2, 16;\n\t"                                                                                         \
      "min.u32 b2, b2, %8;\n\t"                                                                                          \
      "min.u32 b2r, b2r, %8;\n\t"                                                                                        \
      "add.u32 sr, %0, 8;\n\t"                    /* slot of the right child (the left child's is cur) */                \
      "setp.eq.and.u32 pq, %1, %9, pa;\n\t"       /* this lane fills the root: its value is the next output */          \
      "mov.b32 fs, %3;\n\t"
#define HP_STEP_TAIL                                                                                                     \
      "selp.b32 clo, y0, x0, pr;\n\t"                                                                                    \
      "selp.b32 chi, y1, x1, pr;\n\t"                                                                                    \
      "selp.b32 plo, %3, clo, ps;\n\t"                                                                                   \
      "selp.b32 phi, %4, chi, ps;\n\t"                                                                                   \
      "@pa st.shared.v2.u32 [%1], {plo, phi};\n\t"                                                                       \
      "@pq st.shared.v2.u32 [%6], {plo, phi};\n\t"                                                                       \
      "selp.u32 %1, sr, %0, pr;\n\t"              /* the hole moves to the chosen child ... */                           \
      "selp.u32 %0, b2r, b2, pr;\n\t"             /* ... whose children pair is next */                                  \
      "not.pred ps, ps;\n\t"                                                                                             \
      "and.pred pg, pa, ps;\n\t"                                                                                         \
      "selp.u32 %2, 1, 0, pg;\n\t"                                                                                       \
      "}\n"
  if (MAXHEAP)
    asm volatile(HP_STEP_HEAD
                 "max.f32 thr, fs, %5;\n\t"       /* stop test "s >= c || c < lose_below" == "c <= max(s, nextdown(lose_below))" */
                 "mov.b32 fx, x0;\n\t"
                 "mov.b32 fy, y0;\n\t"
                 "setp.lt.f32 pr, fx, fy;\n\t"    /* "child < child+1": the right child only when strictly larger */
                 "max.f32 cv, fx, fy;\n\t"
                 "setp.le.f32 ps, cv, thr;\n\t"
                 HP_STEP_TAIL
                 : "+r"(cur), "+r"(slot), "+r"(act)
                 : "r"(s_lo), "r"(s_hi), "f"(lose_dn), "r"(out_w), "r"(nhb), "r"(capa), "r"(root)
                 : "memory");
  else
    asm volatile(HP_STEP_HEAD
                 "mov.b32 fx, x0;\n\t"
                 "mov.b32 fy, y0;\n\t"
                 "setp.gt.f32 pr, fx, fy;\n\t"    /* "child > child+1": the right child only when strictly smaller */
                 "min.f32 cv, fx, fy;\n\t"
                 "setp.ge.f32 ps, cv, fs;\n\t"    /* "s <= c" */
                 HP_STEP_TAIL
                 : "+r"(cur), "+r"(slot), "+r"(act)
                 : "r"(s_lo), "r"(s_hi), "f"(lose_dn), "r"(out_w), "r"(nhb), "r"(capa), "r"(root)
                 : "memory");
#undef HP_STEP_HEAD
#undef HP_STEP_TAIL
}

// Called by the 32 threads of one warp (lane = 0..31).  A: heap entries (low word = fp32 score bits, high word = token
// id), slot h = heap index h, sentinel padded; n: heap size; outs[k] = k-th extracted root, k = 0..extract (the last
// entry is what would be extracted next).  Returns the number of ticks / held-back starts through the pointers.
template <bool MAXHEAP>
__device__ __forceinline__ void heap_extract_pipe_warp6(unsigned long long *A, const int n, const int extract, const float lose_below,
                                                        unsigned long long *outs, const int maxt, const unsigned lane,
                                                        unsigned &ticks_out, unsigned &stalls_out) {
  constexpr int NL = 16;                                   // extraction x is owned by lane x mod NL
  constexpr unsigned FULL = 0xffffffffu;
  const unsigned hb = hp_smem_u32(A);
  const unsigned ob = hp_smem_u32(outs);
  const unsigned nhb = 0u - hb;
  const unsigned sent = MAXHEAP ? 0xff800000u : 0x7f800000u;
  const unsigned capa = hb + (((unsigned)(maxt >> 1) + 1u) << 4);
  const unsigned root = hb + 8u;
  float lose_dn = lose_below;
  if (MAXHEAP && lose_below > -INFINITY) {
    unsigned b = __float_as_uint(lose_below);
    b = (lose_below > 0.0f) ? b - 1u : (lose_below < 0.0f) ? b + 1u : 0x80000001u;
    lose_dn = __uint_as_float(b);
  }
  unsigned act = 0u, slot = capa, cur = capa;
  unsigned s_lo = sent, s_hi = 0u;
  unsigned out_w = ob;
  int next_x = 0, wait = 0;
  unsigned ticks = 0, stalls = 0;
  unsigned nxt_lo, nxt_hi;
  hp_lds_one(hb + ((unsigned)n << 3), nxt_lo, nxt_hi);
  if (lane == 0 && extract > 0) outs[0] = A[1];
  while (true) {
    hp_step<MAXHEAP>(cur, slot, act, s_lo, s_hi, lose_dn, out_w, nhb, capa, root);
    if (--wait <= 0) {
      if (next_x >= extract) {
        if (!__any_sync(FULL, act != 0u)) break;
      } else {
        const unsigned ms = (unsigned)(n - next_x);
        bool ok = true;
        if (!(MAXHEAP && (__uint_as_float(nxt_lo) < lose_below))) {          // rare with the loser cut
          const unsigned h = (slot - hb) >> 3;
          const int dh = 31 - __clz(h), dms = 31 - __clz(ms);
          ok = !__any_sync(FULL, act != 0u && dms >= dh && (ms >> (dms - dh)) == h);
        }
        if (ok) {
          const bool mine = (lane == ((unsigned)next_x & (NL - 1)));
          const unsigned ma = hb + (ms << 3);
          hp_lds_one_if(mine, ma, s_lo, s_hi);                               // s = A[m]
          hp_sts_one_if(mine, ma, sent, 0u);                                 // slot m leaves the heap
          next_x++;
          out_w = mine ? ob + ((unsigned)next_x << 3) : out_w;               // outs[x + 1]
          hp_lds_one(ma - 8u, nxt_lo, nxt_hi);                               // the next tail slot's content
          act = mine ? 1u : act;
          slot = mine ? root : slot;
          cur = mine ? hb + 16u : cur;
          wait = 2;
        } else stalls++;
      }
    }
    __syncwarp();
    ticks++;
  }
  ticks_out = ticks; stalls_out = stalls;
}

}  // namespace jb200
