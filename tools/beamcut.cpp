// tools/beamcut.cpp -- CPU models of the beam cut (beam_cut in csrc/beam.cu), each checked against the reference's
// select loop (sort_token_upward / sort_token_downward, libjulius/src/beam.c:1342-1447).
//
//   g++ -O2 -o beamcut tools/beamcut.cpp
//   beamcut random <distinct scores> <trials>   random heaps; few distinct scores = many exact ties
//   beamcut --dump <file>                       the cuts of a real decode, recorded by tools/dump_heaps.py
//   beamcut sort <max log2>                     the candidate sort network against std::sort
//
// The models, one per step the kernel runs:
//   1. replay        heap_pad_sentinels + heap_extract_pipe_warp6 / heap_extract_pipe_global (heap_pipe.cuh);
//   2. closed form   heap_select_closed: collection, packed keys, sort (3.), flagging test, closed_relocate lane by lane;
//   3. sort network  sort_tile_pass + the strided stages of heap_select_closed;
//   4. invariant (I) the statement closed_relocate implements, with subtree queries (DESIGN.md, K3, cut item 3).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <random>
#include <string>
#include <vector>

typedef unsigned long long u64;

// the kernel's constants
constexpr int NL = 16;               // extractions in flight, one per lane (heap_pipe.cuh)
constexpr int SORT_TILE = 128;       // keys per warp in sort_tile_pass
constexpr int RELOC_WINDOW = 3;      // 32-key chunks per load round of closed_relocate's scans
constexpr int TIE_LOOKAHEAD = 8;     // how far the flagging test follows a tie group before it assumes the worst

struct Ent { int id; float v; };

static int depth(int h) { return 31 - __builtin_clz(h); }

// ---- the reference ---------------------------------------------------------------------------------------------------
template <bool MAXHEAP> static bool hcmp(float a, float b) { return MAXHEAP ? (a < b) : (a > b); }      // "child < child+1"
template <bool MAXHEAP> static bool hstop(float s, float c) { return MAXHEAP ? (s >= c) : (s <= c); }   // "STVAL >= SVAL(child)"

template <bool MAXHEAP>
static void sift_down(std::vector<Ent> &A, int start, int n) {
  Ent s = A[start];
  int parent = start, child;
  while ((child = parent * 2) <= n) {
    if (child < n && hcmp<MAXHEAP>(A[child].v, A[child + 1].v)) child++;
    if (hstop<MAXHEAP>(s.v, A[child].v)) break;
    A[parent] = A[child];
    parent = child;
  }
  A[parent] = s;
}
template <bool MAXHEAP>
static void heap_build(std::vector<Ent> &A, int n) { for (int root = n / 2; root >= 1; root--) sift_down<MAXHEAP>(A, root, n); }

// build + extraction in place: the k-th extracted root ends in slot n-k, what is left of the heap in slots 1..n-extract
template <bool MAXHEAP>
static void reference_select(std::vector<Ent> &A, int n, int extract) {
  heap_build<MAXHEAP>(A, n);
  int m = n;
  while (m > n - extract) {
    Ent s = A[m];
    A[m] = A[1];
    m--;
    if (m < 1) break;
    A[1] = s;
    sift_down<MAXHEAP>(A, 1, m);
  }
}

// ---- the tree of n slots, as heap_select_closed computes it -------------------------------------------------------------
// closed_subtree_size: the slots of subtree(c) among 1..n, H = depth(n)
static int subtree_size(int c, int n, int H) {
  const int dc = depth(c);
  if (dc > H) return 0;
  const int sh = H - dc;
  const int first = c << sh, width = 1 << sh;
  return (width - 1) + std::max(0, std::min(n - first + 1, width));
}
// pre-order position of slot h: a level of the root path costs 1, and where it turns right the left sibling's subtree
static int preorder(int h, int n, int H) {
  const int d = depth(h);
  int pre = d;
  for (int b = d - 1; b >= 0; b--)
    if ((h >> b) & 1) pre += subtree_size((h >> b) ^ 1, n, H);
  return pre;
}
// order-preserving key of a score (fkey in csrc/common.cuh)
static unsigned fkey(float f) { unsigned b; memcpy(&b, &f, 4); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }

// ---- 1. the pipelined replay ---------------------------------------------------------------------------------------------
// A: the heap area of the kernel, maxt + 4 slots, the input in slots 1..n.  One warp in lock-step ticks: extraction x is
// owned by lane x mod NL and moves its hole one level per tick; a tick (1) reads the children pair of every hole in
// flight, (2) writes the holes and moves them, (3) decides on the holes as they now are whether the next extraction may
// start: not earlier than two ticks after its predecessor, and not while a hole sits on the root path of the tail slot it
// takes -- a vote skipped when that slot held a loser when the predecessor started (a loser never becomes a hole).
// outs[k] = k-th extracted root, k = 0..extract.  Counts ticks and held-back starts.
struct ReplayStats { long ticks = 0, held = 0; };
template <bool MAXHEAP>
static void replay(std::vector<Ent> &A, int n, int extract, int maxt, float lose_below, std::vector<Ent> &outs, ReplayStats &st) {
  const Ent sent{0, MAXHEAP ? -INFINITY : INFINITY};
  for (int i = n + 1; i <= std::min(2 * n + 1, maxt + 1); i++) A[i] = sent;       // heap_pad_sentinels
  A.at(maxt + 2) = A.at(maxt + 3) = sent;
  heap_build<MAXHEAP>(A, n);
  const int cap = maxt / 2 + 1;                                                     // pair index of (maxt+2, maxt+3)
  struct Lane { bool act = false; int x = 0, slot = 0, cur = 0; Ent s{0, 0}; };
  std::vector<Lane> L(NL);
  outs.assign(extract + 1, Ent{-1, 0});
  if (extract > 0) outs[0] = A[1];
  Ent nxt = A[n];                                                                   // content of the next tail slot
  int next_x = 0, wait = 0;
  while (true) {
    Ent rx[NL], ry[NL];
    for (int k = 0; k < NL; k++) if (L[k].act) { rx[k] = A.at(2 * L[k].cur); ry[k] = A.at(2 * L[k].cur + 1); }
    bool any = false;
    for (int k = 0; k < NL; k++) if (L[k].act) {
      Lane &l = L[k];
      const bool right = hcmp<MAXHEAP>(rx[k].v, ry[k].v);
      const Ent c = right ? ry[k] : rx[k];
      const bool stop = hstop<MAXHEAP>(l.s.v, c.v) || (MAXHEAP && c.v < lose_below);
      const Ent put = stop ? l.s : c;
      A[l.slot] = put;
      if (l.slot == 1) outs[l.x + 1] = put;              // what goes into the root is the next extraction's output
      if (stop) l.act = false;
      else { const int child = 2 * l.cur + (right ? 1 : 0); l.slot = child; l.cur = std::min(child, cap); }
      any |= l.act;
    }
    if (--wait <= 0) {
      if (next_x >= extract) {
        if (!any) break;
      } else {
        const int ms = n - next_x, ln = next_x % NL;
        bool blocked = L[ln].act;                          // (heap_extract_pipe_global only; never true: a sift ends
                                                           // within the 2 NL ticks its lane's next start is away)
        if (!(MAXHEAP && nxt.v < lose_below))
          for (int k = 0; k < NL; k++)
            if (L[k].act && depth(ms) >= depth(L[k].slot) && (ms >> (depth(ms) - depth(L[k].slot))) == L[k].slot) blocked = true;
        if (!blocked) {
          Lane &l = L[ln];
          l.s = A[ms]; A[ms] = sent;                       // the slot leaves the heap
          l.x = next_x; l.act = true; l.slot = 1; l.cur = 1;
          next_x++; wait = 2;
          nxt = A[n - next_x];
        } else st.held++;
      }
    }
    st.ticks++;
  }
}

// ---- 3. the sort network ------------------------------------------------------------------------------------------------
static void sort_cx(u64 &a, u64 &b, const bool desc) { if (desc ? (a < b) : (a > b)) std::swap(a, b); }

// sort_tile_pass: key 32 r + l of a tile in register r of lane l; distance 64 and 32 between registers, 16 ... 1 with
// lane l ^ j.  The tiles are independent, so the order in which warps take them does not matter.
static void sort_tile_pass(std::vector<u64> &keys, const int nc, const int np, const int k_lo, const int k_hi) {
  for (int tile = 0; tile * SORT_TILE < np; tile++) {
    u64 v[32][4];
    for (int lane = 0; lane < 32; lane++)
      for (int r = 0; r < 4; r++) { const int i = tile * SORT_TILE + 32 * r + lane; v[lane][r] = (i < nc) ? keys[i] : 0ull; }
    for (int k = k_lo; k <= k_hi; k <<= 1) {
      for (int lane = 0; lane < 32; lane++) {
        const int i0 = tile * SORT_TILE + lane;
        if (k >= 128) { sort_cx(v[lane][0], v[lane][2], (i0 & k) == 0); sort_cx(v[lane][1], v[lane][3], (i0 & k) == 0); }
        if (k >= 64) { sort_cx(v[lane][0], v[lane][1], (i0 & k) == 0); sort_cx(v[lane][2], v[lane][3], ((i0 + 64) & k) == 0); }
      }
      for (int j = std::min(k >> 1, 16); j > 0; j >>= 1) {
        u64 o[32][4];
        for (int lane = 0; lane < 32; lane++) for (int r = 0; r < 4; r++) o[lane][r] = v[lane ^ j][r];     // the shuffle
        for (int lane = 0; lane < 32; lane++) {
          const int i0 = tile * SORT_TILE + lane;
          const bool low = ((lane & j) == 0);
          for (int r = 0; r < 4; r++) {
            const bool keep_max = (low == (((i0 + 32 * r) & k) == 0));
            if (keep_max == (o[lane][r] > v[lane][r])) v[lane][r] = o[lane][r];
          }
        }
      }
    }
    for (int lane = 0; lane < 32; lane++)
      for (int r = 0; r < 4; r++) { const int i = tile * SORT_TILE + 32 * r + lane; if (i < np) keys[i] = v[lane][r]; }
  }
}

// descending; keys[nc..np) read as 0.  A barrier per pass.
static void sort_keys(std::vector<u64> &keys, const int nc, const int np, long &barriers) {
  sort_tile_pass(keys, nc, np, 2, std::min(np, SORT_TILE)); barriers++;
  for (int k = 2 * SORT_TILE; k <= np; k <<= 1) {
    for (int j = k >> 1; j >= SORT_TILE; j >>= 1) {
      for (int i = 0; i < (np >> 1); i++) {
        const int a = ((i & ~(j - 1)) << 1) | (i & (j - 1)), b = a | j;
        sort_cx(keys[a], keys[b], (a & k) == 0);
      }
      barriers++;
    }
    sort_tile_pass(keys, np, np, k, k); barriers++;
  }
}

// ---- 2. the closed form, as heap_select_closed runs it --------------------------------------------------------------------
struct ClosedStats { long leaf_checks = 0, reinserts = 0, chunks = 0; };

static int key_pre(u64 key) { return 0xffff - (int)((key >> 16) & 0xffffu); }
static unsigned key_score(u64 key) { return (unsigned)(key >> 32); }

// the home pre-order positions of the window keys[base .. base + 32 RELOC_WINDOW); 0xffff past nc and for keys[skip]
static void reloc_window_load(const std::vector<u64> &keys, int nc, int base, int skip, int *pre) {
  for (int p = 0; p < 32 * RELOC_WINDOW; p++) {
    const int idx = base + p;
    pre[p] = (idx < nc && idx != skip) ? key_pre(keys[idx]) : 0xffff;
  }
}
// first position >= from of the window whose home position lies in [lo, hi): a ballot per chunk, the first hit decides
static int reloc_window_first(const int *pre, int lo, int hi, int from) {
  for (int c = 0; c < RELOC_WINDOW; c++) {
    unsigned b = 0u;
    for (int lane = 0; lane < 32; lane++) { const int p = 32 * c + lane; if (pre[p] >= lo && pre[p] < hi && p >= from) b |= 1u << lane; }
    if (b) return 32 * c + __builtin_ffs(b) - 1;
  }
  return -1;
}

// closed_relocate, one warp emulated lane by lane: the same windows, ballots and shifts.  Returns 0 where the kernel does.
static int closed_relocate(std::vector<u64> &keys, const int nc, const int n, const int need, std::vector<unsigned> &flags,
                           std::vector<unsigned> &multi, std::vector<unsigned> &pay, ClosedStats &st) {
  const int H = depth(n);
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  for (int w = fwords - 1; w >= 0; w--) {
    unsigned bits = flags[w];
    while (bits) {
      const int b = 31 - __builtin_clz(bits);
      const int m = tail0 + w * 32 + b;
      const int k = n - m + 1;                               // step; this step's root is keys[k-1]
      if (m <= n && m >= 2 && k <= need) {
        const int dm = depth(m);
        const bool is_multi = (multi[(m - tail0) >> 5] >> ((m - tail0) & 31)) & 1u;
        // --- the occupant of leaf m
        int j = 0, a = 1, lo = 0, hi = n, occ = -1;
        bool gone = false;
        st.leaf_checks++;
        for (int base = k - 1; base < nc && occ < 0 && !gone; base += 32 * RELOC_WINDOW) {
          int pre[32 * RELOC_WINDOW];
          reloc_window_load(keys, nc, base, -1, pre);
          st.chunks += std::min(RELOC_WINDOW, (nc - base + 31) / 32);
          int from = 0;
          while (true) {
            const int f = reloc_window_first(pre, lo, hi, from);
            if (f < 0) break;
            if (j == dm) { occ = base + f; break; }
            if (!is_multi && (int)(pay[(unsigned)keys[base + f] & 0xffffu] >> 16) == m) { gone = true; break; }
            j++;
            const int nxt = m >> (dm - j);
            const int lsz = subtree_size(2 * a, n, H);
            if (nxt == 2 * a) { lo = lo + 1; hi = lo + lsz; } else { lo = lo + 1 + lsz; }
            a = nxt;
            from = f + 1;
          }
        }
        if (occ >= k) {
          // --- e = keys[occ] is re-inserted from the root of the heap of m-1 slots
          st.reinserts++;
          const u64 ekey = keys[occ];
          const unsigned esc = key_score(ekey);
          const int msz = m - 1;
          int x = 1; lo = 0; hi = n;
          bool stop = (2 * x > msz);
          for (int base = k; base < nc && !stop; base += 32 * RELOC_WINDOW) {
            int pre[32 * RELOC_WINDOW];
            reloc_window_load(keys, nc, base, occ, pre);
            st.chunks += std::min(RELOC_WINDOW, (nc - base + 31) / 32);
            int from = 0;
            while (!stop) {
              const int f = reloc_window_first(pre, lo, hi, from);
              if (f < 0) break;
              const u64 fk = keys[base + f];
              const int opre = key_pre(fk);
              if (opre == lo) return 0;
              if (esc >= key_score(fk)) { stop = true; break; }
              const int lsz = subtree_size(2 * x, n, H);
              if (opre < lo + 1 + lsz) { x = 2 * x; lo = lo + 1; hi = lo + lsz; }
              else { x = 2 * x + 1; lo = lo + 1 + lsz; }
              if (2 * x > msz) { stop = true; break; }
              from = f + 1;
            }
          }
          // --- e's home is x: new key, new place inside its tie group
          const u64 nkey = (ekey & 0xffffffff0000ffffull) | ((u64)(0xffffu - (unsigned)lo) << 16);
          int cnt = 0;
          const int wb = std::max(k, occ - 16), we = wb + 31;
          const bool lo_ok = (wb == k) || (key_score(keys[wb]) > esc);
          const bool hi_ok = (we >= nc) || (key_score(keys[we]) < esc);
          if (lo_ok && hi_ok) {
            cnt = wb - k;
            for (int lane = 0; lane < 32; lane++) { const int idx = wb + lane; if (idx < nc && idx != occ && keys[idx] > nkey) cnt++; }
          } else {
            for (int base = k; base < nc; base += 32) {
              bool any_le = false;
              for (int lane = 0; lane < 32; lane++) {
                const int idx = base + lane;
                const bool gt = (idx < nc) && idx != occ && keys[idx] > nkey;
                if (gt) cnt++;
                if ((idx < nc) && idx != occ && !gt) any_le = true;
              }
              if (any_le) break;
            }
          }
          const int ins = k + cnt;
          if (ins < occ) {
            for (int top = occ; top > ins; top -= 32) {
              u64 v[32];
              for (int lane = 0; lane < 32; lane++) { const int idx = top - lane; v[lane] = (idx > ins) ? keys[idx - 1] : 0ull; }
              for (int lane = 0; lane < 32; lane++) { const int idx = top - lane; if (idx > ins) keys[idx] = v[lane]; }
            }
          } else if (ins > occ) {
            for (int bot = occ; bot < ins; bot += 32) {
              u64 v[32];
              for (int lane = 0; lane < 32; lane++) { const int idx = bot + lane; v[lane] = (idx < ins) ? keys[idx + 1] : 0ull; }
              for (int lane = 0; lane < 32; lane++) { const int idx = bot + lane; if (idx < ins) keys[idx] = v[lane]; }
            }
          }
          keys[ins] = nkey;
          unsigned &pp = pay[(unsigned)nkey & 0xffffu];
          pp = ((unsigned)x << 16) | (pp & 0xffffu);
          if (x >= tail0 && x < m) { flags[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); multi[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); }
        }
      }
      bits = flags[w] & ((b == 0) ? 0u : ((1u << b) - 1u));
    }
  }
  return 1;
}

// H0: the built max-heap.  Returns the kernel's outcome, 0 = replay, 1 = closed form, 2 = closed form with relocations,
// and out[k] = k-th extracted token for 1 and 2; plain[k] the same from the sort alone.  The sort and payload areas are
// taken to hold every candidate set (a select whose candidates overflow them is replayed: a matter of their sizes).
static int closed_select(const std::vector<Ent> &H0, int n, int need, float lose_below, std::vector<int> &out,
                         std::vector<int> &plain, ClosedStats &st) {
  if (n >= 65536 || !(lose_below > -INFINITY)) return 0;
  const int H = depth(n);
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  // 1. candidates, packed keys and payload
  std::vector<u64> keys;
  std::vector<unsigned> pay;
  for (int h = 1; h <= n; h++) if (H0[h].v >= lose_below) {
    const unsigned ci = (unsigned)keys.size();
    keys.push_back(((u64)fkey(H0[h].v) << 32) | ((u64)(0xffffu - (unsigned)preorder(h, n, H)) << 16) | ci);
    pay.push_back(((unsigned)h << 16) | (unsigned)H0[h].id);
  }
  const int nc = (int)keys.size();
  int np = 1; while (np < nc) np <<= 1;
  if (nc > 65535 || nc < need) return 0;
  // 2. sort
  keys.resize(np);
  long barriers = 0;
  sort_keys(keys, nc, np, barriers);
  plain.resize(need);
  for (int k = 0; k < need; k++) plain[k] = (int)(pay[(unsigned)keys[k] & 0xffffu] & 0xffffu);
  // 3. the test: flag the tail candidates that may still be in their leaf when it is taken
  std::vector<unsigned> flags(fwords, 0u), multi(fwords, 0u);
  bool need_reloc = false;
  const unsigned theta = key_score(keys[need - 1]);
  for (int i = 0; i < nc; i++) {
    const unsigned sk = key_score(keys[i]);
    if (sk < theta) continue;
    const int slot = (int)(pay[(unsigned)keys[i] & 0xffffu] >> 16);
    if (slot < tail0) continue;
    const bool tied = (i > 0 && key_score(keys[i - 1]) == sk) || (i + 1 < nc && key_score(keys[i + 1]) == sk);
    int last = i;
    if (tied) {
      int g = 0;
      while (last + 1 < nc && key_score(keys[last + 1]) == sk && g < TIE_LOOKAHEAD) { last++; g++; }
      if (g == TIE_LOOKAHEAD) last = nc;
    }
    if (last + 1 < n - slot + 1 + depth(slot)) continue;
    flags[(slot - tail0) >> 5] |= 1u << ((slot - tail0) & 31);
    if (tied) need_reloc = true;
  }
  int relocated = 0;
  if (need_reloc) {
    if (!closed_relocate(keys, nc, n, need, flags, multi, pay, st)) return 0;
    relocated = 1;
  }
  // 4. survivors
  out.resize(need);
  for (int k = 0; k < need; k++) out[k] = (int)(pay[(unsigned)keys[k] & 0xffffu] & 0xffffu);
  return 1 + relocated;
}

// ---- 4. the invariant (I), readable ----------------------------------------------------------------------------------------
// While every extraction's s is a loser the heap evolves by pull-ups, and
//   (I)  slot x holds the best remaining element of subtree(x) that no ancestor of x holds,
// "best" = (score descending, pre-order position of the element's HOME slot ascending), which is the extraction order.
// A tail slot that still holds a candidate when it is taken breaks the pull-ups: the element is re-inserted from the root.
// (I) survives if its home moves to where it lands.  Here: the candidates in that order, and at each step whose tail slot
// is the home of a live candidate, (I) evaluated down the path to the slot, and a re-insertion replayed on the implicit
// heap with two "best remaining element of a subtree" queries a level.
struct Cand { float v; int pre; int id; int home; };
struct Invariant {
  int n, H;
  std::vector<Cand> c;
  std::vector<int> R;        // the order: indices into c; the live part is R[first_alive..]
  // best live candidate of subtree(x) that is not in excl; -1 = none (the slot holds a loser)
  int best(int x, int first_alive, const std::vector<int> &excl) const {
    if (x > n) return -1;
    const int lo = preorder(x, n, H), hi = lo + subtree_size(x, n, H);
    for (size_t r = first_alive; r < R.size(); r++) {
      const int i = R[r];
      if (c[i].pre >= lo && c[i].pre < hi && std::find(excl.begin(), excl.end(), i) == excl.end()) return i;
    }
    return -1;
  }
};
static void invariant_select(const std::vector<Ent> &H0, int n, int need, float lose_below, std::vector<int> &out) {
  Invariant d{n, depth(n), {}, {}};
  for (int h = 1; h <= n; h++) if (H0[h].v >= lose_below) d.c.push_back(Cand{H0[h].v, preorder(h, n, d.H), H0[h].id, h});
  const int nc = (int)d.c.size();
  auto before = [&](int a, int b) { return d.c[a].v != d.c[b].v ? d.c[a].v > d.c[b].v : d.c[a].pre < d.c[b].pre; };
  for (int i = 0; i < nc; i++) d.R.push_back(i);
  std::sort(d.R.begin(), d.R.end(), before);
  out.clear();
  for (int k = 1; k <= need && k <= nc; k++) {
    const int m = n - k + 1;                       // the slot this step takes its s from
    const int root_elem = d.R[k - 1];
    out.push_back(d.c[root_elem].id);
    if (m <= 1) break;
    bool home = false;
    for (size_t r = k - 1; r < d.R.size(); r++) home |= (d.c[d.R[r]].home == m);
    if (!home) continue;
    // (I) down the path root .. m
    std::vector<int> excl;
    int occ = -1;
    for (int j = 0; j <= depth(m); j++) {
      occ = d.best(m >> (depth(m) - j), k - 1, excl);
      if (occ < 0) break;                          // a loser up here: everything below is a loser too
      excl.push_back(occ);
    }
    if (occ < 0 || occ == root_elem) continue;     // slot m holds a loser
    // e = occ is taken from leaf m and re-inserted from the root of the heap of m-1 slots
    const int e = occ, msz = m - 1;
    std::vector<int> path{root_elem, e};
    int x = 1;
    while (2 * x <= msz) {
      const int o1 = d.best(2 * x, k - 1, path);
      const int o2 = (2 * x + 1 <= msz) ? d.best(2 * x + 1, k - 1, path) : -1;
      if (o1 < 0 && o2 < 0) break;                 // both children are losers
      const bool right = o1 < 0 || (o2 >= 0 && d.c[o1].v < d.c[o2].v);
      const int oc = right ? o2 : o1;
      if (d.c[e].v >= d.c[oc].v) break;            // "STVAL >= SVAL(child)"
      path.push_back(oc);
      x = 2 * x + (right ? 1 : 0);
    }
    // e's home moves to x, and its place in the order with it (behind this step's root)
    d.c[e].home = x; d.c[e].pre = preorder(x, n, d.H);
    d.R.erase(std::find(d.R.begin(), d.R.end(), e));
    int ins = k;
    while (ins < (int)d.R.size() && before(d.R[ins], e)) ins++;
    d.R.insert(d.R.begin() + ins, e);
  }
}

// ---- drivers -----------------------------------------------------------------------------------------------------------------
struct Tally {
  long up = 0, down = 0, outcome[3] = {0, 0, 0}, plain_right = 0, with_reinserts = 0;
  long bad_replay = 0, bad_closed = 0, bad_invariant = 0;
  ReplayStats rup, rdown;
  ClosedStats cs;
  long mismatches() const { return bad_replay + bad_closed + bad_invariant; }
};

static bool same_ids(const std::vector<int> &got, const std::vector<Ent> &R, int n, int need) {
  for (int k = 0; k < need; k++) if (got[k] != R[n - k].id) return false;
  return true;
}

// one select of the scores base[1..n] through every model that applies.  P: the kernel's heap area, maxt + 4 slots;
// what lies above slot n must not matter, so it holds tokens that would win every comparison.
static void one_select(const std::vector<Ent> &base, int n, int need, float lose_below, int maxt, Tally &t) {
  const bool upward = need < n - need;
  const int extract = upward ? need : n - need;
  std::vector<Ent> R = base, P(maxt + 4, Ent{-2, upward ? INFINITY : -INFINITY}), outs;
  std::copy(base.begin() + 1, base.begin() + n + 1, P.begin() + 1);
  if (!upward) {
    t.down++;
    reference_select<false>(R, n, extract);
    replay<false>(P, n, extract, maxt, -INFINITY, outs, t.rdown);
    for (int k = 0; k < extract; k++) P[n - k] = outs[k];
    for (int i = 1; i <= n; i++) if (P[i].id != R[i].id) { t.bad_replay++; break; }
    return;
  }
  t.up++;
  reference_select<true>(R, n, extract);
  // the replay with the loser cut: the extraction order
  std::vector<Ent> P2 = P;
  replay<true>(P, n, extract, maxt, lose_below, outs, t.rup);
  for (int k = 0; k < extract; k++) if (outs[k].id != R[n - k].id) { t.bad_replay++; break; }
  // without the cut (multipath select #1, select_exact): the whole array, the extracted roots back in the tail
  ReplayStats unused;
  replay<true>(P2, n, extract, maxt, -INFINITY, outs, unused);
  for (int k = 0; k < extract; k++) P2[n - k] = outs[k];
  for (int i = 1; i <= n; i++) if (P2[i].id != R[i].id) { t.bad_replay++; break; }
  // the closed form answers every select (0 = the relocation pass gave up)
  std::vector<Ent> H0 = base;
  heap_build<true>(H0, n);
  std::vector<int> got, plain;
  const long reinserts = t.cs.reinserts;
  const int outcome = closed_select(H0, n, need, lose_below, got, plain, t.cs);
  t.outcome[outcome]++;
  if (!outcome || !same_ids(got, R, n, need)) t.bad_closed++;
  if (outcome && same_ids(plain, R, n, need)) t.plain_right++;
  if (t.cs.reinserts > reinserts) t.with_reinserts++;
  invariant_select(H0, n, need, lose_below, got);
  if ((int)got.size() != need || !same_ids(got, R, n, need)) t.bad_invariant++;
}

static void print_mismatches(const Tally &t) {
  printf("mismatches %ld (replay %ld, closed form %ld, invariant %ld)\n", t.mismatches(), t.bad_replay, t.bad_closed, t.bad_invariant);
}

// random heaps: n up to 2600, upward and downward selects, lose_below the need-th score less 0, 0.5 or 1.0
static int random_mode(int distinct, int trials) {
  srand(1);
  Tally t;
  for (int tr = 0; tr < trials; tr++) {
    const int n = 3 + rand() % 2600, need = 1 + rand() % (n - 1);
    const int maxt = ((std::max(n, 64) + 63 + rand() % 500) + 3) & ~3;
    std::vector<Ent> base(n + 1, Ent{0, 0.0f});
    std::vector<float> scores;
    for (int i = 1; i <= n; i++) { base[i] = Ent{i - 1, -(float)(rand() % distinct) / 7.0f}; scores.push_back(base[i].v); }
    std::sort(scores.begin(), scores.end(), std::greater<float>());
    const float lose_below = scores[need - 1] - (float)(rand() % 3) * 0.5f;
    one_select(base, n, need, lose_below, maxt, t);
  }
  printf("selects: upward %ld, downward %ld; relocation pass in %ld, re-insertions %ld\n", t.up, t.down, t.outcome[2], t.cs.reinserts);
  print_mismatches(t);
  return t.mismatches() != 0;
}

// the cuts of a real decode; lose_below = the need-th score less 0.25 stands in for the histogram's bound.  The shares
// are those of bench.py's cut counters: closed / upward and relocated / upward.
static int dump_mode(const char *path) {
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); return 2; }
  Tally t;
  int hdr[2];
  while (fread(hdr, 4, 2, f) == 2) {
    const int n = hdr[0], need = hdr[1];
    std::vector<Ent> A(n + 1, Ent{0, 0.0f});
    for (int i = 1; i <= n; i++) { A[i].id = i - 1; if (fread(&A[i].v, 4, 1, f) != 1) { fclose(f); return 2; } }
    std::vector<float> sc;
    for (int i = 1; i <= n; i++) sc.push_back(A[i].v);
    std::sort(sc.begin(), sc.end(), std::greater<float>());
    one_select(A, n, need, sc[need - 1] - 0.25f, (n + 64 + 3) & ~3, t);
  }
  fclose(f);
  const double up = std::max(1L, t.up), down = std::max(1L, t.down);
  printf("selects: upward %ld, downward %ld\n", t.up, t.down);
  printf("replay: %.0f ticks and %.1f held-back starts per upward select, %.0f ticks and %.1f held-back starts per downward select\n",
         t.rup.ticks / up, t.rup.held / up, t.rdown.ticks / down, t.rdown.held / down);
  printf("closed form: %.1f %% of the upward selects, relocated %.1f %%; the sort alone right in %.1f %%, re-insertions in %.1f %%\n",
         100.0 * (t.outcome[1] + t.outcome[2]) / up, 100.0 * t.outcome[2] / up, 100.0 * t.plain_right / up, 100.0 * t.with_reinserts / up);
  printf("per cut: %.1f leaf checks, %.1f re-insertions, %.1f 32-key chunk reads\n", t.cs.leaf_checks / up, t.cs.reinserts / up, t.cs.chunks / up);
  print_mismatches(t);
  return t.mismatches() != 0;
}

// every power of two np from 2 to 2^max_log2, with nc = np, np/2 + 1 (the fewest candidates that need this np) and in
// between; random distinct non-zero keys, as the kernel's are (candidate index in the low 16 bits)
static int sort_mode(int max_log2) {
  std::mt19937_64 rng(1);
  long bad = 0, ran = 0;
  for (int np = 2; np <= (1 << max_log2); np <<= 1) {
    long barriers = 0;
    for (int tr = 0; tr < 12; tr++) {
      const int nc = (tr % 3 == 0) ? np : (tr % 3 == 1) ? np / 2 + 1 : np / 2 + 1 + (int)(rng() % (np / 2));
      std::vector<u64> keys(np), want;
      for (int i = 0; i < np; i++) keys[i] = ((rng() | 1ull) << 16) | (u64)i;
      want.assign(keys.begin(), keys.begin() + nc);
      std::sort(want.begin(), want.end(), std::greater<u64>());
      want.resize(np, 0ull);
      barriers = 0;
      sort_keys(keys, nc, np, barriers);
      ran++;
      if (keys != want && bad++ < 5) printf("  mismatch: np %d nc %d\n", np, nc);
    }
    printf("np %5d: %ld barriers (a barrier per stage: %d)\n", np, barriers, __builtin_ctz(np) * (__builtin_ctz(np) + 1) / 2);
  }
  printf("sorts %ld, mismatches %ld\n", ran, bad);
  return bad != 0;
}

int main(int argc, char **argv) {
  const std::string mode = argc > 1 ? argv[1] : "";
  if (mode == "random" && argc > 3) return random_mode(atoi(argv[2]), atoi(argv[3]));
  if (mode == "--dump" && argc > 2) return dump_mode(argv[2]);
  if (mode == "sort" && argc > 2) return sort_mode(atoi(argv[2]));
  fprintf(stderr, "usage: beamcut random <distinct scores> <trials> | --dump <file> | sort <max log2>\n");
  return 2;
}
