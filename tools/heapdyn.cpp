// tools/heapdyn.cpp -- CPU model of the "closed form with relocations" for the upward beam cut, checked against the
// reference's loop (sort_token_upward, libjulius/src/beam.c:1342-1384).
//
//   g++ -O2 -o /tmp/heapdyn tools/heapdyn.cpp && /tmp/heapdyn [score divisor] [trials] [distinct scores]
//   /tmp/heapdyn --dump <file written by tools/dump_heaps.py>
//
// Idea.  While every extraction's s (the tail slot's content) is a loser, the heap evolves by pure pull-ups and
//   (I)  the slot x holds the best remaining element of subtree(x) that is not held by an ancestor of x,
// "best" = (score descending, pre-order position of the element's HOME slot ascending), and the extraction order is that
// order (tools/heapsim.cpp, closed_form_select).  A tail slot whose content is a candidate that is still there when the
// slot is taken breaks this: the element is re-inserted from the root and lands on the chain of larger children where its
// score says -- above everything it ties with.  But (I) survives if the element's home is moved to where it lands: it is
// at least as good as both sub-trees below it, so it IS the best remaining element of that subtree.  So: keep the
// candidates sorted, walk the steps, and at the few steps whose tail slot still holds a candidate (decided by evaluating
// (I) down the path to that leaf) replay that one re-insertion on the implicit heap (another walk down, two "best
// remaining element of a subtree" queries a level), move the element's home and its place in the order.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

struct Ent { int id; float v; };

static void sift_down(std::vector<Ent> &A, int start, int n) {
  Ent s = A[start];
  int parent = start, child;
  while ((child = parent * 2) <= n) {
    if (child < n && A[child].v < A[child + 1].v) child++;
    if (s.v >= A[child].v) break;
    A[parent] = A[child];
    parent = child;
  }
  A[parent] = s;
}
static void heap_build(std::vector<Ent> &A, int n) { for (int root = n / 2; root >= 1; root--) sift_down(A, root, n); }
// reference extraction on a built heap: out[k] = k-th extracted id
static void reference_extract(std::vector<Ent> A, int n, int need, std::vector<int> &out) {
  out.clear();
  int m = n;
  while (m > n - need) {
    Ent s = A[m];
    out.push_back(A[1].id);
    A[m] = A[1];
    m--;
    if (m < 1) break;
    A[1] = s;
    sift_down(A, 1, m);
  }
}

static int subtree_size(int c, int n) {
  if (c > n) return 0;
  int H = 31 - __builtin_clz(n), dc = 31 - __builtin_clz(c);
  if (dc > H) return 0;
  const int full = (1 << (H - dc)) - 1;
  const long first = (long)c << (H - dc), width = 1L << (H - dc);
  long last_cnt = (long)n - first + 1; if (last_cnt < 0) last_cnt = 0; if (last_cnt > width) last_cnt = width;
  return full + (int)last_cnt;
}
static int preorder(int h, int n) {
  int pre = 0, cur = 1;
  const int d = 31 - __builtin_clz(h);
  for (int b = d - 1; b >= 0; b--) {
    const int bit = (h >> b) & 1;
    pre += 1;
    if (bit) pre += subtree_size(cur * 2, n);
    cur = cur * 2 + bit;
  }
  return pre;
}

struct Cand { float v; int pre; int id; int home; };
static long g_events = 0, g_checks = 0, g_frames = 0, g_levels = 0;

// order R: indices into c, sorted by (v desc, pre asc); alive = position >= first_alive
struct Dyn {
  int n;
  std::vector<Cand> c;
  std::vector<int> R;        // current order
  std::vector<int> posR;     // inverse
  // best alive candidate of subtree(x) that is not in `excl`; -1 = none (the slot holds a loser)
  int best(int x, int first_alive, const std::vector<int> &excl) const {
    if (x > n) return -1;
    const int lo = preorder(x, n), hi = lo + subtree_size(x, n);
    for (size_t r = first_alive; r < R.size(); r++) {
      const int i = R[r];
      if (c[i].pre < lo || c[i].pre >= hi) continue;
      bool ex = false;
      for (int e : excl) if (e == i) { ex = true; break; }
      if (!ex) return i;
    }
    return -1;
  }
};

// returns false when it gives up (never, in this model); out[k] = id of the k-th extracted
static bool closed_dynamic(const std::vector<Ent> &H0, int n, int need, float lose_below, std::vector<int> &out) {
  Dyn d; d.n = n;
  for (int h = 1; h <= n; h++) if (H0[h].v >= lose_below) d.c.push_back(Cand{H0[h].v, preorder(h, n), H0[h].id, h});
  const int nc = (int)d.c.size();
  if (nc < need) return false;
  d.R.resize(nc);
  for (int i = 0; i < nc; i++) d.R[i] = i;
  std::sort(d.R.begin(), d.R.end(), [&](int a, int b) { return d.c[a].v != d.c[b].v ? d.c[a].v > d.c[b].v : d.c[a].pre < d.c[b].pre; });
  // candidates by home slot (a slot can be the home of several after relocations)
  std::vector<std::vector<int>> at_home(n + 2);
  for (int i = 0; i < nc; i++) at_home[d.c[i].home].push_back(i);
  d.posR.assign(nc, 0);
  for (int r = 0; r < nc; r++) d.posR[d.R[r]] = r;
  out.clear();
  g_frames++;
  for (int k = 1; k <= need; k++) {
    const int m = n - k + 1;                       // the slot this step takes its s from
    const int root_elem = d.R[k - 1];
    out.push_back(d.c[root_elem].id);
    if (m <= 1) break;
    // does slot m hold a candidate?  only if some alive candidate has its home there
    bool any = false;
    for (int i : at_home[m]) if (d.posR[i] >= k - 1) any = true;
    if (!any) continue;
    g_checks++;
    // (I) down the path root .. m
    std::vector<int> excl;
    int occ = -1;
    const int dm = 31 - __builtin_clz(m);
    for (int j = 0; j <= dm; j++) {
      const int a = m >> (dm - j);
      occ = d.best(a, k - 1, excl);
      g_levels++;
      if (occ < 0) break;                          // a loser up here: everything below is a loser too
      excl.push_back(occ);
    }
    if (occ < 0) continue;                         // slot m holds a loser
    if (occ == root_elem) continue;                // (m == 1 only)
    // EVENT: candidate e = occ is taken from leaf m and re-inserted from the root of the heap of m-1 slots
    g_events++;
    const int e = occ;
    const int msz = m - 1;
    std::vector<int> path_excl; path_excl.push_back(root_elem); path_excl.push_back(e);
    int x = 1;
    while (true) {
      const int c1 = 2 * x, c2 = 2 * x + 1;
      if (c1 > msz) break;
      const int o1 = d.best(c1, k - 1, path_excl);
      const int o2 = (c2 <= msz) ? d.best(c2, k - 1, path_excl) : -1;
      g_levels += 2;
      int child, oc;
      if (o1 < 0 && o2 < 0) break;                 // both children are losers: e stays above them
      if (o1 < 0) { child = c2; oc = o2; }
      else if (o2 < 0) { child = c1; oc = o1; }
      else if (d.c[o1].v < d.c[o2].v) { child = c2; oc = o2; }
      else { child = c1; oc = o1; }
      if (d.c[e].v >= d.c[oc].v) break;            // "STVAL >= SVAL(child)"
      path_excl.push_back(oc);
      x = child;
    }
    // e's home moves to x; its place in the order moves accordingly (among the alive part after this step's root)
    {
      auto &lst = at_home[d.c[e].home];
      lst.erase(std::find(lst.begin(), lst.end(), e));
      d.c[e].home = x; d.c[e].pre = preorder(x, n);
      at_home[x].push_back(e);
      const int old = d.posR[e];
      d.R.erase(d.R.begin() + old);
      int ins = k;                                  // first position after the element extracted in this step
      while (ins < (int)d.R.size()) {
        const Cand &q = d.c[d.R[ins]];
        const bool before = (q.v != d.c[e].v) ? (q.v > d.c[e].v) : (q.pre < d.c[e].pre);
        if (!before) break;
        ins++;
      }
      d.R.insert(d.R.begin() + ins, e);
      for (int r = std::min(old, ins); r <= std::max(old, ins) && r < (int)d.R.size(); r++) d.posR[d.R[r]] = r;
    }
  }
  return true;
}


// ---- the same, in the form the kernel runs it ---------------------------------------------------------------------
// One sorted key array (score desc, home pre-order position asc); everything is a forward scan over it:
//   * which element sits in leaf m at step k: assign the levels of the path root..m top-down while walking the alive part
//     of the order -- level j goes to the first element not yet used whose home lies in subtree(a_j) (nested intervals of
//     pre-order positions), and m holds a candidate iff level depth(m) gets one;
//   * where a re-inserted element e lands: walk the order behind the root; the first element of subtree(x) is the occupant
//     of one of x's children (the larger one, the left one on a tie: that IS the order); e stays at x if its score is >=
//     that element's, else the hole moves into the child whose subtree holds that element's home.
struct Key { float v; int pre; int id; };
static bool key_before(const Key &a, const Key &b) { return a.v != b.v ? a.v > b.v : a.pre < b.pre; }
static long g2_scan_elems = 0;
static bool closed_dynamic_scan(const std::vector<Ent> &H0, int n, int need, float lose_below, std::vector<int> &out) {
  std::vector<Key> K;
  std::vector<char> flagged(n + 2, 0);                       // tail slots that are the home of a candidate
  for (int h = 1; h <= n; h++) if (H0[h].v >= lose_below) {
    K.push_back(Key{H0[h].v, preorder(h, n), H0[h].id});
    if (h >= n - need + 1) flagged[h] = 1;
  }
  const int nc = (int)K.size();
  if (nc < need) return false;
  std::stable_sort(K.begin(), K.end(), key_before);
  for (int m = n; m >= n - need + 1 && m >= 2; m--) {
    if (!flagged[m]) continue;
    const int k = n - m + 1;                                 // step (1-based); the root at this step is K[k-1]
    // --- occupant of leaf m
    const int dm = 31 - __builtin_clz(m);
    int j = 0, a = 1, lo = 0, hi = n;                        // level, its path node, interval of pre-order positions
    int occ = -1;
    for (int idx = k - 1; idx < nc; idx++) {
      g2_scan_elems++;
      if (K[idx].pre < lo || K[idx].pre >= hi) continue;
      if (j == dm) { occ = idx; break; }
      // level j is taken; next level: the child of a on the way to m
      j++;
      const int nxt = m >> (dm - j);
      const int lsz = subtree_size(2 * a, n);
      if (nxt == 2 * a) { lo = lo + 1; hi = lo + lsz; } else { lo = lo + 1 + lsz; /* hi unchanged */ }
      a = nxt;
    }
    if (occ < 0 || occ == k - 1) continue;                   // a loser (or m is the root)
    // --- re-insertion of e = K[occ] from the root of the heap of m-1 slots
    const Key e = K[occ];
    const int msz = m - 1;
    int x = 1; lo = 0; hi = n;
    for (int idx = k; idx < nc; idx++) {
      if (2 * x > msz) break;                                // x has no children left
      if (idx == occ) continue;
      g2_scan_elems++;
      if (K[idx].pre < lo || K[idx].pre >= hi) continue;
      if (K[idx].pre == lo) return false;                    // (cannot happen: an unplaced element whose home is x)
      if (e.v >= K[idx].v) break;                            // "STVAL >= SVAL(child)": e stays at x
      const int lsz = subtree_size(2 * x, n);
      if (K[idx].pre < lo + 1 + lsz) { x = 2 * x; lo = lo + 1; hi = lo + lsz; }
      else { x = 2 * x + 1; lo = lo + 1 + lsz; }
    }
    // --- e's home is x now
    Key ne = e; ne.pre = lo;
    K.erase(K.begin() + occ);
    int ins = k;
    while (ins < (int)K.size() && key_before(K[ins], ne)) ins++;
    K.insert(K.begin() + ins, ne);
    if (x >= n - need + 1 && x < m) flagged[x] = 1;
  }
  out.resize(need);
  for (int k = 0; k < need; k++) out[k] = K[k].id;
  return true;
}

// ---- lane-by-lane emulation of closed_relocate (csrc/beam.cu): the same windows, ballots and shifts -----------------------
typedef unsigned long long u64;
static unsigned fkey_of(float f) { unsigned b; memcpy(&b, &f, 4); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
static int emu_subtree_size(int c, int n, int H) {
  const int dc = 31 - __builtin_clz(c);
  if (dc > H) return 0;
  const int sh = H - dc;
  const int first = c << sh, width = 1 << sh;
  return (width - 1) + std::max(0, std::min(n - first + 1, width));
}
// the scans read the order in windows of EMU_WINDOW chunks of 32 keys (RELOC_WINDOW in beam.cu): lane l of chunk c
// holds position 32c + l; a ballot per chunk, the first chunk with a match decides
constexpr int EMU_WINDOW = 3;
static void emu_window_load(const std::vector<u64> &keys, const int nc, const int base, const int skip, int *pre) {
  for (int p = 0; p < 32 * EMU_WINDOW; p++) {
    const int idx = base + p;
    pre[p] = (idx < nc && idx != skip) ? 0xffff - (int)((keys[idx] >> 16) & 0xffffu) : -1;
  }
}
static int emu_window_first(const int *pre, const int lo, const int hi, const int from) {
  for (int c = 0; c < EMU_WINDOW; c++) {
    unsigned b = 0u;
    for (int lane = 0; lane < 32; lane++) { const int p = 32 * c + lane; if (pre[p] >= lo && pre[p] < hi && p >= from) b |= 1u << lane; }
    if (b) return 32 * c + __builtin_ffs(b) - 1;
  }
  return -1;
}
static long g3_chunks = 0, g3_checks = 0, g3_events = 0, g3_frames = 0, g3_ch_occ_event = 0, g3_ch_occ_gone = 0, g3_ch_occ_none = 0, g3_n_gone = 0, g3_n_none = 0, g3_ch_chain = 0, g3_ch_cnt = 0;
static int emu_relocate(std::vector<u64> &keys, const int nc, const int n, const int need, std::vector<unsigned> &flags, std::vector<unsigned> &multi, std::vector<unsigned> &pay) {
  const int H = 31 - __builtin_clz(n);
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  for (int w = fwords - 1; w >= 0; w--) {
    unsigned bits = flags[w];
    while (bits) {
      const int b = 31 - __builtin_clz(bits);
      const int m = tail0 + w * 32 + b;
      const int k = n - m + 1;
      if (m <= n && m >= 2 && k <= need) {
        const int dm = 31 - __builtin_clz(m);
        const bool is_multi = (multi[(m - tail0) >> 5] >> ((m - tail0) & 31)) & 1u;
        int j = 0, a = 1, lo = 0, hi = n, occ = -1;
        bool gone = false;
        g3_checks++;
        const long c0 = g3_chunks;
        for (int base = k - 1; base < nc && occ < 0 && !gone; base += 32 * EMU_WINDOW) {
          int pre[32 * EMU_WINDOW];
          emu_window_load(keys, nc, base, -1, pre);
          int from = 0;
          g3_chunks += std::min(EMU_WINDOW, (nc - base + 31) / 32);     // chunks that hold keys
          while (true) {
            const int f = emu_window_first(pre, lo, hi, from);
            if (f < 0) break;
            if (j == dm) { occ = base + f; break; }
            // the leaf's own candidate, pulled up to level j: nothing but a loser can be in the leaf (unless a re-inserted
            // element landed there too)
            if (!is_multi && (int)(pay[(unsigned)keys[base + f] & 0xffffu] >> 16) == m) { gone = true; break; }
            j++;
            const int nxt = m >> (dm - j);
            const int lsz = emu_subtree_size(2 * a, n, H);
            if (nxt == 2 * a) { lo = lo + 1; hi = lo + lsz; } else { lo = lo + 1 + lsz; }
            a = nxt;
            from = f + 1;
          }
        }
        if (occ >= k) g3_ch_occ_event += g3_chunks - c0; else if (gone) { g3_ch_occ_gone += g3_chunks - c0; g3_n_gone++; } else { g3_ch_occ_none += g3_chunks - c0; g3_n_none++; }
        if (occ >= k) {
          const long c1 = g3_chunks;
          const u64 ekey = keys[occ];
          const unsigned esc = (unsigned)(ekey >> 32);
          g3_events++;
          const int msz = m - 1;
          int x = 1; lo = 0; hi = n;
          bool stop = (2 * x > msz);
          for (int base = k; base < nc && !stop; base += 32 * EMU_WINDOW) {
            int pre[32 * EMU_WINDOW];
            emu_window_load(keys, nc, base, occ, pre);
            int from = 0;
            g3_chunks += std::min(EMU_WINDOW, (nc - base + 31) / 32);     // chunks that hold keys
            while (!stop) {
              const int f = emu_window_first(pre, lo, hi, from);
              if (f < 0) break;
              const u64 fk = keys[base + f];
              const unsigned osc = (unsigned)(fk >> 32);
              const int opre = 0xffff - (int)((fk >> 16) & 0xffffu);
              if (opre == lo) return 0;
              if (esc >= osc) { stop = true; break; }
              const int lsz = emu_subtree_size(2 * x, n, H);
              if (opre < lo + 1 + lsz) { x = 2 * x; lo = lo + 1; hi = lo + lsz; }
              else { x = 2 * x + 1; lo = lo + 1 + lsz; }
              if (2 * x > msz) { stop = true; break; }
              from = f + 1;
            }
          }
          g3_ch_chain += g3_chunks - c1;
          const u64 nkey = (ekey & 0xffffffff0000ffffull) | ((u64)(0xffffu - (unsigned)lo) << 16);
          // the new place is inside e's tie group: one window around occ, unless the group is wider than that
          int cnt = 0;
          {
            const int wb = std::max(k, occ - 16);
            const bool lo_ok = (wb == k) || ((unsigned)(keys[wb] >> 32) > esc);
            const int we = wb + 31;
            const bool hi_ok = (we >= nc) || ((unsigned)(keys[we] >> 32) < esc);
            g3_ch_cnt++;
            if (lo_ok && hi_ok) {
              cnt = wb - k;
              for (int lane = 0; lane < 32; lane++) { const int idx = wb + lane; if (idx < nc && idx != occ && keys[idx] > nkey) cnt++; }
            } else {
              for (int base = k; base < nc; base += 32) {
                bool any_le = false;
                g3_ch_cnt++;
                for (int lane = 0; lane < 32; lane++) {
                  const int idx = base + lane;
                  const bool gt = (idx < nc) && idx != occ && keys[idx] > nkey;
                  if (gt) cnt++;
                  if ((idx < nc) && idx != occ && !gt) any_le = true;
                }
                if (any_le) break;
              }
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
          { unsigned &pp = pay[(unsigned)nkey & 0xffffu]; pp = ((unsigned)x << 16) | (pp & 0xffffu); }
          if (x >= tail0 && x < m) { flags[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); multi[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); }
        }
      }
      bits = flags[w] & ((b == 0) ? 0u : ((1u << b) - 1u));
    }
  }
  return 1;
}
// the kernel's heap_select_closed around it: collect, sort descending by the packed key, relocate, read the order off
static bool closed_emulated(const std::vector<Ent> &H0, int n, int need, float lose_below, std::vector<int> &out) {
  if (n >= 65536) return false;
  const int H = 31 - __builtin_clz(n);
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  std::vector<unsigned> flags(fwords, 0u), pay;
  std::vector<u64> keys;
  for (int h = 1; h <= n; h++) if (H0[h].v >= lose_below) {
    int pre = 0, cur = 1;
    for (int bb = (31 - __builtin_clz(h)) - 1; bb >= 0; bb--) { const int bit = (h >> bb) & 1; pre += 1 + (bit ? emu_subtree_size(cur * 2, n, H) : 0); cur = cur * 2 + bit; }
    const int ci = (int)keys.size();
    keys.push_back(((u64)fkey_of(H0[h].v) << 32) | ((u64)(0xffffu - (unsigned)pre) << 16) | (unsigned)ci);
    pay.push_back(((unsigned)h << 16) | (unsigned)H0[h].id);
  }
  const int nc = (int)keys.size();
  if (nc < need || nc > 65535) return false;
  std::sort(keys.begin(), keys.end(), std::greater<u64>());
  // which tail candidates may still be in their leaf when it is taken (the kernel's test loop)
  std::vector<unsigned> multi(fwords, 0u);
  bool need_reloc = false;
  const unsigned theta = (unsigned)(keys[need - 1] >> 32);
  for (int i = 0; i < nc; i++) {
    const unsigned sk = (unsigned)(keys[i] >> 32);
    if (sk < theta) continue;
    const int slot = (int)(pay[(unsigned)keys[i] & 0xffffu] >> 16);
    if (slot < tail0) continue;
    const int kstep = n - slot + 1, dd = 31 - __builtin_clz(slot);
    const bool tied = (i > 0 && (unsigned)(keys[i - 1] >> 32) == sk) || (i + 1 < nc && (unsigned)(keys[i + 1] >> 32) == sk);
    int last = i;                                   // last index of the tie group (bounded look-ahead; beyond it: assume the worst)
    if (tied) { int g = 0; while (last + 1 < nc && (unsigned)(keys[last + 1] >> 32) == sk && g < 8) { last++; g++; } if (g == 8) last = nc; }
    if (last + 1 < kstep + dd) continue;            // cannot be in its slot any more, wherever in its tie group it ends up
    flags[(slot - tail0) >> 5] |= 1u << ((slot - tail0) & 31);
    if (tied) need_reloc = true;
  }
  g3_frames++;
  if (need_reloc && !emu_relocate(keys, nc, n, need, flags, multi, pay)) return false;
  out.resize(need);
  for (int k = 0; k < need; k++) out[k] = (int)(pay[(unsigned)keys[k] & 0xffffu] & 0xffffu);
  return true;
}

static int run_one(std::vector<Ent> A, int n, int need, float lose_below, long &bad) {
  heap_build(A, n);
  std::vector<int> ref, dyn;
  reference_extract(A, n, need, ref);
  if (!closed_dynamic(A, n, need, lose_below, dyn)) return 0;
  for (int k = 0; k < need; k++) if (ref[k] != dyn[k]) { bad++; return -(k + 1); }
  std::vector<int> dyn2;
  if (!closed_dynamic_scan(A, n, need, lose_below, dyn2)) { bad++; return -1000000; }
  for (int k = 0; k < need; k++) if (ref[k] != dyn2[k]) { bad++; return -(k + 1) - 2000000; }
  std::vector<int> dyn3;
  if (!closed_emulated(A, n, need, lose_below, dyn3)) { bad++; return -3000000; }
  for (int k = 0; k < need; k++) if (ref[k] != dyn3[k]) { bad++; return -(k + 1) - 4000000; }
  return 1;
}

static int dump_mode(const char *path) {
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); return 2; }
  long nup = 0, bad = 0;
  int hdr[2];
  while (fread(hdr, 4, 2, f) == 2) {
    const int n = hdr[0], need = hdr[1];
    std::vector<Ent> A(n + 2, Ent{0, 0.0f});
    for (int i = 1; i <= n; i++) { A[i].id = i - 1; if (fread(&A[i].v, 4, 1, f) != 1) return 2; }
    if (!(need < n - need)) continue;
    nup++;
    std::vector<float> sc; for (int i = 1; i <= n; i++) sc.push_back(A[i].v);
    std::sort(sc.begin(), sc.end(), std::greater<float>());
    const float lose_below = sc[need - 1] - 0.25f;
    const int r = run_one(A, n, need, lose_below, bad);
    if (r < 0 && bad <= 5) printf("  mismatch: n %d need %d first at extraction %d\n", n, need, -r - 1);
  }
  printf("upward selects %ld: mismatches %ld; per select: %.1f leaf checks, %.1f re-insertions, %.1f subtree queries; scan form: %.0f elements visited\n", nup, bad,
         (double)g_checks / std::max(1L, g_frames), (double)g_events / std::max(1L, g_frames), (double)g_levels / std::max(1L, g_frames), (double)g2_scan_elems / std::max(1L, g_frames));
  printf("kernel form: %.1f leaf checks, %.1f re-insertions, %.1f 32-key chunks per select\n", (double)g3_checks / std::max(1L, g3_frames), (double)g3_events / std::max(1L, g3_frames), (double)g3_chunks / std::max(1L, g3_frames));
  printf("  chunks per select: occupant scans that end in an event %.1f, in 'pulled up' %.1f (%.1f scans), in 'nobody' %.1f (%.1f scans); chain walks %.1f; insert-position counts %.1f\n",
         (double)g3_ch_occ_event / g3_frames, (double)g3_ch_occ_gone / g3_frames, (double)g3_n_gone / g3_frames, (double)g3_ch_occ_none / g3_frames, (double)g3_n_none / g3_frames, (double)g3_ch_chain / g3_frames, (double)g3_ch_cnt / g3_frames);
  return bad != 0;
}

int main(int argc, char **argv) {
  if (argc > 2 && std::string(argv[1]) == "--dump") return dump_mode(argv[2]);
  const double divisor = argc > 1 ? atof(argv[1]) : 7.0;
  const int trials = argc > 2 ? atoi(argv[2]) : 3000;
  const int modulus = argc > 3 ? atoi(argv[3]) : 20000;
  srand(1);
  long bad = 0, ran = 0;
  for (int tr = 0; tr < trials; tr++) {
    const int nmax = getenv("HEAPDYN_NMAX") ? atoi(getenv("HEAPDYN_NMAX")) : 2600;
    const int n = 3 + rand() % nmax;
    int need = 1 + rand() % (n - 1);
    if (!(need < n - need)) need = std::max(1, (n - 1) / 2 - rand() % std::max(1, n / 4));
    if (!(need < n - need) || need < 1) continue;
    std::vector<Ent> A(n + 2, Ent{0, 0.0f});
    std::vector<float> sc;
    for (int i = 1; i <= n; i++) { A[i] = Ent{i - 1, -(float)(rand() % modulus) / (float)divisor}; sc.push_back(A[i].v); }
    std::sort(sc.begin(), sc.end(), std::greater<float>());
    const float lose_below = sc[need - 1] - (float)(rand() % 3) * 0.5f;
    ran++;
    const int r = run_one(A, n, need, lose_below, bad);
    if (r < 0 && bad <= 5) printf("  mismatch: trial %d n %d need %d first at extraction %d\n", tr, n, need, -r - 1);
  }
  printf("trials %ld, mismatches %ld; per select: %.1f leaf checks, %.1f re-insertions, %.1f subtree queries; scan form: %.0f elements visited\n", ran, bad,
         (double)g_checks / std::max(1L, g_frames), (double)g_events / std::max(1L, g_frames), (double)g_levels / std::max(1L, g_frames), (double)g2_scan_elems / std::max(1L, g_frames));
  printf("kernel form: %.1f leaf checks, %.1f re-insertions, %.1f 32-key chunks per select\n", (double)g3_checks / std::max(1L, g3_frames), (double)g3_events / std::max(1L, g3_frames), (double)g3_chunks / std::max(1L, g3_frames));
  return bad != 0;
}
