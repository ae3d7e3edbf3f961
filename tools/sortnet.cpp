// CPU model of the candidate sort of the closed-form beam cut (heap_select_closed step 2 in csrc/beam.cu): the bitonic
// network with its stages of partner distance < 128 run per tile of 128 keys over (tile, lane, register) indices -- key
// 32 r + l of a tile in register r of lane l, distance 64 and 32 between registers, 16 ... 1 with lane l ^ j -- and the
// stages of distance >= 128 strided over the whole array.  Checked against std::sort, descending, for every power of two
// np from 2 to 8192 with nc = np and with nc < np (the pass pads keys[nc..np) with zeros itself), on random distinct keys.
//   g++ -O2 -o /tmp/sortnet tools/sortnet.cpp && /tmp/sortnet [trials per size]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <vector>

typedef unsigned long long u64;
constexpr int SORT_TILE = 128;

static void sort_cx(u64 &a, u64 &b, const bool desc) { if (desc ? (a < b) : (a > b)) std::swap(a, b); }

// sort_tile_pass of beam.cu; the tiles are independent, so the order in which warps take them does not matter
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

int main(int argc, char **argv) {
  const int trials = argc > 1 ? atoi(argv[1]) : 20;
  std::mt19937_64 rng(1);
  long bad = 0, ran = 0;
  for (int np = 2; np <= 8192; np <<= 1) {
    long barriers = 0;
    for (int tr = 0; tr < trials; tr++) {
      // nc = np, np/2 + 1 (the fewest candidates that need this np), and something in between
      const int nc = (tr % 3 == 0) ? np : (tr % 3 == 1) ? np / 2 + 1 : np / 2 + 1 + (int)(rng() % (np / 2));
      std::vector<u64> keys(np), want;
      // the kernel's keys are distinct and non-zero: the candidate index is in the low 16 bits, a score key above it;
      // what lies in keys[nc..np) before the sort must not matter
      for (int i = 0; i < np; i++) keys[i] = ((rng() | 1ull) << 16) | (u64)i;
      want.assign(keys.begin(), keys.begin() + nc);
      std::sort(want.begin(), want.end(), std::greater<u64>());
      want.resize(np, 0ull);
      barriers = 0;
      sort_keys(keys, nc, np, barriers);
      ran++;
      if (keys != want) { if (bad++ < 5) printf("  mismatch: np %d nc %d\n", np, nc); }
    }
    printf("np %5d: %ld barriers (a barrier per stage: %d)\n", np, barriers, __builtin_ctz(np) * (__builtin_ctz(np) + 1) / 2);
  }
  printf("sorts %ld, mismatches %ld\n", ran, bad);
  return bad != 0;
}
