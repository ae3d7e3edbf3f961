// beam.cu -- K3: pass-1 lexicon-tree token passing, one persistent thread block per utterance.
//
// Stands in for libjulius/src/beam.c get_back_trellis_init/_proceed/_end + finalize_1st_pass
// (:1825, :2663, :3052, :3133), outprob_style (outprob_style.c:354-494), the factoring look-ups
// (factoring_sub.c:942-1143, ngram_access.c:249-305) and the word-trellis store/sort
// (backtrellis.c:190-267,438-478), stock "fast" switches: N-gram LMs on normal trees (beam_kernel<false, .>) and
// multipath trees (beam_kernel_mp); DFA grammars on the category tree (beam_kernel<true, .> = the same body with the
// three grammar-mode differences compiled in).  outprob_style's pseudo-phone set score is outprob_cd in common.cuh, the
// same code that fills the cd-set columns of the scorer's rows.
//
// Why this is not a transliteration.  The reference walks the survivors of frame t-1 one by one
// and lets each arc "propagate" into a per-node slot; ties are won by whoever arrived first, new
// tokens are numbered in order of first arrival, and the beam is cut by an in-place heap select
// whose OUTPUT ORDER (it decides next frame's arrival order) depends on the heap's mechanics.
// Scores sit on a coarse fp32 grid (|score| ~ 3e4 => ulp 2^-9), so exact ties are routine and
// every one of these order effects is observable in the word trellis.  The kernel computes the
// same fixed point with parallel primitives that are order-equivalent by construction:
//   * every candidate transition gets the sequence number it would have had in the sequential
//     walk:  seq = (survivor position j) * 2^18 + (arc index | n_intra + isolated-root index);
//     the factoring pass gets j = n_survivors;
//   * per destination node:  first arrival   = atomicMin(seq)          (who creates the token)
//                            winning content = atomicMax(score, ~seq)  (strict '<' keeps the incumbent)
//   * new-token numbering = rank of the creators in arrival order (one bit per candidate position, popcount prefix);
//   * inter-word transitions into the "isolated" roots are pre-reduced per root over the frame's
//     word-end tokens (max is associative; first/winner seqs are carried along); the per-last-word
//     bigram rows the reference caches lazily (iw_sc_cache) are tabulated once at create time;
//   * the beam cut reproduces the reference's heap select exactly (beam_cut): bottom-up heap
//     construction is level-parallel (siftdowns of one level touch disjoint subtrees), the
//     extraction order comes from a closed form (heap_select_closed) or from a replay by one warp
//     with up to 16 extractions in flight (heap_pipe.cuh), and the other warps reset the per-node
//     slots for the next frame meanwhile.
// All frames of an utterance run inside one kernel launch; tokens, node slots and candidates
// live in per-utterance global scratch (L2 resident), the sort/heap array in shared memory.
//
// Compiled with --fmad=false: every float decision uses the reference's fp32 expression order.
#include "common.cuh"
#include "heap_pipe.cuh"
#include <vector>
#include <algorithm>

struct jb200_gmm;
struct jb200_dnn;
namespace jb200 {
int dnn_fix_context(jb200_dnn *h);
int dnn_forward_device(jb200_dnn *h, const float *d_in, int T, float *d_rows, int row_stride, cudaStream_t st, const SpliceMap &sm);
int gmm_device(const jb200_gmm *h);
int gmm_dim(const jb200_gmm *h);
int gmm_launch_states(jb200_gmm *h, const float *d_feats, int T, float *d_rows, int row_stride, cudaStream_t st,
                      const int *seg_off, const int *seg_start, int n_seg);
CdSets gmm_cdsets(const jb200_gmm *h);

static constexpr int BEAM_THREADS = 256;
static constexpr int NWARP = BEAM_THREADS / 32;
static constexpr int SEQ_LOCAL_BITS = 18;
static constexpr unsigned SEQ_LOCAL = 1u << SEQ_LOCAL_BITS;
static constexpr int MAX_WORDS = 150;      // MAXSEQNUM, libsent/include/sent/speech.h:50

struct __align__(16) NodeRec { float self_a, next_a; int arc_off, arc_n; int stend, next; int scid, out; };   // 32 B; (scid,out) is one aligned 8-byte word; next = the node next_a leads to
struct __align__(8) Tok { float score; int node; int tre; int cword; float lscore; int tre_wid; };              // 24 B
struct __align__(16) Cand { float score; int node; float lscore; int src; };                                     // 16 B
struct __align__(16) CandB { int tre; int cword; int tre_wid; int out; };                                        // 16 B: what the winner hands to the new token
struct __align__(16) IsoCand { float score; int e; float lscore; int first_e; };                                 // 16 B
struct __align__(8) WEnd { int j; int atom; int last_word; float base; int transp2; int nintra; };              // 24 B

// per-node arrival slot: who reached the node first (creator) and who reached it best (content); one aligned
// 16-byte record so that the two atomics, the reset and the later reads of a node touch a single sector
struct __align__(16) NodeSlot { unsigned long long bestkey; int firstseq; int pad; };
struct SlotView {
  NodeSlot *s;
  __device__ __forceinline__ int *fs(int node) const { return &s[node].firstseq; }
  __device__ __forceinline__ unsigned long long *bk(int node) const { return &s[node].bestkey; }
  __device__ __forceinline__ void set(int node, int firstseq, unsigned long long bestkey) const {
    __stcg(reinterpret_cast<uint4 *>(s + node), make_uint4((unsigned)bestkey, (unsigned)(bestkey >> 32), (unsigned)firstseq, 0u));
  }
  __device__ __forceinline__ void reset(int node) const { set(node, 0x7fffffff, 0ull); }
};

// One launch of a beam kernel covers frames [t0, t1) of an utterance: the whole utterance (FIRST|FINAL), or one piece of
// it -- the batch pipeline cuts utterances into chunks so that the scoring of chunk c+1 runs beside the token passing of
// chunk c, and a stream (jb200_stream_*) advances as its input arrives, which is how the reference drives pass 1
// (decode_proceed, one frame per call, libjulius/src/pass1.c:112-254).  Everything an utterance carries from frame to
// frame lives in its global work area already; the few scalars the kernel keeps in shared memory are parked in UttState.
static constexpr int CHUNK_FIRST = 1, CHUNK_FINAL = 2, CHUNK_SKIP = 4;   // SKIP: nothing to do for this utterance in this launch
struct ChunkDesc { int t0, t1, flags, row_base; };   // score row of frame t: rows + (row_base + t) * row_stride
struct UttState {
  int ns, natoms, tnum_prev, slots_clean, overflow, stopped, cur;   // cur: the multipath kernel's current token list
  float thr; int t_done;
  // best partial sentence at the last frame done (bt_current_max, beam.c:876-921): filled when BeamParams.interim is set
  int interim_frame, interim_nwords; float interim_score; int pad_;
  long long prof[8];
};

// The beam-cut counters (BeamParams::cut_counters), summed over all frames since create
enum CutCounter {
  CUT_SEQ_FALLBACKS,     // fall-backs to the plain sequential replay: there are none, always 0
  CUT_REPLAY_TICKS,      // replay ticks
  CUT_REPLAY_EXTRACTS,   // extractions replayed
  CUT_HELD_BACK,         // held-back starts of the replay (counted, not reported)
  CUT_UPWARD,            // upward selects
  CUT_CLOSED,            // of which closed form
  CUT_RELOCATED,         // of which with relocations
  CUT_GLOBAL_WHOLE,      // global-memory heap: replays on a shared-memory copy of the whole heap
  CUT_GLOBAL_TOP_TAIL,   // global-memory heap: replays on the heap itself, its top and tail copied
  CUT_SLOTS = 16         // slots allocated
};

struct BeamParams {
  // tree
  const NodeRec *nodes; const int *arc_to; const float *arc_a;
  const int *rset_ctx; const int *word_ctx; int n_ctx;
  const int *iso_node; const int *iso_id; int n_iso; const float *iw;
  const int *shared_node; const float *shared_f; int n_shared;
  // multipath trees: the roots carry no output, so cross-word transitions land one arc further
  // (beam.c:2467-2500, :2584-2605): the successors of the isolated / shared roots, root-major
  int multipath; const int *isoarc_node; const int *isoarc_iso; const float *isoarc_a; int n_isoarc;
  const int *sharc_node; const int *sharc_shared; const float *sharc_a; int n_sharc;
  const float *wordend_a; const uint8_t *is_transp; const int *wton; const float *cprob;
  const float *fscore; const int *scword;
  const float *uni_prob; const float *uni_bow; const int *bi_bgn; const int *bi_num; const int *bi_wid; const float *bi_prob;
  int lm_mode, lm_unk_id; float lm_unk_num_log;
  float lm_weight, lm_penalty, lm_penalty_trans, prune_width;
  int head_node, tail_silwid, beam, n_nodes;
  // cd sets
  CdSets cd;
  // batch
  const float *rows; int row_stride; const int *frame_off;
  // per-utterance work areas (index = blockIdx.x)
  Tok *tok; int *order; NodeSlot *slots; Cand *cand; CandB *candb; Tok *surv; IsoCand *iso; WEnd *wend;
  jb200_atom *atoms_raw; int *newidx; int *group0; int *counts;
  const long long *atom_off;
  // compact outputs
  jb200_atom *atoms_out; unsigned long long *atom_counter; long long atoms_out_cap;
  jb200_utt_result *results; int *words;
  long long *prof;            // [n_utts][8] cycle counters per phase, or NULL
  unsigned *bitmask; int *wordpre;   // per-utterance arrival-order bitmask [maxbits/32] and its word prefix counts
  unsigned long long *cut_counters;           // [CUT_SLOTS], indexed by CutCounter
  unsigned long long *lmc; int lmc_bits;      // memo of max_successor_prob, 2^lmc_bits entries (0 = off)
  int maxt, maxc, maxw, maxbits;
  // token sets too large for shared memory (wide beams on large trees): the heap-select array lives in global memory
  // ([n_utts][maxt+4] entries) and shared memory only holds the closed form's sort area (sort_cap 8-byte keys)
  unsigned long long *heap_g; int sort_cap, qcap;      // qcap: 8-byte entries of the shared-memory area in front of offs (>= sort_cap)
  // grammar (DFA) mode, appended so that the offsets of everything above stay what the N-gram kernels were built with
  const uint8_t *cp_allowed; const int *init_node; const float *init_lscore; int n_init; float penalty1;
  // chunked launches
  const ChunkDesc *chunk; UttState *state; int interim; int *interim_words;   // [n_utts][MAX_WORDS]
  int atoms_in_place;       // streams: the finalized atoms of utterance u go to atoms_out + atom_off[u] (no batch compaction)
  unsigned long long *heap_chk;   // JB200_CHECK_HEAP on a multipath tree: [n_utts][maxt+4] input of the sequential replay
};

// ---- small device helpers ----------------------------------------------------------------------
__device__ __forceinline__ unsigned fkey(float f) {
  unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ int search_bigram(const BeamParams &p, int wc, int w) {
  int left = __ldg(p.bi_bgn + wc);
  if (left < 0) return -1;
  int right = left + __ldg(p.bi_num + wc) - 1;
  while (left < right) {
    int mid = (left + right) / 2;
    if (__ldg(p.bi_wid + mid) < w) left = mid + 1; else right = mid;
  }
  return (__ldg(p.bi_wid + left) == w) ? left : -1;
}

// bi_prob_normal / _additional(_oldbin) / _compute, ngram_access.c:288-405
__device__ float bigram_prob(const BeamParams &p, int w1, int w2) {
  int n2; float prob;
  if (p.lm_mode == JB200_BI_NORMAL || p.lm_mode == JB200_BI_ADDITIONAL_OLDBIN) {
    if ((n2 = search_bigram(p, w1, w2)) >= 0) prob = __ldg(p.bi_prob + n2);
    else prob = __ldg(p.uni_bow + w1) + __ldg(p.uni_prob + w2);
  } else if (p.lm_mode == JB200_BI_ADDITIONAL) {
    if ((n2 = search_bigram(p, w2, w1)) >= 0) prob = __ldg(p.bi_prob + n2);
    else prob = __ldg(p.uni_bow + w1) + __ldg(p.uni_prob + w2);
  } else {
    if ((n2 = search_bigram(p, w2, w1)) >= 0) prob = __ldg(p.bi_prob + n2);
    else prob = __ldg(p.uni_bow + w2) + __ldg(p.uni_prob + w1);
    prob = prob + __ldg(p.uni_prob + w2) - __ldg(p.uni_prob + w1);
  }
  if (w2 != p.lm_unk_id) return prob;
  return prob - p.lm_unk_num_log;
}

// max_successor_prob, factoring_sub.c:942-1012 (1-gram factoring build).  The reference keeps a per-node
// one-entry cache of the bigram look-up (factoring_sub.c:984-1006); here a direct-mapped table shared by
// all utterances memoises the pure function (last word, successor-word slot) -> value, because the binary
// search is ~10 dependent global loads and the same pairs recur every frame while a token waits on the
// node in front of a single-word branch.  One 64-bit word per entry: key in the high half, value bits in
// the low half, written and read atomically as a unit.
__device__ __forceinline__ float max_successor_prob(const BeamParams &p, int lastword, int scid) {
  if (lastword < 0) return 0.0f;
  if (scid < 0) return __ldg(p.fscore - scid);
  unsigned long long *slot = nullptr;
  unsigned key = 0u;
  if (p.lmc_bits > 0) {
    key = ((unsigned)lastword << 16) | (unsigned)scid;
    slot = p.lmc + ((key * 2654435761u) >> (32 - p.lmc_bits));
    const unsigned long long e = __ldcg(slot);
    if ((unsigned)(e >> 32) == key) return __uint_as_float((unsigned)e);
  }
  int w = __ldg(p.scword + scid);
  const float v = bigram_prob(p, __ldg(p.wton + lastword), __ldg(p.wton + w)) + __ldg(p.cprob + w);
  if (slot) __stcg(slot, ((unsigned long long)key << 32) | __float_as_uint(v));
  return v;
}

// outprob_style, outprob_style.c:354-494 with the context resolution tabulated on the host
__device__ __forceinline__ float outprob_style(const BeamParams &p, const float *__restrict__ row, int out, int last_wid) {
  const int style = (unsigned)out >> 28, ref = out & 0x0fffffff;
  if (style == JB200_AS_STATE) return __ldg(row + ref);
  if (style == JB200_AS_LSET) return outprob_cd(p.cd, row, ref);
  const int col = (last_wid < 0) ? p.n_ctx : __ldg(p.word_ctx + last_wid);
  const int r = __ldg(p.rset_ctx + (size_t)ref * (p.n_ctx + 1) + col);
  if (r >= 0) return __ldg(row + r);
  return outprob_cd(p.cd, row, -r - 1);
}

// block-wide exclusive scan of one int per thread; *total = block sum.  Ends with a barrier.
__device__ __forceinline__ int block_excl_scan(int v, int *warp_sums, int *total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = (lane < NWARP) ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    if (lane < NWARP) warp_sums[lane] = s;   // inclusive
  }
  __syncthreads();
  const int base = (wid == 0) ? 0 : warp_sums[wid - 1];
  *total = warp_sums[NWARP - 1];
  const int r = base + x - v;
  __syncthreads();
  return r;
}

__device__ __forceinline__ void cand_atomics(const SlotView &slots,
                                             int node, float score, unsigned seq_first, unsigned seq_win) {
  atomicMin(slots.fs(node), (int)seq_first);
  unsigned long long key = ((unsigned long long)fkey(score) << 32) | (unsigned)(~seq_win);
  atomicMax(slots.bk(node), key);
}

// heap entries: high 32 bits = token id, low 32 bits = fp32 score bits.  Heap index h (1-based) lives
// in slot h, so the sibling pair (2p, 2p+1) is one aligned 16-byte word.
__device__ __forceinline__ float hval(unsigned long long e) { return __uint_as_float((unsigned)(e & 0xffffffffu)); }

template <bool MAXHEAP>
__device__ __forceinline__ bool hcmp(float a, float b) { return MAXHEAP ? (a < b) : (a > b); }      // "child < child+1"
template <bool MAXHEAP>
__device__ __forceinline__ bool hstop(float s, float c) { return MAXHEAP ? (s >= c) : (s <= c); }   // "STVAL >= SVAL(child)"

template <bool MAXHEAP>
__device__ __forceinline__ void sift_down(unsigned long long *A, int start, int n) {
  // the inner loop of sort_token_upward / _downward, beam.c:1355-1368 / :1421-1434
  const unsigned long long s = A[start];
  const float sv = hval(s);
  int parent = start, child;
  while ((child = parent * 2) <= n) {
    const ulonglong2 pr = *reinterpret_cast<const ulonglong2 *>(A + child);
    unsigned long long c = pr.x;
    if (child < n && hcmp<MAXHEAP>(hval(pr.x), hval(pr.y))) { child++; c = pr.y; }
    if (hstop<MAXHEAP>(sv, hval(c))) break;
    A[parent] = c;
    parent = child;
  }
  A[parent] = s;
}

// one extraction step chain, two tree levels per shared-memory round trip
template <bool MAXHEAP>
__device__ __forceinline__ void sift_root_2level(unsigned long long *A, const unsigned long long s, const int m) {
  const float sv = hval(s);
  int parent = 1;
  while (true) {
    int child = parent * 2;
    if (child > m) break;
    // children pair and the four grandchildren (slots 4p..4p+3), loaded together
    const ulonglong2 pr = *reinterpret_cast<const ulonglong2 *>(A + child);
    const int g = parent * 4;
    ulonglong2 g01 = make_ulonglong2(0ull, 0ull), g23 = make_ulonglong2(0ull, 0ull);
    if (g <= m) g01 = *reinterpret_cast<const ulonglong2 *>(A + g);
    if (g + 2 <= m) g23 = *reinterpret_cast<const ulonglong2 *>(A + g + 2);
    // level 1
    unsigned long long c = pr.x; bool right = false;
    if (child < m && hcmp<MAXHEAP>(hval(pr.x), hval(pr.y))) { right = true; c = pr.y; }
    if (hstop<MAXHEAP>(sv, hval(c))) break;
    A[parent] = c;
    parent = child + (right ? 1 : 0);
    // level 2 (children of the chosen child are g01 or g23)
    child = parent * 2;
    if (child > m) break;
    const ulonglong2 q = right ? g23 : g01;
    unsigned long long c2 = q.x; bool right2 = false;
    if (child < m && hcmp<MAXHEAP>(hval(q.x), hval(q.y))) { right2 = true; c2 = q.y; }
    if (hstop<MAXHEAP>(sv, hval(c2))) break;
    A[parent] = c2;
    parent = child + (right2 ? 1 : 0);
  }
  A[parent] = s;
}

template <bool MAXHEAP>
__device__ void heap_build(unsigned long long *A, int n) {
  // build: roots n/2 .. 1; all roots of one tree level are independent (disjoint subtrees) and the
  // sequential order visits deeper levels first, so a level-synchronous sweep is equivalent.
  const int half = n >> 1;
  if (half >= 1) {
    for (int L = 31 - __clz(half); L >= 0; L--) {
      const int lo = 1 << L;
      const int hi = min((2 << L) - 1, half);
      for (int i = lo + (int)threadIdx.x; i <= hi; i += BEAM_THREADS) sift_down<MAXHEAP>(A, i, n);
      __syncthreads();
    }
  }
}

// Sequential extraction replay (beam.c:1370-1384): s = last; last = root; shrink; sift s from the root.
template <bool MAXHEAP>
__device__ void heap_extract_seq(unsigned long long *A, int n, int extract) {
  if (threadIdx.x == 0) {
    int m = n;
    while (m > n - extract) {
      const unsigned long long s = A[m];
      A[m] = A[1];
      m--;
      if (m >= 1) sift_root_2level<MAXHEAP>(A, s, m);
    }
  }
  __syncthreads();
}

// The pipelined replay (heap_pipe.cuh) for a heap in GLOBAL memory -- the token set of a wide beam on a large tree does
// not fit shared memory (-b 4000 on the 60k-word tree: up to 34k tokens a frame).  Same schedule, plain generic loads and
// stores that bypass L1 (another lane wrote the line one tick ago); a tick costs an L2 round trip instead of a
// shared-memory one, so this path is for the frames the closed form cannot answer.  outs: shared memory.
__device__ __forceinline__ ulonglong2 ldcg_pair(const unsigned long long *p) {
  const uint4 v = __ldcg(reinterpret_cast<const uint4 *>(p));
  return make_ulonglong2(((unsigned long long)v.y << 32) | v.x, ((unsigned long long)v.w << 32) | v.z);
}
// Shared-memory copies that go with a global-memory heap (write-through, so global stays the truth):
//   top  : slots [0, cs) -- the top levels of the tree, which every extraction walks;
//   tail : slots [tail_first, tail_first + tail_n) -- where the extractions take their s from.
// Deeper levels are touched only by the few sifts that follow winners all the way down.
struct HeapCache {
  unsigned long long *top; int cs;
  unsigned long long *tail; int tail_first, tail_n;
};

template <bool MAXHEAP>
__device__ void heap_extract_pipe_global(unsigned long long *A, const int n, const int extract, const float lose_below,
                                         unsigned long long *outs, const int maxt, const HeapCache hc,
                                         unsigned &ticks_out, unsigned &stalls_out) {
  constexpr int NL = 16;
  constexpr unsigned FULL = 0xffffffffu;
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long sent = MAXHEAP ? 0xff800000ull : 0x7f800000ull;
  const int cap = (maxt >> 1) + 1;                          // pair (maxt+2, maxt+3): always sentinels
  auto load_slot = [&](int i) -> unsigned long long {
    if (i < hc.cs) return hc.top[i];
    if (i >= hc.tail_first && i < hc.tail_first + hc.tail_n) return hc.tail[i - hc.tail_first];
    return __ldcg(A + i);
  };
  auto store_slot = [&](int i, unsigned long long v) {
    __stcg(A + i, v);
    if (i < hc.cs) hc.top[i] = v;
    else if (i >= hc.tail_first && i < hc.tail_first + hc.tail_n) hc.tail[i - hc.tail_first] = v;
  };
  bool act = false;
  int slot = 0, cur = cap, my_x = 0;                        // hole index, pair index of its children (slots 2cur, 2cur+1)
  unsigned long long s = sent;
  int next_x = 0, wait = 0;
  unsigned ticks = 0, stalls = 0;
  if (lane == 0 && extract > 0) outs[0] = load_slot(1);
  unsigned long long nxt = load_slot(n);
  while (true) {
    // (1) children pair of the hole
    ulonglong2 pr = make_ulonglong2(sent, sent);
    if (act) {
      const int i = 2 * cur;
      if (i + 1 < hc.cs) pr = *reinterpret_cast<const ulonglong2 *>(hc.top + i);
      else if (i >= hc.tail_first && i + 1 < hc.tail_first + hc.tail_n) pr = make_ulonglong2(hc.tail[i - hc.tail_first], hc.tail[i + 1 - hc.tail_first]);
      else pr = ldcg_pair(A + i);
    }
    // (2) fill the hole, move one level down or end
    if (act) {
      const float xv = hval(pr.x), yv = hval(pr.y), sv = hval(s);
      const bool right = hcmp<MAXHEAP>(xv, yv);
      const unsigned long long c = right ? pr.y : pr.x;
      const float cv = hval(c);
      const bool stop = hstop<MAXHEAP>(sv, cv) || (MAXHEAP && cv < lose_below);
      const unsigned long long put = stop ? s : c;
      store_slot(slot, put);
      if (slot == 1) outs[my_x + 1] = put;
      if (stop) act = false;
      else { slot = 2 * cur + (right ? 1 : 0); cur = min(slot, cap); }
    }
    __syncwarp();
    // (3) may the next extraction start?  (holes as they are after the move)
    if (--wait <= 0) {
      if (next_x >= extract) { if (!__any_sync(FULL, act)) break; }
      else {
        const int ms = n - next_x;
        const int ln = next_x & (NL - 1);
        bool blocks = act && ((int)lane == ln);
        // a tail slot holding a loser is never a hole and never decides anything (loser cut), and a loser stays a loser
        if (!(MAXHEAP && hval(nxt) < lose_below)) {
          const int dh = 31 - __clz(max(slot, 1)), dms = 31 - __clz(ms);
          blocks = blocks || (act && dms >= dh && (ms >> (dms - dh)) == slot);
        }
        if (!__any_sync(FULL, blocks)) {
          if ((int)lane == ln) {
            s = load_slot(ms);
            store_slot(ms, sent);
            my_x = next_x; act = true; slot = 1; cur = 1;
          }
          next_x++; wait = 2;
          nxt = load_slot(n - next_x);                    // the next tail slot's content (every lane: a broadcast)
        } else stalls++;
      }
    }
    __syncwarp();
    ticks++;
  }
  ticks_out = ticks; stalls_out = stalls;
}

// work for the otherwise idle warps during an extraction replay: reset the per-node slots of the tokens created in this
// frame (clear_tokens, beam.c:1122, moved ahead of the next frame)
struct SlotClear {
  const Tok *tok; int n; SlotView slots;
  __device__ __forceinline__ void run(int first, int stride) const {
    for (int i = first; i < n; i += stride) {
      const int node = tok[i].node;
      slots.reset(node);
    }
  }
};

// Freed tail slots and everything between n+1 and the last child slot hold a sentinel (-inf for the max-heap, +inf for
// the min-heap), and so does the pair (maxt+2, maxt+3): both bounds tests of the reference loop ("child <= n",
// "child < n") fall out of the value comparisons -- a missing right child never wins, a missing pair stops the sift.
template <bool MAXHEAP>
__device__ __forceinline__ void heap_pad_sentinels(unsigned long long *A, const int n, const int maxt) {
  const unsigned long long sent = MAXHEAP ? 0xff800000ull : 0x7f800000ull;
  const int hi = min(2 * n + 1, maxt + 1);
  for (int i = n + 1 + (int)threadIdx.x; i <= hi; i += BEAM_THREADS) A[i] = sent;
  if (threadIdx.x < 2) A[maxt + 2 + threadIdx.x] = sent;
}

// The work areas of the heap select, the same in every beam kernel.  Shared memory: [heap (maxt+4 entries) | offs], or,
// when the token set is too large for shared memory and the heap lives in global memory (heap_g),
// [qcap entries: the closed form's sort area and the replay's copy of the heap | offs | copy of the tail slots].
// offs: 2 x (beam+2) ints that hold the kernels' per-survivor offsets; they are dead during the cut, which keeps its
// histogram, the closed form's payload and the extracted roots (outv) there.
extern __shared__ __align__(16) unsigned char beam_smem[];
struct CutAreas {
  unsigned long long *heap;             // slot h = heap index h
  int *offs;
  unsigned long long *gq; int gqn;      // global heap only: the shared-memory area in front of offs
  unsigned long long *gtail; int gtn;   // global heap only: the shared-memory copy of the tail slots behind offs
  __device__ __forceinline__ unsigned long long *outv() const { return reinterpret_cast<unsigned long long *>(offs); }
};
__device__ __forceinline__ CutAreas cut_areas(const BeamParams &p) {
  unsigned long long *const smem_q = reinterpret_cast<unsigned long long *>(beam_smem);
  CutAreas a;
  a.heap = p.heap_g ? p.heap_g + (size_t)blockIdx.x * (p.maxt + 4) : smem_q;
  a.offs = reinterpret_cast<int *>(smem_q + (p.heap_g ? p.qcap : p.maxt + 4));
  a.gq = p.heap_g ? smem_q : nullptr;
  a.gqn = p.heap_g ? p.qcap : 0;
  a.gtail = p.heap_g ? reinterpret_cast<unsigned long long *>(a.offs + 2 * (p.beam + 2)) : nullptr;
  a.gtn = p.heap_g ? p.beam + 1 : 0;
  return a;
}

// Extraction replay of the heap ca.heap[1..n] (sentinel padded): the k-th extracted root goes to outv[k].  Warp 0
// replays, the other warps run idle_work.  Ends with a barrier.
template <bool MAXHEAP>
__device__ void heap_extract_fast(const CutAreas &ca, const int n, const int extract, const float lose_below, const int maxt,
                                  unsigned long long *stats, const SlotClear *idle_work = nullptr) {
  unsigned long long *const A = ca.heap, *const outv = ca.outv(), *const gcache = ca.gq;
  HeapCache hc{nullptr, 0, nullptr, 0, 0};
  if (!__isShared(A) && n + 8 <= ca.gqn) {
    // global-memory heap that fits the shared-memory area as a whole (select #1 of a multipath frame, and the smaller
    // frames of a wide beam): replay on a shared-memory copy at shared-memory speed, then write the arrangement back
    const int lmaxt = (ca.gqn - 4) & ~1;
    for (int i = threadIdx.x; i <= n; i += BEAM_THREADS) gcache[i] = A[i];
    heap_pad_sentinels<MAXHEAP>(gcache, n, lmaxt);
    __syncthreads();
    if (threadIdx.x >= 32 && idle_work) idle_work->run((int)threadIdx.x - 32, BEAM_THREADS - 32);
    if (threadIdx.x < 32) {
      unsigned ticks, stalls;
      heap_extract_pipe_warp6<MAXHEAP>(gcache, n, extract, lose_below, outv, lmaxt, threadIdx.x, ticks, stalls);
      if (threadIdx.x == 0) {
        atomicAdd(stats + CUT_REPLAY_TICKS, (unsigned long long)ticks); atomicAdd(stats + CUT_REPLAY_EXTRACTS, (unsigned long long)extract);
        atomicAdd(stats + CUT_HELD_BACK, (unsigned long long)stalls); atomicAdd(stats + CUT_GLOBAL_WHOLE, 1ull);
      }
    }
    __syncthreads();
    for (int i = 1 + threadIdx.x; i <= n; i += BEAM_THREADS) A[i] = gcache[i];
    __syncthreads();
    return;
  }
  if (!__isShared(A)) {
    // global-memory heap: copy its top levels and its tail into shared memory first (all threads)
    hc.top = gcache; hc.cs = min(ca.gqn, maxt + 4) & ~1;
    for (int i = threadIdx.x; i < hc.cs; i += BEAM_THREADS) gcache[i] = A[i];
    if (ca.gtn >= extract) {
      hc.tail = ca.gtail; hc.tail_first = n - extract + 1; hc.tail_n = extract;
      for (int i = threadIdx.x; i < extract; i += BEAM_THREADS) ca.gtail[i] = A[hc.tail_first + i];
    }
    __syncthreads();
  }
  if (threadIdx.x >= 32 && idle_work) idle_work->run((int)threadIdx.x - 32, BEAM_THREADS - 32);
  // warp 0: up to 16 extractions in flight, one tree level per tick each (heap_pipe.cuh)
  if (threadIdx.x < 32) {
    unsigned ticks, stalls;
    if (!__isShared(A)) heap_extract_pipe_global<MAXHEAP>(A, n, extract, lose_below, outv, maxt, hc, ticks, stalls);
    else heap_extract_pipe_warp6<MAXHEAP>(A, n, extract, lose_below, outv, maxt, threadIdx.x, ticks, stalls);
    if (threadIdx.x == 0) {
      atomicAdd(stats + CUT_REPLAY_TICKS, (unsigned long long)ticks); atomicAdd(stats + CUT_REPLAY_EXTRACTS, (unsigned long long)extract);
      atomicAdd(stats + CUT_HELD_BACK, (unsigned long long)stalls);
      if (!__isShared(A)) atomicAdd(stats + CUT_GLOBAL_TOP_TAIL, 1ull);
    }
  }
  __syncthreads();
}

// ---- closed form of an upward select ------------------------------------------------------------------------------
// When every sift of the extraction loop ends on a loser (an element that is never extracted) an extraction is a pure
// "pull-up": the hole at the root is filled by the larger child (the left one on a tie), and so on down.  Two elements of
// equal score then keep their relative PRE-ORDER position in the tree for ever -- the one in the right subtree of their
// lowest common ancestor could only overtake by being strictly larger than everything in the left subtree -- and the
// root is first in pre-order, hence
//        extraction order = (score descending, pre-order position in the BUILT heap ascending).
// A re-inserted winner (the tail slot an extraction takes holds an element that will itself be extracted) sinks from the
// root instead and may land ahead of elements it ties with; it cannot disturb the order of anybody else.  Such an
// element e sits in a tail slot p of the built heap (tail slots are leaves, nothing is promoted into a leaf, so a tail
// slot holds its original content or an earlier extraction's s, itself a tail content) and when p is taken, at step
// k = n-p+1, the k-1 elements extracted so far and the d = depth(p) elements on the slots above p are all ahead of e.
// So if  rank(e) < k + d  for every tail element that ties with another candidate, no re-insertion can matter and the
// closed form is exact; otherwise the relocation pass below follows the re-insertions.  tools/beamcut.cpp models
// collection, sort, test and relocation pass as this function runs them and checks them against the plain loop.
//
// All threads call it after heap_build<true>.  Candidates = elements >= lose_below (a lower bound of the need-th largest
// score); they are sorted with a bitonic network in `keys` (shared memory: the free part of the heap array, slots
// n+1.., or a dedicated area when the heap itself lives in global memory), keys
//   [ order-preserving score key : 32 | 0xffff - pre-order position : 16 | candidate index : 16 ]  descending,
// payload (slot << 16 | token id) in `pay`.  Returns 1 and fills ordn[0..need) (visiting order = reverse extraction order)
// or returns 0 with the heap intact (everything above slot n must be padded again before a replay).
__device__ __forceinline__ int closed_subtree_size(const int c, const int n, const int H) {
  const int dc = 31 - __clz(c);
  if (dc > H) return 0;
  const int sh = H - dc;
  const int first = c << sh, width = 1 << sh;
  return (width - 1) + max(0, min(n - first + 1, width));
}

// The relocation pass reads the order in windows of RELOC_WINDOW x 32 keys: the loads of a window are independent, and a
// scan that passes a whole window without a match costs one load round and RELOC_WINDOW ballots instead of RELOC_WINDOW
// dependent chunk iterations (the pass runs on one warp while the block waits, so its dependent chain is what it costs).
constexpr int RELOC_WINDOW = 3;
// The home pre-order positions of the window keys[base .. base + 32 RELOC_WINDOW), two 16-bit positions per register
// (chunk c in half c & 1 of pre[c >> 1]); 0xffff for keys past nc and for keys[skip]: no interval [lo, hi) of the n < 65536
// slots holds it.
__device__ __forceinline__ void reloc_window_load(const unsigned long long *keys, const int nc, const int base, const int skip, const int lane,
                                                  unsigned (&pre)[(RELOC_WINDOW + 1) / 2]) {
#pragma unroll
  for (int c = 0; c < RELOC_WINDOW; c++) {
    const int idx = base + 32 * c + lane;
    const unsigned p = (idx < nc && idx != skip) ? 0xffffu - (unsigned)((keys[idx] >> 16) & 0xffffu) : 0xffffu;
    if (c & 1) pre[c >> 1] |= p << 16; else pre[c >> 1] = p;
  }
}
// first position >= from of the window (chunk c, lane l = position 32c + l) whose home pre-order position lies in
// [lo, hi); -1 if none
__device__ __forceinline__ int reloc_window_first(const unsigned (&pre)[(RELOC_WINDOW + 1) / 2], const int lo, const int hi, const int from, const int lane) {
  // the ballots of the chunks do not depend on each other: all of them, then the first hit
  int f = -1;
#pragma unroll
  for (int c = RELOC_WINDOW - 1; c >= 0; c--) {
    const int p = (int)((pre[c >> 1] >> (16 * (c & 1))) & 0xffffu);
    const unsigned b = __ballot_sync(0xffffffffu, p >= lo && p < hi && 32 * c + lane >= from);
    if (b) f = 32 * c + __ffs(b) - 1;
  }
  return f;
}

// ---- the closed form WITH re-insertions ----------------------------------------------------------------------------
// While every extraction's s is a loser the heap evolves by pull-ups and
//   (I)  slot x holds the best remaining element of subtree(x) that no ancestor of x holds,
// "best" = (score descending, pre-order position of the element's HOME slot ascending) -- which is also the extraction
// order.  A tail leaf that still holds a candidate when it is taken breaks the pure pull-up picture: the element is
// re-inserted from the root and lands on the chain of larger children where its score says, ABOVE whatever it ties with.
// (I) survives if the element's home moves to where it lands (it is at least as good as both sub-trees below it).  So the
// sorted candidate keys ARE the heap: for every flagged tail slot m, high slots first (step k = n-m+1),
//   * who sits in leaf m: walk the alive part of the order (index >= k-1) and hand out the levels of the path root..m --
//     level j goes to the first unused element whose home lies in subtree(a_j) (nested intervals of pre-order
//     positions); m holds a candidate iff level depth(m) gets one;
//   * where that element e lands: walk the order behind the root; the first element of subtree(x) is the occupant of the
//     larger child of x (the left one on a tie: that is the order); e stays at x if its score is >= that element's
//     ("STVAL >= SVAL(child)", beam.c:1362), else the hole moves into the child whose subtree holds that element's home;
//   * e's key gets the landing slot's pre-order position and moves to its place in the order (behind this step's root).
// tools/beamcut.cpp emulates it lane by lane, exact on recorded cuts of real decodes and on random heaps with as few as
// 2 distinct scores.  One warp; returns 0 on anything unexpected (the caller replays the loop instead).
__device__ __forceinline__ int closed_relocate(unsigned long long *keys, const int nc, const int n, const int need, unsigned *flags, unsigned *multi,
                                            unsigned *pay, const int lane) {
  constexpr unsigned FULL = 0xffffffffu;
  const int H = 31 - __clz(n);
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  for (int w = fwords - 1; w >= 0; w--) {
    unsigned bits = flags[w];
    while (bits) {
      const int b = 31 - __clz(bits);
      const int m = tail0 + w * 32 + b;
      const int k = n - m + 1;                              // step; this step's root is keys[k-1]
      if (m <= n && m >= 2 && k <= need) {
        const int dm = 31 - __clz(m);
        const bool is_multi = (multi[(m - tail0) >> 5] >> ((m - tail0) & 31)) & 1u;    // a re-inserted element landed in this leaf too
        // --- the occupant of leaf m
        int j = 0, a = 1, lo = 0, hi = n, occ = -1;
        bool gone = false;
        for (int base = k - 1; base < nc && occ < 0 && !gone; base += 32 * RELOC_WINDOW) {
          unsigned pre[(RELOC_WINDOW + 1) / 2];
          reloc_window_load(keys, nc, base, -1, lane, pre);
          int from = 0;
          while (true) {
            const int f = reloc_window_first(pre, lo, hi, from, lane);
            if (f < 0) break;
            if (j == dm) { occ = base + f; break; }
            // the leaf's own candidate, pulled up to level j: only a loser can be in the leaf now
            if (!is_multi && (int)(pay[(unsigned)keys[base + f] & 0xffffu] >> 16) == m) { gone = true; break; }
            j++;
            const int nxt = m >> (dm - j);
            const int lsz = closed_subtree_size(2 * a, n, H);
            if (nxt == 2 * a) { lo = lo + 1; hi = lo + lsz; } else { lo = lo + 1 + lsz; }
            a = nxt;
            from = f + 1;
          }
        }
        if (occ >= k) {
          // --- e = keys[occ] is re-inserted from the root of the heap of m-1 slots
          __syncwarp();
          const unsigned long long ekey = keys[occ];
          const unsigned esc = (unsigned)(ekey >> 32);
          const int msz = m - 1;
          int x = 1; lo = 0; hi = n;
          bool stop = (2 * x > msz);
          for (int base = k; base < nc && !stop; base += 32 * RELOC_WINDOW) {
            unsigned pre[(RELOC_WINDOW + 1) / 2];
            reloc_window_load(keys, nc, base, occ, lane, pre);
            int from = 0;
            while (!stop) {
              const int f = reloc_window_first(pre, lo, hi, from, lane);
              if (f < 0) break;
              const unsigned long long fk = keys[base + f];
              const unsigned osc = (unsigned)(fk >> 32);
              const int opre = 0xffff - (int)((fk >> 16) & 0xffffu);
              if (opre == lo) return 0;                     // an unplaced element whose home is x: cannot happen
              if (esc >= osc) { stop = true; break; }        // e stays at x
              const int lsz = closed_subtree_size(2 * x, n, H);
              if (opre < lo + 1 + lsz) { x = 2 * x; lo = lo + 1; hi = lo + lsz; }
              else { x = 2 * x + 1; lo = lo + 1 + lsz; }
              if (2 * x > msz) { stop = true; break; }
              from = f + 1;
            }
          }
          // --- e's home is x (pre-order position lo): new key, new place among the alive elements behind this step's root
          const unsigned long long nkey = (ekey & 0xffffffff0000ffffull) | ((unsigned long long)(0xffffu - (unsigned)lo) << 16);
          // the new place is inside e's tie group: one window around occ, unless the group is wider than that
          int cnt = 0;
          {
            const int wb = max(k, occ - 16), we = wb + 31;
            const bool lo_ok = (wb == k) || ((unsigned)(keys[wb] >> 32) > esc);
            const bool hi_ok = (we >= nc) || ((unsigned)(keys[we] >> 32) < esc);
            if (lo_ok && hi_ok) {
              const int idx = wb + lane;
              const bool gt = (idx < nc) && idx != occ && keys[idx] > nkey;
              cnt = (wb - k) + __popc(__ballot_sync(FULL, gt));
            } else {
              for (int base = k; base < nc; base += 32) {
                const int idx = base + lane;
                const bool gt = (idx < nc) && idx != occ && keys[idx] > nkey;
                const unsigned mask = __ballot_sync(FULL, gt);
                cnt += __popc(mask);
                const bool le = (idx < nc) && idx != occ && !gt;
                if (__any_sync(FULL, le)) break;             // sorted descending: nothing greater further on
              }
            }
          }
          const int ins = k + cnt;
          if (ins < occ) {
            // shift keys[ins .. occ-1] up by one, from the top end
            for (int top = occ; top > ins; top -= 32) {
              const int idx = top - lane;                     // destination index
              unsigned long long v = 0ull;
              if (idx > ins) v = keys[idx - 1];
              __syncwarp();
              if (idx > ins) keys[idx] = v;
              __syncwarp();
            }
          } else if (ins > occ) {
            // shift keys[occ+1 .. ins] down by one, from the bottom end
            for (int bot = occ; bot < ins; bot += 32) {
              const int idx = bot + lane;                     // destination index
              unsigned long long v = 0ull;
              if (idx < ins) v = keys[idx + 1];
              __syncwarp();
              if (idx < ins) keys[idx] = v;
              __syncwarp();
            }
          }
          if (lane == 0) {
            keys[ins] = nkey;
            unsigned *pp = pay + ((unsigned)nkey & 0xffffu);
            *pp = ((unsigned)x << 16) | (*pp & 0xffffu);        // home slot of the candidate
            if (x >= tail0 && x < m) { flags[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); multi[(x - tail0) >> 5] |= 1u << ((x - tail0) & 31); }
          }
          __syncwarp();
        }
      }
      // next flagged slot below b in this word (a re-insertion may have flagged one)
      bits = flags[w] & ((b == 0) ? 0u : ((1u << b) - 1u));
    }
  }
  return 1;
}

// ---- the bitonic network's stages with partner distance < SORT_TILE, inside a warp --------------------------------------
// A warp takes a tile of SORT_TILE consecutive keys into registers, key 32 r + l of the tile in register r of lane l (the
// loads and stores of a warp are consecutive 8-byte words): partner distance 64 and 32 is a compare-exchange between two
// registers of a lane, 16 … 1 one with lane l ^ j through a shuffle.  One load → stages → store pass and ONE block barrier
// run every stage (k, j) with k_lo <= k <= k_hi and j < SORT_TILE, where the strided form pays a barrier per stage.
// Descending where bit k of the key's index is clear, as in the strided stages.  Keys at index >= nc read as 0 (the
// padding up to np), keys at index >= np do not exist.  All threads call it; ends with the barrier.
constexpr int SORT_TILE = 128;
__device__ __forceinline__ void sort_cx(unsigned long long &a, unsigned long long &b, const bool desc) {
  if (desc ? (a < b) : (a > b)) { const unsigned long long t = a; a = b; b = t; }
}
__device__ __forceinline__ void sort_tile_pass(unsigned long long *keys, const int nc, const int np, const int k_lo, const int k_hi) {
  const int lane = threadIdx.x & 31;
  for (int i0 = (threadIdx.x >> 5) * SORT_TILE + lane; i0 - lane < np; i0 += (BEAM_THREADS >> 5) * SORT_TILE) {
    unsigned long long v[4];
#pragma unroll
    for (int r = 0; r < 4; r++) v[r] = (i0 + 32 * r < nc) ? keys[i0 + 32 * r] : 0ull;
    for (int k = k_lo; k <= k_hi; k <<= 1) {
      if (k >= 128) { sort_cx(v[0], v[2], (i0 & k) == 0); sort_cx(v[1], v[3], (i0 & k) == 0); }
      if (k >= 64) { sort_cx(v[0], v[1], (i0 & k) == 0); sort_cx(v[2], v[3], ((i0 + 64) & k) == 0); }
      for (int j = min(k >> 1, 16); j > 0; j >>= 1) {
        const bool low = ((lane & j) == 0);
#pragma unroll
        for (int r = 0; r < 4; r++) {
          const unsigned long long o = __shfl_xor_sync(0xffffffffu, v[r], j);
          const bool keep_max = (low == (((i0 + 32 * r) & k) == 0));
          if (keep_max == (o > v[r])) v[r] = o;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 4; r++) if (i0 + 32 * r < np) keys[i0 + 32 * r] = v[r];
  }
  __syncthreads();
}

__device__ int heap_select_closed(unsigned long long *heap, const int n, const int need, const float lose_below, const int maxt,
                                  unsigned long long *keys, const int key_cap, unsigned *pay, const int pay_cap,
                                  int *ordn, int *s_scratch /* [2] shared ints */) {
  const int tid = threadIdx.x;
  int relocated = 0;
  if (n >= 65536 || maxt >= 65536 || !(lose_below > -INFINITY)) return 0;
  // tail slots (the slots the extractions take their s from) that are the home of a candidate: one bit each, at the end of pay
  // (a second bit per slot: a re-inserted element has landed there as well)
  const int tail0 = n - need + 1, fwords = (need + 31) >> 5;
  unsigned *const flags = pay + pay_cap - fwords, *const multi = pay + pay_cap - 2 * fwords;
  const bool have_flags = (2 * fwords < pay_cap);
  if (tid == 0) { s_scratch[0] = 0; s_scratch[1] = 0; }
  if (have_flags) for (int i = tid; i < 2 * fwords; i += BEAM_THREADS) multi[i] = 0u;
  __syncthreads();
  // 1. candidates (a handle per candidate from a shared counter, one atomic per warp and pass)
  const int H = 31 - __clz(n);
  const int cap = min(min(key_cap, have_flags ? pay_cap - 2 * fwords : pay_cap), 65535);   // the flag words sit behind the payload
  for (int h0 = 1; h0 <= n; h0 += BEAM_THREADS) {
    const int h = h0 + tid;
    unsigned long long e = 0ull;
    bool is_c = false;
    if (h <= n) { e = heap[h]; is_c = (hval(e) >= lose_below); }
    const unsigned m = __ballot_sync(0xffffffffu, is_c);
    int base = 0;
    if ((tid & 31) == 0 && m) base = atomicAdd(&s_scratch[0], __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (is_c) {
      const int ci = base + __popc(m & ((1u << (tid & 31)) - 1u));
      if (ci < cap) {
        keys[ci] = ((unsigned long long)fkey(hval(e)) << 32) | (unsigned)ci;
        pay[ci] = ((unsigned)h << 16) | (unsigned)(e >> 32);
      }
    }
  }
  __syncthreads();
  const int nc = s_scratch[0];
  int np = 1; while (np < nc) np <<= 1;
  if (nc > cap || np > key_cap || nc < need) return 0;      // uniform: s_scratch[0] is read after the barrier
  const bool can_relocate = have_flags;
  // the pre-order position of each candidate's slot in the complete tree of n slots goes into its key: one candidate per
  // thread, so that the warps walk the root paths converged (inside the collection loop only the candidates' lanes would).
  // A level of the path costs 1, and where it turns right the left sibling's subtree (closed_subtree_size of it).
  for (int ci = tid; ci < nc; ci += BEAM_THREADS) {
    const int h = (int)(pay[ci] >> 16), d = 31 - __clz(h);
    int pre = d;
    for (int b = d - 1; b >= 0; b--) {
      if ((h >> b) & 1) {
        const int sh = H - (d - b), width = 1 << sh;
        pre += (width - 1) + max(0, min(n - ((((h >> b) ^ 1)) << sh) + 1, width));
      }
    }
    keys[ci] |= (unsigned long long)(0xffffu - (unsigned)pre) << 16;
  }
  __syncthreads();
  // 2. bitonic sort, descending: the stages inside a tile in one pass per run of them (the first pass also pads
  //    keys[nc..np) with zeros), the others one strided pass over the keys each
  sort_tile_pass(keys, nc, np, 2, min(np, SORT_TILE));
  for (int k = 2 * SORT_TILE; k <= np; k <<= 1) {
    for (int j = k >> 1; j >= SORT_TILE; j >>= 1) {
      for (int i = tid; i < (np >> 1); i += BEAM_THREADS) {
        const int a = ((i & ~(j - 1)) << 1) | (i & (j - 1)), b = a | j;
        const unsigned long long ka = keys[a], kb = keys[b];
        const bool desc = ((a & k) == 0);
        if (desc ? (ka < kb) : (ka > kb)) { keys[a] = kb; keys[b] = ka; }
      }
      __syncthreads();
    }
    sort_tile_pass(keys, np, np, k, k);
  }
  // 3. the test: which tail candidates may still be in their leaf when it is taken?  If slot p still held e at step
  //    k = n-p+1, the k-1 elements extracted so far and the d = depth(p) elements above p would all be ahead of e, so
  //    rank(e) >= k + d.  The rank of an element changes only when an element of its own score is re-inserted, so an untied
  //    e with rank < k + d is gone for sure, and a tied one if even the last place of its tie group is < k + d.  The others
  //    are flagged; if none of the flagged ties with anybody no re-insertion can matter (the plain closed form is exact).
  const unsigned theta = (unsigned)(keys[need - 1] >> 32);
  for (int i = tid; i < nc; i += BEAM_THREADS) {
    const unsigned long long ki = keys[i];
    const unsigned sk = (unsigned)(ki >> 32);
    if (sk < theta) continue;
    const int slot = (int)(pay[(unsigned)ki & 0xffffu] >> 16);
    if (slot < tail0) continue;
    const bool tied = (i > 0 && (unsigned)(keys[i - 1] >> 32) == sk) || (i + 1 < nc && (unsigned)(keys[i + 1] >> 32) == sk);
    int last = i;
    if (tied) { int g = 0; while (last + 1 < nc && (unsigned)(keys[last + 1] >> 32) == sk && g < 8) { last++; g++; } if (g == 8) last = nc; }
    const int kstep = n - slot + 1, d = 31 - __clz(slot);
    if (last + 1 < kstep + d) continue;
    if (have_flags) atomicOr(flags + ((slot - tail0) >> 5), 1u << ((slot - tail0) & 31));
    if (tied) s_scratch[1] = 1;
  }
  __syncthreads();
  if (s_scratch[1]) {
    // 3b. a tied tail element may still be in its leaf when the leaf is taken: follow the few re-insertions exactly on the
    //     implicit heap (closed_relocate); warp 0, the others wait
    if (!can_relocate) return 0;
    if (tid < 32) { const int ok = closed_relocate(keys, nc, n, need, flags, multi, pay, tid); if (tid == 0) s_scratch[1] = ok ? 2 : 1; }
    __syncthreads();
    if (s_scratch[1] != 2) return 0;
    relocated = 1;
  }
  // 4. survivors in visiting order: last extracted first
  for (int k = tid; k < need; k += BEAM_THREADS) ordn[k] = (int)(pay[(unsigned)keys[need - 1 - k] & 0xffffu] & 0xffffu);
  return 1 + relocated;
}


// trace_backptr (beam.c:253-301): the word ids of the atoms from `a` back to the sentence start, in sentence order, into
// w[0..MAX_WORDS); returns their count.  One thread.
__device__ int trace_backptr(const jb200_atom *atoms, int a, int *w) {
  int n = 0;
  w[n++] = atoms[a].wid;
  while (atoms[a].begintime > 0) {
    a = atoms[a].last;
    if (a < 0 || n >= MAX_WORDS) break;
    w[n++] = atoms[a].wid;
  }
  for (int i = 0; i < n / 2; i++) { const int x = w[i]; w[i] = w[n - 1 - i]; w[n - 1 - i] = x; }
  return n;
}

// bt_current_max (beam.c:876-921): the best trellis word among those stored in the frame just done (raw atoms lo..hi-1,
// end time frame-1), the most recently stored one on a tie (the reference walks its list newest first and keeps the
// first maximum), traced back to the sentence start.  One thread.
__device__ void interim_best(const BeamParams &p, const int u, const jb200_atom *araw, const int lo, const int hi, const int frame) {
  UttState *st = p.state + u;
  int best = -1; float mx = JB200_LOG_ZERO;
  for (int a = hi - 1; a >= lo; a--) if (mx < araw[a].backscore) { mx = araw[a].backscore; best = a; }
  st->interim_frame = frame - 1;
  if (best < 0) { st->interim_nwords = 0; st->interim_score = JB200_LOG_ZERO; return; }
  st->interim_nwords = trace_backptr(araw, best, p.interim_words + (size_t)u * MAX_WORDS); st->interim_score = mx;
}

// phase cycle accounting (thread 0 only; negligible cost)
#define PROF_MARK(k) do { if (tid == 0) { long long _n = clock64(); s_prof[k] += _n - s_tprev; s_tprev = _n; } } while (0)

// ---- the beam cut: sort_token_no_order (beam.c:1492-1520) of n > need = beam tokens ------------------------------
// heap[1..n] holds (token id << 32 | score bits); s_maxkey = fkey of the largest score among them.  Fills ordn[0..need)
// with the survivors in the reference's order: upward (need < n - need) the extracted maxima, last extracted first;
// downward what is left of the heap.  The node slots of the n tokens `tn` are dead from here on and are reset for the
// next frame on the side.  All threads call it; each thread's own ordn entries are written when it returns (no barrier).
__device__ __forceinline__ void beam_cut(const BeamParams &p, const CutAreas &ca, const int n, const unsigned &s_maxkey,
                                         const Tok *tn, const SlotView &slots, int *ordn, long long *s_prof, long long &s_tprev) {
  __shared__ unsigned s_losekey;
  __shared__ int s_cf[2];
  const int tid = threadIdx.x;
  const int need = p.beam, maxt = p.maxt;
  unsigned long long *const heap = ca.heap, *const outv = ca.outv();
  const SlotClear sc{tn, n, slots};
  if (need < n - need) {
    // lower bound of the need-th largest score from a 1024-bin histogram of the order-preserving keys (bin width ~0.5
    // in score units, adapted to the magnitude of the best score)
    constexpr int NB = 1024;
    int *hist = ca.offs;
    const int nb = min(NB, 2 * (p.beam + 2));
    for (int i = tid; i < nb; i += BEAM_THREADS) hist[i] = 0;
    __syncthreads();
    const unsigned maxkey = s_maxkey;
    const int e = (int)((((maxkey & 0x80000000u) ? (maxkey & 0x7fffffffu) : ~maxkey) >> 23) & 0xffu) - 127;
    const int sh = max(0, min(24, 22 - e));
    for (int r = tid; r < n; r += BEAM_THREADS) {
      const unsigned key = fkey(hval(heap[r + 1]));
      const unsigned bin = min((unsigned)(nb - 1), (maxkey - key) >> sh);
      atomicAdd(&hist[bin], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int cum = 0, found = -1;
      for (int b0 = 0; b0 < nb && found < 0; b0 += 32) {
        const int v = (b0 + tid < nb) ? hist[b0 + tid] : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (tid >= o) x += y; }
        const unsigned hit = __ballot_sync(0xffffffffu, cum + x >= need);
        if (hit) found = b0 + __ffs(hit) - 1;
        cum += __shfl_sync(0xffffffffu, x, 31);
      }
      if (tid == 0) {
        unsigned lk = 0u;
        if (found >= 0 && found < nb - 1) {
          const unsigned long long drop = (unsigned long long)(found + 1) << sh;
          lk = (drop < maxkey) ? maxkey - (unsigned)drop : 0u;
        }
        s_losekey = lk;
      }
    }
    __syncthreads();
    const unsigned lk = s_losekey;
    const float lose_below = (lk == 0u) ? -INFINITY : __uint_as_float((lk & 0x80000000u) ? (lk & 0x7fffffffu) : ~lk);
    heap_build<true>(heap, n); PROF_MARK(7);
    // closed form of the extraction order when no re-inserted element can matter (heap_select_closed), else the replay;
    // the node slots are reset before the sort
    sc.run(tid, BEAM_THREADS);
    const int closed = heap_select_closed(heap, n, need, lose_below, maxt, ca.gq ? ca.gq : heap + n + 1, ca.gq ? p.sort_cap : maxt + 3 - n,
                                          reinterpret_cast<unsigned *>(ca.offs), 2 * (p.beam + 2), ordn, s_cf);
    if (tid == 0) {
      atomicAdd(p.cut_counters + CUT_UPWARD, 1ull);
      if (closed) atomicAdd(p.cut_counters + CUT_CLOSED, 1ull);
      if (closed == 2) atomicAdd(p.cut_counters + CUT_RELOCATED, 1ull);
    }
    if (!closed) {
      heap_pad_sentinels<true>(heap, n, maxt);
      __syncthreads();
      heap_extract_fast<true>(ca, n, need, lose_below, maxt, p.cut_counters);
      for (int k = tid; k < need; k += BEAM_THREADS) ordn[k] = (int)(outv[need - 1 - k] >> 32);
    }
  } else {
    // downward: no loser cut, no closed form; the idle warps reset the node slots during the replay
    heap_pad_sentinels<false>(heap, n, maxt);
    heap_build<false>(heap, n); PROF_MARK(7);
    heap_extract_fast<false>(ca, n, n - need, -INFINITY, maxt, p.cut_counters, &sc);
    for (int k = tid; k < need; k += BEAM_THREADS) ordn[k] = (int)(heap[k + 1] >> 32);
  }
}

// finalize_1st_pass (bt_relocate_rw + bt_sort_rw, backtrellis.c:218-267,438-478) + find_1pass_result + trace_backptr; all
// three kernels end with it.  The pass-1 result is, for an N-gram (beam.c:394-424), the </s> atom of the latest end frame
// that holds one; for a grammar (beam.c:435-458), the best atom of the latest end frame that holds any, whatever its word.
// All threads call it.
template <bool GRAMMAR>
__device__ __forceinline__ void finalize_utt(const BeamParams &p, const int u, const int tid, const int T, jb200_atom *araw, int *newidx,
                                             const int *group0, jb200_utt_result *res, int *words,
                                             int &s_natoms, int &s_overflow, int &s_found, long long &s_outbase,
                                             long long *s_prof, long long &s_tprev) {
  // group g = atoms with end frame g (raw atoms are grouped by creation frame already);
  // inside a group order by word id (unique per group in this build: one token per node).
  const int natoms = s_natoms;
  for (int a = tid; a < natoms; a += BEAM_THREADS) {
    const jb200_atom me = araw[a];
    const int lo = group0[me.endtime], hi = group0[me.endtime + 1];
    int rank = 0;
    for (int b = lo; b < hi; b++) rank += (araw[b].wid < me.wid) ? 1 : 0;
    newidx[a] = lo + rank;
  }
  if (tid == 0) {
    if (p.atoms_in_place) s_outbase = p.atom_off[u];        // streams: each utterance keeps its own output region
    else {
      unsigned long long base = atomicAdd(p.atom_counter, (unsigned long long)natoms);
      if ((long long)(base + natoms) > p.atoms_out_cap) { s_overflow = 1; s_outbase = -1; }
      else s_outbase = (long long)base;
    }
  }
  __syncthreads();
  const long long ob = s_outbase;
  const bool can_write = (ob >= 0);
  const int kept = can_write ? natoms : 0;
  for (int a = tid; a < kept; a += BEAM_THREADS) {
    jb200_atom me = araw[a];
    me.last = (me.last < 0) ? -1 : newidx[me.last];
    p.atoms_out[ob + newidx[a]] = me;
    // the result's end frame
    if ((GRAMMAR || me.wid == p.tail_silwid) && me.backscore > JB200_LOG_ZERO) atomicMax(&s_found, me.endtime);
  }
  __threadfence_block();
  __syncthreads();

  if (tid == 0) {
    int status = 0, nw = 0; float score = 0.0f;
    const int last_time = s_found;
    if (kept == 0 || last_time < 0) status = -1;
    else {
      const jb200_atom *const atoms = p.atoms_out + ob;
      const int lo = group0[last_time], hi = group0[last_time + 1];
      int best = -1;
      if constexpr (GRAMMAR) {
        float maxscore = JB200_LOG_ZERO;
        for (int b = lo; b < hi; b++) {                    // rw[last_time][] order = word id order; strict '<' keeps the first maximum
          const jb200_atom x = atoms[b];
          if (maxscore < x.backscore) { maxscore = x.backscore; best = b; }
        }
      } else {
        for (int b = lo; b < hi; b++) {                    // the group's only </s> atom
          const jb200_atom x = atoms[b];
          if (x.wid == p.tail_silwid && x.backscore > JB200_LOG_ZERO) { best = b; break; }
        }
      }
      if (best < 0) status = -1;
      else { nw = trace_backptr(atoms, best, words); score = atoms[best].backscore; }
    }
    jb200_utt_result r;
    r.status = status; r.n_frames = T; r.n_atoms = kept; r.n_words = nw; r.score = score;
    r.atom_offset = ob; r.word_offset = u * MAX_WORDS; r.overflow = s_overflow;
    *res = r;
    PROF_MARK(7);
    if (p.prof) for (int k = 0; k < 8; k++) p.prof[(size_t)u * 8 + k] = s_prof[k];
  }
}

// ---- what the normal-tree and the multipath kernel share ------------------------------------------------------------
// Utterance u's part of the per-utterance work areas.  The isolated-root table is sized with the host's stride
// max(n_iso, n_isoarc, 1) (n_isoarc = 0 on normal trees).
struct UttAreas {
  Tok *tok0; int *ord0; SlotView slots; Cand *cand; CandB *candb; IsoCand *iso; WEnd *wend;
  Tok *surv;                            // normal trees: the survivors of the previous frame, in visiting order
  unsigned *bits; int *wpre;
  jb200_atom *araw; int *newidx; int atom_cap;
  int *group0;                          // [T+1]: first raw atom of end-frame group g
  int *counts; jb200_utt_result *res; int *words;
};
__device__ __forceinline__ UttAreas utt_areas(const BeamParams &p, const int u) {
  const int f_begin = p.frame_off[u];   // only addresses the work areas: a launch covers the frames its ChunkDesc names
  const long long a0 = p.atom_off[u];
  UttAreas a;
  a.tok0 = p.tok + (size_t)u * 2 * p.maxt;
  a.ord0 = p.order + (size_t)u * 2 * p.maxt;
  a.slots = SlotView{p.slots + (size_t)u * p.n_nodes};
  a.cand = p.cand + (size_t)u * p.maxc;
  a.candb = p.candb + (size_t)u * p.maxc;
  a.surv = p.surv + (size_t)u * (p.beam + 2);
  a.iso = p.iso + (size_t)u * max(max(p.n_iso, p.n_isoarc), 1);
  a.wend = p.wend + (size_t)u * p.maxw;
  a.bits = p.bitmask + (size_t)u * (p.maxbits >> 5);
  a.wpre = p.wordpre + (size_t)u * (p.maxbits >> 5);
  a.atom_cap = (int)(p.atom_off[u + 1] - a0);
  a.araw = p.atoms_raw + a0;
  a.newidx = p.newidx + a0;
  a.group0 = p.group0 + (size_t)f_begin + u;
  a.counts = p.counts + (size_t)f_begin * 2;
  a.res = p.results + u;
  a.words = p.words + (size_t)u * MAX_WORDS;
  return a;
}

// tid 0: the scalars a kernel keeps in shared memory, fresh at the utterance's first chunk, else as the last launch parked them
__device__ __forceinline__ void resume_scalars(const bool first, const UttState *ust, int &natoms, int &overflow, float &thr, int &ns,
                                               long long *prof) {
  if (first) { natoms = 0; overflow = 0; thr = JB200_LOG_ZERO; ns = 0; for (int k = 0; k < 8; k++) prof[k] = 0; }
  else { natoms = ust->natoms; overflow = ust->overflow; thr = ust->thr; ns = ust->ns; for (int k = 0; k < 8; k++) prof[k] = ust->prof[k]; }
}

// tid 0, at the end of a chunk that is not the utterance's last: park those scalars (everything else already lives in the
// utterance's global work area) and, when asked, the best partial sentence.  The word ends of frame T-1 were stored in
// frame T-1 (multipath: in half B of frame T-1), with end time T-2.
__device__ __forceinline__ void park_scalars(const BeamParams &p, const int u, const UttAreas &ua, const int T, const int natoms,
                                             const int overflow, const float thr, const int ns, const int cur, const int tnum_prev,
                                             const int stopped, const bool slots_clean, long long *prof, const long long tprev) {
  UttState *const ust = p.state + u;
  ust->natoms = natoms; ust->overflow = overflow; ust->thr = thr; ust->ns = ns; ust->cur = cur;
  ust->tnum_prev = tnum_prev; ust->stopped = stopped; ust->slots_clean = slots_clean ? 1 : 0;
  ust->t_done = T;
  long long _n = clock64(); prof[7] += _n - tprev;
  for (int k = 0; k < 8; k++) ust->prof[k] = prof[k];
  if (p.interim) interim_best(p, u, ua.araw, (T >= 2 && stopped < 0) ? ua.group0[T - 2] : natoms, natoms, T - 1);
}

// save_trellis (beam.c:2209): the trellis word of word-end token tk, ending at frame endtime
__device__ __forceinline__ jb200_atom trellis_atom(const Tok &tk, const int wid, const int endtime, const jb200_atom *araw) {
  jb200_atom a;
  a.wid = wid; a.backscore = tk.score;
  a.begintime = (tk.tre < 0 ? -1 : araw[tk.tre].endtime) + 1;
  a.endtime = endtime; a.last = tk.tre; a.lscore = tk.lscore;
  return a;
}

// Word-internal candidate k of token tk on node nr (beam_intra_word_core, beam.c:2004-2177): k = 0 the self-loop if there
// is one, then the arc to nr.next if there is one, then the explicit arcs.  Entering another node that carries a 1-gram
// factoring id replaces the token's LM term by the node's.  WITH_OUT: out = the destination node's output, read with
// scid as one 8-byte load.  The multipath kernel adds no output here and reads scid alone: the paired load made it
// 1.8 % slower on dnn60k_mp (H100 80GB HBM3, 400 W limit).
struct IntraArc { int next; float score, lscore; int out; };
template <bool WITH_OUT>
__device__ __forceinline__ IntraArc intra_arc(const BeamParams &p, const Tok &tk, const NodeRec &nr, const int k) {
  int next; float pa;
  const int has_self = (nr.self_a != JB200_LOG_ZERO), has_next = (nr.next_a != JB200_LOG_ZERO);
  if (has_self && k == 0) { next = tk.node; pa = nr.self_a; }
  else if (has_next && k == has_self) { next = nr.next; pa = nr.next_a; }
  else { const int a = k - has_self - has_next; next = __ldg(p.arc_to + nr.arc_off + a); pa = __ldg(p.arc_a + nr.arc_off + a); }
  float tmpsum = tk.score + pa;
  float lsc = JB200_LOG_ZERO;
  int out_next = nr.out;
  if (next != tk.node) {
    int scid;
    if constexpr (WITH_OUT) {
      const int2 so = __ldg(reinterpret_cast<const int2 *>(&p.nodes[next].scid));
      scid = so.x;
      out_next = so.y;
    } else scid = p.nodes[next].scid;
    if (scid != 0) {
      lsc = max_successor_prob(p, tk.cword, scid) * p.lm_weight + p.lm_penalty;
      tmpsum -= tk.lscore;
      tmpsum += lsc;
    }
  }
  if (lsc == JB200_LOG_ZERO) lsc = tk.lscore;
  return IntraArc{next, tmpsum, lsc, out_next};
}

// the word-internal candidates of a survivor on node nr that passes the score envelope: one per arc
__device__ __forceinline__ int arc_count(const NodeRec &nr) {
  return (nr.self_a != JB200_LOG_ZERO) + (nr.next_a != JB200_LOG_ZERO) + nr.arc_n;
}

// the survivor j < ns whose candidates offs[j] <= c < offs[j+1] include candidate c
__device__ __forceinline__ int cand_owner(const int *offs, const int ns, const int c) {
  int lo = 0, hi = ns;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (offs[mid] <= c) lo = mid; else hi = mid; }
  return lo;
}

// Arrival order (create_token numbering, beam.c:1147-1162).  Candidate `local` of source j arrives as seq_no(j, local);
// the first arrival at a node creates its token, and the best (the first of equals) gives it its content.  A creator
// sets the bit at its position in arrival order, and the tokens are numbered by the rank of their bits.
__device__ __forceinline__ unsigned seq_no(const int j, const int local) { return (unsigned)j * SEQ_LOCAL + (unsigned)local; }
__device__ __forceinline__ bool first_arrival(const SlotView &slots, const int node, const unsigned seq) {
  return (unsigned)__ldcg(slots.fs(node)) == seq;
}
__device__ __forceinline__ unsigned winner_seq(const SlotView &slots, const int node) {
  return ~(unsigned)(__ldcg(slots.bk(node)) & 0xffffffffu);
}
__device__ __forceinline__ void mark_creator(unsigned *bits, const int pos) { atomicOr(bits + (pos >> 5), 1u << (pos & 31)); }
// wbits = bits[pos >> 5]
__device__ __forceinline__ int creation_rank(const unsigned wbits, const int *wpre, const int pos) {
  return wpre[pos >> 5] + __popc(wbits & ((1u << (pos & 31)) - 1u));
}

// Word end tk on node stend at slot ai of the trellis (save_trellis, beam.c:2209, ending at frame endtime; save = false
// stores nothing and flags an overflow) and, when the word may be followed (is_tr), cross-word source wi: the survivor j,
// base = the score the next word starts from (beam.c:2306-2307: plus wordend_a, WORDEND_A, except on multipath trees),
// and the first isolated-root candidate at nintra.  The best source goes to *webest; beam.c:2308 keeps the FIRST maximum.
// (wordend_a is read here, not by the caller: read before the branches, it delays the caller's token loads.)
template <bool WORDEND_A>
__device__ __forceinline__ void word_end(const BeamParams &p, const UttAreas &ua, const Tok &tk, const int stend,
                                         const int endtime, const bool save, const int ai, const bool is_tr, const int wi,
                                         const int j, const int nintra, unsigned long long *webest,
                                         int *overflow) {
  if (save && ai < ua.atom_cap) ua.araw[ai] = trellis_atom(tk, stend, endtime, ua.araw);
  else *overflow = 1;
  if (!is_tr) return;
  if (wi < p.maxw && ai < ua.atom_cap) {
    WEnd w;
    const int transp = p.is_transp[stend];
    w.j = j; w.atom = ai; w.last_word = transp ? tk.cword : stend;
    w.base = tk.score;
    if constexpr (WORDEND_A) w.base += __ldg(p.wordend_a + stend);
    w.transp2 = (transp && tk.cword >= 0 && p.is_transp[tk.cword]) ? 1 : 0;
    w.nintra = nintra;
    ua.wend[wi] = w;
    if (w.base > JB200_LOG_ZERO) atomicMax(webest, ((unsigned long long)fkey(w.base) << 32) | (unsigned)(~(unsigned)wi));
  } else *overflow = 1;
}

// the score word end w hands to the next word with LM term lsc (beam.c:2430-2442, :2574-2578)
__device__ __forceinline__ float cross_word_score(const BeamParams &p, const WEnd &w, const float lsc) {
  float tmpsum = w.base;
  tmpsum += lsc;
  if (w.transp2) tmpsum += p.lm_penalty_trans;
  return tmpsum;
}

// Cross-word transitions into isolated root col (beam_inter_word, beam.c:2336-2500), pre-reduced over the word ends
// wend[0..E) in visiting order: the first that reaches it and the best (the first maximum).  ROOT_ARC: a multipath
// tree's root carries no output, and the candidate lands on a successor of the root through an arc of score pa.
template <bool GRAMMAR, bool ROOT_ARC>
__device__ __forceinline__ IsoCand reduce_word_ends(const BeamParams &p, const WEnd *wend, const int E, const int col, const float pa) {
  float best = JB200_LOG_ZERO, bestl = 0.0f; int beste = -1, firste = -1;
  for (int e = 0; e < E; e++) {
    const WEnd w = wend[e];
    float lsc;
    if constexpr (GRAMMAR) {
      // category-pair constraint of (ending word, root's word) and the insertion penalty (beam.c:2404-2411, :2444-2450)
      if (!__ldg(p.cp_allowed + (size_t)w.last_word * p.n_iso + col)) continue;
      lsc = p.penalty1 + __ldg(p.cprob + w.last_word);
    } else {
      const float tmpprob = __ldg(p.iw + (size_t)w.last_word * p.n_iso + col);
      lsc = tmpprob * p.lm_weight + p.lm_penalty;
    }
    float v = cross_word_score(p, w, lsc);
    if constexpr (ROOT_ARC) v = v + pa;
    if (v > JB200_LOG_ZERO) {
      if (firste < 0) firste = e;
      if (beste < 0 || best < v) { best = v; beste = e; bestl = lsc; }
    }
  }
  IsoCand ic; ic.score = best; ic.e = beste; ic.lscore = bestl; ic.first_e = firste;
  return ic;
}

// 1-gram factoring (beam_inter_word_factoring, beam.c:2549-2616): the score the best word end wb gives shared root i,
// and in lsc its LM term
__device__ __forceinline__ float factoring_score(const BeamParams &p, const WEnd &wb, const int i, float &lsc) {
  lsc = __ldg(p.shared_f + i) * p.lm_weight + p.lm_penalty;
  return cross_word_score(p, wb, lsc);
}

// what a token entering the next word from word end w carries of it
__device__ __forceinline__ void enter_from(Tok &nt, const WEnd &w, const jb200_atom *araw) {
  nt.tre = w.atom; nt.cword = w.last_word; nt.tre_wid = araw[w.atom].wid;
}

// init_nodescore, N-gram (beam.c:1631-1665): the frame-0 token on the head silence nr = nodes[head_node], before any output
__device__ __forceinline__ Tok head_token(const BeamParams &p, const NodeRec &nr) {
  Tok tk;
  float ll = (nr.scid != 0) ? max_successor_prob(p, -1, nr.scid) : 0.0f;
  ll = ll * p.lm_weight + p.lm_penalty;
  tk.lscore = ll; tk.tre = -1; tk.cword = -1; tk.tre_wid = -1; tk.node = p.head_node; tk.score = ll;
  return tk;
}

// creation order (create_token numbering, beam.c:1147-1162): wpre[w] = the creators marked in bits[0..w); returns their
// total.  All threads call it; no barrier after the last wpre write (none at all when nwords == 0).
__device__ __forceinline__ int rank_creators(const unsigned *bits, int *wpre, const int nwords, int *s_warp) {
  int carry = 0;
  for (int w0 = 0; w0 < nwords; w0 += BEAM_THREADS) {
    const int w = w0 + (int)threadIdx.x;
    const int cnt = (w < nwords) ? __popc(__ldcg(bits + w)) : 0;
    int tot;
    const int ex = block_excl_scan(cnt, s_warp, &tot);
    if (w < nwords) wpre[w] = carry + ex;
    carry += tot;
  }
  return carry;
}

// tid 0, end of frame t: its created and surviving token counts, and the next frame's score envelope (the best score
// created in the frame less prune_width; LOG_ZERO when off or when nothing was created)
__device__ __forceinline__ void end_frame(const BeamParams &p, int *counts, const int t, const int ncre, const int ns_new,
                                          const unsigned pmaxkey, int &ns, float &thr) {
  counts[2 * t] = ncre; counts[2 * t + 1] = ns_new;
  ns = ns_new;
  if (p.prune_width >= 0.0f && pmaxkey != 0u) {
    const unsigned b = (pmaxkey & 0x80000000u) ? (pmaxkey & 0x7fffffffu) : ~pmaxkey;
    thr = __uint_as_float(b) - p.prune_width;
  } else thr = JB200_LOG_ZERO;
}

// Self-check of a heap select (JB200_CHECK_HEAP, compiled into the CHECK instantiations of the kernels only): the plain
// sequential select (heap_build + heap_extract_seq) of the select's input chk[1..n], compared with what the kernel made --
// the whole arrangement heap[1..n] (multipath select #1: select #2 starts from it), or, with heap == nullptr, the survivors
// in visiting order ordn[0..need) (the normal kernels' cut, multipath select #2).  Overflow code 4 on a difference.  With
// tok != nullptr the input is first rebuilt from the tokens in creation order (chk may then be the cut's own heap array,
// dead after the cut).  With overflow == nullptr it only copies heap[1..n] to chk (the input of multipath select #2, which
// the cut destroys).  All threads call it.
__device__ __noinline__ void check_select(unsigned long long *chk, const int n, const int need, const Tok *tok,
                                          const unsigned long long *heap, const int *ordn, int *overflow) {
  if (!overflow) {
    for (int h = 1 + (int)threadIdx.x; h <= n; h += BEAM_THREADS) chk[h] = heap[h];
    __syncthreads();
    return;
  }
  const bool upward = (need < n - need);
  __syncthreads();
  if (tok) for (int r = threadIdx.x; r < n; r += BEAM_THREADS) chk[r + 1] = ((unsigned long long)(unsigned)r << 32) | __float_as_uint(tok[r].score);
  __syncthreads();
  if (upward) { heap_build<true>(chk, n); heap_extract_seq<true>(chk, n, need); }
  else { heap_build<false>(chk, n); heap_extract_seq<false>(chk, n, n - need); }
  bool bad = false;
  if (heap) {
    for (int h = 1 + (int)threadIdx.x; h <= n; h += BEAM_THREADS) bad |= (chk[h] != heap[h]);
  } else {
    const int start = upward ? n - need : 0;
    for (int k = threadIdx.x; k < need; k += BEAM_THREADS) bad |= (ordn[k] != (int)(chk[start + k + 1] >> 32));
  }
  if (bad) *overflow = 4;
  __syncthreads();
}

// ---- the kernel ------------------------------------------------------------------------------------
static constexpr int BEAM_MINBLOCKS = 4;
// The normal-tree kernel, for an N-gram (1-gram factoring, bigram rows) or, GRAMMAR, a DFA grammar on the category tree.
// The grammar differs in three places: the frame-0 tokens, the inter-word LM term and the pass-1 result (finalize_utt).
// CHECK: the JB200_CHECK_HEAP build (the self-check stays out of the shipped kernels' register budget).
template <bool GRAMMAR, bool CHECK>
__global__ void __launch_bounds__(BEAM_THREADS, BEAM_MINBLOCKS)
beam_kernel(const BeamParams p) {
  const int u = blockIdx.x;
  const int tid = threadIdx.x;
  // this launch covers frames [ck.t0, ck.t1) of the utterance (ChunkDesc)
  const ChunkDesc ck = p.chunk[u];
  if (ck.flags & CHUNK_SKIP) return;
  const bool ck_first = (ck.flags & CHUNK_FIRST) != 0, ck_final = (ck.flags & CHUNK_FINAL) != 0;
  const UttState *const ust = p.state + u;
  const int T = ck.t1;                               // frames so far; the utterance's length when ck_final
  const int MAXT = p.maxt, MAXC = p.maxc, MAXW = p.maxw;

  const CutAreas ca = cut_areas(p);
  unsigned long long *const heap = ca.heap;
  int *const offs = ca.offs;                          // [beam+2] candidate payload offsets per survivor
  int *const poff = offs + (p.beam + 2);              // [beam+2] arrival-order bit positions per survivor
  __shared__ int s_warp[NWARP + 1];
  __shared__ int s_E, s_natoms, s_ns, s_overflow, s_found;
  __shared__ unsigned s_pmaxkey;
  __shared__ unsigned long long s_webest;
  __shared__ float s_thr;
  __shared__ long long s_outbase;
  __shared__ long long s_prof[8], s_tprev;

  const UttAreas ua = utt_areas(p, u);

  if (tid == 0) {
    s_found = -1; s_tprev = clock64();
    resume_scalars(ck_first, ust, s_natoms, s_overflow, s_thr, s_ns, s_prof);
  }
  __syncthreads();

  if constexpr (GRAMMAR) {
  // ================= frame 0: init_nodescore, grammar branch (beam.c:1669-1760): one token per sentence-initial
  // word (duplicates of a shared first node were dropped when the list was made); n_init <= beam, so the first
  // sort_token_no_order (:1883) leaves them in creation order
  if (T > 0 && ck_first) {
    const float *row0 = p.rows + (size_t)ck.row_base * p.row_stride;
    for (int i = tid; i < p.n_init; i += BEAM_THREADS) {
      const int node = __ldg(p.init_node + i);
      Tok tk;
      tk.lscore = __ldg(p.init_lscore + i); tk.tre = -1; tk.cword = -1; tk.tre_wid = -1; tk.node = node;
      tk.score = outprob_style(p, row0, p.nodes[node].out, -1) + tk.lscore;
      ua.tok0[i] = tk;
      ua.surv[i] = tk;
      ua.ord0[i] = i;
    }
    if (tid == 0) { s_ns = p.n_init; ua.counts[0] = p.n_init; ua.counts[1] = p.n_init; }
  }
  } else {
  // ================= frame 0: init_nodescore (beam.c:1631-1665) + first sort (:1883) =================
  if (T > 0 && ck_first && tid == 0) {
    const NodeRec nr = p.nodes[p.head_node];
    Tok tk = head_token(p, nr);
    tk.score += outprob_style(p, p.rows + (size_t)ck.row_base * p.row_stride, nr.out, -1);
    ua.tok0[0] = tk;
    ua.surv[0] = tk;
    ua.ord0[0] = 0;
    s_ns = 1;
    ua.counts[0] = 1; ua.counts[1] = 1;
  }
  }
  __syncthreads();

  int tnum_prev = ck_first ? ((T > 0) ? (GRAMMAR ? p.n_init : 1) : 0) : ust->tnum_prev;      // tokens created in the previous frame (clear phase)
  int stopped = ck_first ? -1 : ust->stopped;       // frame at which the beam ran empty (beam.c:3012-3015), -1 = alive
  bool slots_clean = ck_first ? false : (ust->slots_clean != 0);   // the previous frame's node slots were already reset under its beam cut

  // ================= frames 1..T-1: get_back_trellis_proceed (beam.c:2663-3019) =================
  for (int t = max(ck.t0, 1); t < T && stopped < 0; t++) {
    // one token list is enough here: the survivors of t-1 live on in `ua.surv` (compact, in visiting order), so frame t's
    // tokens may overwrite frame t-1's -- half the per-utterance token footprint in L2 (the multipath kernel still
    // reads the old list through its order array and keeps two)
    Tok *const tn = ua.tok0;
    int *const ordn = ua.ord0;
    const int ns = s_ns;
    const float thr = s_thr;
    const float *row = p.rows + (size_t)((long long)ck.row_base + t) * p.row_stride;

    // ---- P0: clear_tokens (beam.c:1122): reset the node slots used by frame t-1 (normally done already
    //          under that frame's beam cut, see beam_cut)
    if (!slots_clean) SlotClear{ua.tok0, tnum_prev, ua.slots}.run(tid, BEAM_THREADS);
    slots_clean = false;
    if (tid == 0) { s_webest = 0ull; s_pmaxkey = 0u; ua.group0[t - 1] = s_natoms; }
    __syncthreads();
    PROF_MARK(0);

    // ---- P1: per survivor: candidate counts, word ends, trellis atoms (save_trellis, beam.c:2209)
    int cand_total, nbits;
    {
      int carry_c = 0, carry_a = s_natoms, carry_w = 0;
      for (int j0 = 0; j0 < ns; j0 += BEAM_THREADS) {
        const int j = j0 + tid;
        int nin = 0, is_we = 0, is_tr = 0;
        Tok tk; NodeRec nr;
        if (j < ns) {
          tk = ua.surv[j];
          nr = p.nodes[tk.node];
          if ((tk.score > JB200_LOG_ZERO) && !(tk.score < thr)) {
            nin = arc_count(nr);
            if (nr.stend >= 0) { is_we = 1; is_tr = (nr.stend != p.tail_silwid); }
          }
        }
        int tot_c, tot_a, tot_w;
        const int oc = block_excl_scan(nin, s_warp, &tot_c);
        const int oa = block_excl_scan(is_we, s_warp, &tot_a);
        const int ow = block_excl_scan(is_tr, s_warp, &tot_w);
        if (j < ns) {
          offs[j] = carry_c + oc;
          // arrival-order position of this survivor's first candidate: its word-internal arcs,
          // then (for a word end that may continue) one slot per isolated root
          poff[j] = carry_c + oc + (carry_w + ow) * p.n_iso;
          if (is_we)
            word_end<true>(p, ua, tk, nr.stend, t - 1, true, carry_a + oa, is_tr, carry_w + ow, j, nin, &s_webest, &s_overflow);
        }
        carry_c += tot_c; carry_a += tot_a; carry_w += tot_w;
      }
      cand_total = carry_c;
      nbits = carry_c + carry_w * p.n_iso + p.n_shared;
      if (tid == 0) { offs[ns] = carry_c; poff[ns] = carry_c + carry_w * p.n_iso; s_natoms = min(carry_a, ua.atom_cap); s_E = min(carry_w, MAXW); }
      // carry_a > atom_cap: some word ends got no atom and no wend entry, and wend[0..E) would hold stale entries
      if (cand_total > MAXC || carry_w > MAXW || nbits > p.maxbits || carry_a > ua.atom_cap) { if (tid == 0) s_overflow = 1; cand_total = 0; nbits = 0; }
    }
    const int nwords = (nbits + 31) >> 5;
    for (int w = tid; w < nwords; w += BEAM_THREADS) ua.bits[w] = 0u;
    __syncthreads();
    PROF_MARK(1);
    const int E = (nbits > 0) ? s_E : 0;

    // ---- P2a: word-internal transitions (beam_intra_word(_core), beam.c:2004-2177), one thread per
    //           candidate (survivors near the tree roots fan out 10-20 ways: per-survivor loops leave most
    //           of the block idle); the owner of candidate c is found by bisection of the offsets
    for (int c = tid; c < cand_total; c += BEAM_THREADS) {
      const int j = cand_owner(offs, ns, c);
      const int k = c - offs[j];
      const Tok tk = ua.surv[j];
      const IntraArc ar = intra_arc<true>(p, tk, p.nodes[tk.node], k);
      Cand cd; cd.score = ar.score; cd.node = ar.next; cd.lscore = ar.lscore; cd.src = j;
      ua.cand[c] = cd;
      CandB cb; cb.tre = tk.tre; cb.cword = tk.cword; cb.tre_wid = tk.tre_wid; cb.out = ar.out;
      ua.candb[c] = cb;
      if (ar.score > JB200_LOG_ZERO) cand_atomics(ua.slots, ar.next, ar.score, seq_no(j, k), seq_no(j, k));
    }
    // ---- P2b: cross-word transitions into isolated roots (beam_inter_word, beam.c:2271-2517),
    //           pre-reduced per root over this frame's word ends, visited in survivor order
    for (int i = tid; i < p.n_iso; i += BEAM_THREADS) {
      const IsoCand ic = reduce_word_ends<GRAMMAR, false>(p, ua.wend, E, __ldg(p.iso_id + i), 0.0f);
      ua.iso[i] = ic;
      if (ic.first_e >= 0) {
        const WEnd wf = ua.wend[ic.first_e], wb = ua.wend[ic.e];
        cand_atomics(ua.slots, __ldg(p.iso_node + i), ic.score, seq_no(wf.j, wf.nintra + i), seq_no(wb.j, wb.nintra + i));
      }
    }
    // ---- P2c: best word end -> shared (1-gram factored) roots (beam_inter_word_factoring, :2549-2616)
    const unsigned long long webest = s_webest;
    const bool have_we = (webest != 0ull) && (nbits > 0);
    WEnd wbest; wbest.base = 0.0f; wbest.atom = -1; wbest.last_word = -1; wbest.transp2 = 0; wbest.j = 0; wbest.nintra = 0;
    if (have_we) {
      wbest = ua.wend[(unsigned)(~(unsigned)(webest & 0xffffffffu))];
      for (int i = tid; i < p.n_shared; i += BEAM_THREADS) {
        float lsc;
        const float tmpsum = factoring_score(p, wbest, i, lsc);
        if (tmpsum < thr) continue;
        if (tmpsum > JB200_LOG_ZERO) cand_atomics(ua.slots, __ldg(p.shared_node + i), tmpsum, seq_no(ns, i), seq_no(ns, i));
      }
    }
    __syncthreads();
    PROF_MARK(2);

    // ---- P3: creators = candidates that were the first to reach their node; one bit each at the
    //          candidate's position in sequential arrival order
    for (int c = tid; c < cand_total; c += BEAM_THREADS) {
      const Cand cd = ua.cand[c];
      if (!(cd.score > JB200_LOG_ZERO)) continue;
      const int k = c - offs[cd.src];
      if (first_arrival(ua.slots, cd.node, seq_no(cd.src, k))) mark_creator(ua.bits, poff[cd.src] + k);
    }
    for (int i = tid; i < p.n_iso; i += BEAM_THREADS) {
      const IsoCand ic = ua.iso[i];
      if (ic.first_e < 0) continue;
      const WEnd wf = ua.wend[ic.first_e];
      if (first_arrival(ua.slots, __ldg(p.iso_node + i), seq_no(wf.j, wf.nintra + i))) mark_creator(ua.bits, poff[wf.j] + wf.nintra + i);
    }
    if (have_we) {
      for (int i = tid; i < p.n_shared; i += BEAM_THREADS)
        if (first_arrival(ua.slots, __ldg(p.shared_node + i), seq_no(ns, i))) mark_creator(ua.bits, poff[ns] + i);
    }
    __syncthreads();
    PROF_MARK(3);

    // ---- P4: creation order = rank of the set bits
    int ncre = rank_creators(ua.bits, ua.wpre, nwords, s_warp);
    if (ncre > MAXT) { if (tid == 0) s_overflow = 1; ncre = 0; }
    __syncthreads();
    PROF_MARK(4);

    // ---- P5: materialise tokens with the winner's content, add the output probability (beam.c:2944)
    auto materialise = [&](int pos, int node) {
      const unsigned wbits = __ldcg(ua.bits + (pos >> 5));
      if (!((wbits >> (pos & 31)) & 1u)) return;
      const int r = creation_rank(wbits, ua.wpre, pos);
      const unsigned seqw = winner_seq(ua.slots, node);
      const int j = (int)(seqw >> SEQ_LOCAL_BITS), local = (int)(seqw & (SEQ_LOCAL - 1));
      Tok nt; nt.node = node;
      int out;
      if (j == ns) {                                    // factoring pass
        nt.score = factoring_score(p, wbest, local, nt.lscore);
        enter_from(nt, wbest, ua.araw);
        out = p.nodes[node].out;
      } else {
        const int c0 = offs[j], nin = offs[j + 1] - c0;
        if (local < nin) {                              // word-internal candidate: everything travels with it
          const Cand cd = ua.cand[c0 + local];
          const CandB cb = ua.candb[c0 + local];
          nt.score = cd.score; nt.lscore = cd.lscore; nt.tre = cb.tre; nt.cword = cb.cword; nt.tre_wid = cb.tre_wid;
          out = cb.out;
        } else {                                        // isolated-root candidate
          const IsoCand ic = ua.iso[local - nin];
          const WEnd w = ua.wend[ic.e];
          nt.score = ic.score; nt.lscore = ic.lscore;
          enter_from(nt, w, ua.araw);
          out = p.nodes[node].out;
        }
      }
      nt.score += outprob_style(p, row, out, nt.tre_wid);
      tn[r] = nt;
      heap[r + 1] = ((unsigned long long)(unsigned)r << 32) | __float_as_uint(nt.score);
      atomicMax(&s_pmaxkey, fkey(nt.score));
    };
    if (ncre > 0) {
      for (int c = tid; c < cand_total; c += BEAM_THREADS) {
        const Cand cd = ua.cand[c];
        if (!(cd.score > JB200_LOG_ZERO)) continue;
        materialise(poff[cd.src] + (c - offs[cd.src]), cd.node);
      }
      for (int i = tid; i < p.n_iso; i += BEAM_THREADS) {
        const IsoCand ic = ua.iso[i];
        if (ic.first_e < 0) continue;
        const WEnd wf = ua.wend[ic.first_e];
        materialise(poff[wf.j] + wf.nintra + i, __ldg(p.iso_node + i));
      }
      if (have_we)
        for (int i = tid; i < p.n_shared; i += BEAM_THREADS) materialise(poff[ns] + i, __ldg(p.shared_node + i));
    }
    __syncthreads();
    PROF_MARK(5);

    // ---- P6: beam cut = the reference's heap select (sort_token_no_order, beam.c:1492-1520)
    const int ns_new = min(ncre, p.beam);
    if (ncre <= p.beam) {
      for (int k = tid; k < ns_new; k += BEAM_THREADS) ordn[k] = k;
    } else {
      beam_cut(p, ca, ncre, s_pmaxkey, tn, ua.slots, ordn, s_prof, s_tprev);
      slots_clean = true;
      // the heap array is dead after the cut: the self-check rebuilds its input there
      if constexpr (CHECK) check_select(heap, ncre, p.beam, tn, nullptr, ordn, &s_overflow);
    }
    // the survivors in visiting order, compact (every thread re-reads the order entries it wrote itself)
    for (int k = tid; k < ns_new; k += BEAM_THREADS) ua.surv[k] = tn[ordn[k]];
    PROF_MARK(6);
    if (tid == 0) end_frame(p, ua.counts, t, ncre, ns_new, s_pmaxkey, s_ns, s_thr);
    tnum_prev = ncre;
    __syncthreads();
    if (ncre == 0) { stopped = t; break; }      // beam.c:3012-3015: no nodes left, search terminated
  }

  if (!ck_final) {
    if (tid == 0) park_scalars(p, u, ua, T, s_natoms, s_overflow, s_thr, s_ns, 0, tnum_prev, stopped, slots_clean, s_prof, s_tprev);
    return;
  }
  const int groups = (stopped >= 0) ? stopped : T;   // number of end-frame groups kept by finalize (framelen)

  // ================= get_back_trellis_end (normal version, beam.c:3076-3086) =================
  {
    const int ns = (T > 0) ? s_ns : 0;
    if (tid == 0 && T > 0 && groups == T) ua.group0[T - 1] = s_natoms;
    __syncthreads();
    int carry_a = s_natoms;
    for (int j0 = 0; j0 < ns; j0 += BEAM_THREADS) {
      const int j = j0 + tid;
      int is_we = 0; Tok tk; int stend = -1;
      if (j < ns) { tk = ua.surv[j]; stend = p.nodes[tk.node].stend; is_we = (stend >= 0); }
      int tot;
      const int oa = block_excl_scan(is_we, s_warp, &tot);
      if (is_we) {
        const int ai = carry_a + oa;
        if (ai < ua.atom_cap) ua.araw[ai] = trellis_atom(tk, stend, T - 1, ua.araw);     // save_trellis(t = samplenum)
        else s_overflow = 1;
      }
      carry_a += tot;
    }
    if (tid == 0) { s_natoms = min(carry_a, ua.atom_cap); ua.group0[groups] = s_natoms; }
    // leave the node slots clean for the next utterance that uses this work area
    if (!slots_clean) SlotClear{ua.tok0, tnum_prev, ua.slots}.run(tid, BEAM_THREADS);
    __syncthreads();
  }

  finalize_utt<GRAMMAR>(p, u, tid, T, ua.araw, ua.newidx, ua.group0, ua.res, ua.words, s_natoms, s_overflow, s_found, s_outbase, s_prof, s_tprev);
}

// ---- the multipath kernel ----------------------------------------------------------------------------
// get_back_trellis_proceed, MULTIPATH branch (beam.c:2752-2828, :2930-2941).  Trees of multipath models
// carry non-emitting word-begin / word-end nodes, and a frame runs in two halves:
//   A  word-internal transitions of the survivors of t-1 (no output probability yet), then the beam cut
//      (heap select #1) on the bare transition scores;
//   B  the word-end tokens among THOSE survivors are stored as trellis words and expanded across words
//      into the same frame's token set (onto the successors of the roots); then the output probabilities
//      of all emitting tokens are added and the beam is cut again (heap select #2).
// Select #2 runs on the token index array exactly as select #1 left it (remaining heap + extracted tail)
// with the tokens of half B appended, so select #1 is replayed in full, in place -- no loser cut there.
// Half B reuses the per-node slots: a token made in half A keeps the slot with firstseq = id - 2^30 (< 0:
// "exists") and bestkey = (score, seq 0), so later arrivals only replace its content when strictly better.
template <bool MAXHEAP>
__device__ __forceinline__ int select_exact(const CutAreas &ca, int n, int need, int *ordn, int maxt, unsigned long long *stats) {
  // sort_token_no_order (beam.c:1492-1520) replayed in full; the extracted roots are put back into the
  // tail slots where the in-place algorithm leaves them (k-th extracted at slot n-k).  Returns the first
  // survivor's slot.
  unsigned long long *const heap = ca.heap, *const outv = ca.outv();
  const int extract = MAXHEAP ? need : n - need;
  heap_pad_sentinels<MAXHEAP>(heap, n, maxt);
  heap_build<MAXHEAP>(heap, n);
  heap_extract_fast<MAXHEAP>(ca, n, extract, -INFINITY, maxt, stats);
  for (int k = threadIdx.x; k < extract; k += BEAM_THREADS) heap[n - k] = outv[k];
  __syncthreads();
  const int start = MAXHEAP ? n - need : 0;
  for (int k = threadIdx.x; k < need; k += BEAM_THREADS) ordn[k] = (int)(heap[start + k + 1] >> 32);
  return start;
}

static constexpr int TOK_EXISTS = 0x40000000;

// CHECK: the JB200_CHECK_HEAP build of the kernel (the self-check stays out of the shipped kernel's register budget)
template <bool CHECK>
__global__ void __launch_bounds__(BEAM_THREADS, BEAM_MINBLOCKS)
beam_kernel_mp(const BeamParams p) {
  const int u = blockIdx.x;
  const int tid = threadIdx.x;
  // this launch covers frames [ck.t0, ck.t1) of the utterance (ChunkDesc)
  const ChunkDesc ck = p.chunk[u];
  if (ck.flags & CHUNK_SKIP) return;
  const bool ck_first = (ck.flags & CHUNK_FIRST) != 0, ck_final = (ck.flags & CHUNK_FINAL) != 0;
  const UttState *const ust = p.state + u;
  const int T = ck.t1;                               // frames so far; the utterance's length when ck_final
  const int MAXT = p.maxt, MAXC = p.maxc, MAXW = p.maxw;

  const CutAreas ca = cut_areas(p);
  unsigned long long *const heap = ca.heap;
  int *const offs = ca.offs;                           // [beam+2] candidate offsets per survivor
  __shared__ int s_warp[NWARP + 1];
  __shared__ int s_E, s_natoms, s_ns, s_cur, s_overflow, s_found;
  __shared__ unsigned s_pmaxkey, s_hmaxkey;
  __shared__ unsigned long long s_webest;
  __shared__ float s_thr;
  __shared__ long long s_outbase;
  __shared__ long long s_prof[8], s_tprev;

  const UttAreas ua = utt_areas(p, u);

  if (tid == 0) {
    s_found = -1; s_tprev = clock64();
    resume_scalars(ck_first, ust, s_natoms, s_overflow, s_thr, s_ns, s_prof);
    s_cur = ck_first ? 0 : ust->cur;
  }
  __syncthreads();

  // init_nodescore (beam.c:1631-1665): the word-begin node of <s> has no output (:1654-1656)
  if (T > 0 && ck_first && tid == 0) {
    ua.tok0[0] = head_token(p, p.nodes[p.head_node]);
    ua.ord0[0] = 0;
    s_ns = 1;
  }
  __syncthreads();

  int tnum_prev = ck_first ? ((T > 0) ? 1 : 0) : ust->tnum_prev;
  int stopped = ck_first ? -1 : ust->stopped;       // frame at which the beam ran empty (beam.c:3012-3015), -1 = alive
  int n_left = 0;             // tokens of the unfinished (final) frame whose node slots are still set
  bool slots_clean = ck_first ? false : (ust->slots_clean != 0);   // the previous frame's node slots were already reset under its second beam cut

  // frames 0..T-1 (pass1.c:239-245 calls proceed(0) right after init), then proceed(T, final) (beam.c:3066-3072)
  const int t_last = ck_final ? T : T - 1;
  for (int t = ck.t0; t <= t_last && T > 0 && stopped < 0; t++) {
    const bool final = (t == T);
    const int cur = s_cur, nxt = cur ^ 1;
    Tok *tl = ua.tok0 + (size_t)cur * MAXT, *tn = ua.tok0 + (size_t)nxt * MAXT;
    int *ordl = ua.ord0 + (size_t)cur * MAXT, *ordn = ua.ord0 + (size_t)nxt * MAXT;
    const int ns = s_ns;
    const float thr = s_thr;
    const float *row = final ? p.rows : p.rows + (size_t)((long long)ck.row_base + t) * p.row_stride;   // the final half frame reads no scores

    // ---- P0: clear_tokens (normally done already under the previous frame's select #2)
    if (!slots_clean) SlotClear{tl, tnum_prev, ua.slots}.run(tid, BEAM_THREADS);
    slots_clean = false;
    if (tid == 0) { s_webest = 0ull; s_pmaxkey = fkey(JB200_LOG_ZERO); s_hmaxkey = 0u; if (t > 0) ua.group0[t - 1] = s_natoms; }
    __syncthreads();
    PROF_MARK(0);

    // ---- A1: candidate counts per survivor
    int cand_total;
    {
      int carry_c = 0;
      for (int j0 = 0; j0 < ns; j0 += BEAM_THREADS) {
        const int j = j0 + tid;
        int nin = 0;
        if (j < ns) {
          const Tok tk = tl[ordl[j]];
          const NodeRec nr = p.nodes[tk.node];
          if ((tk.score > JB200_LOG_ZERO) && !(tk.score < thr)) nin = arc_count(nr);
        }
        int tot_c;
        const int oc = block_excl_scan(nin, s_warp, &tot_c);
        if (j < ns) offs[j] = carry_c + oc;
        carry_c += tot_c;
      }
      cand_total = carry_c;
      if (tid == 0) offs[ns] = carry_c;
      if (cand_total > MAXC || cand_total > p.maxbits) { if (tid == 0) s_overflow = 1; cand_total = 0; }
    }
    int nwords = (cand_total + 31) >> 5;
    for (int w = tid; w < nwords; w += BEAM_THREADS) ua.bits[w] = 0u;
    __syncthreads();
    PROF_MARK(1);

    // ---- A2: word-internal transitions (beam_intra_word(_core), beam.c:2004-2177), one thread per
    //           candidate (survivors near the tree roots fan out 10-20 ways: per-survivor loops leave most
    //           of the block idle); the owner of candidate c is found by bisection of the offsets
    for (int c = tid; c < cand_total; c += BEAM_THREADS) {
      const int j = cand_owner(offs, ns, c);
      const int k = c - offs[j];
      const Tok tk = tl[ordl[j]];
      const NodeRec nr = p.nodes[tk.node];
      const IntraArc ar = intra_arc<false>(p, tk, nr, k);
      Cand cd; cd.score = ar.score; cd.node = ar.next; cd.lscore = ar.lscore; cd.src = j;
      ua.cand[c] = cd;
      if (ar.score > JB200_LOG_ZERO) cand_atomics(ua.slots, ar.next, ar.score, seq_no(j, k), seq_no(j, k));
    }
    __syncthreads();
    PROF_MARK(2);

    // ---- A3: creators, in arrival order = candidate order
    for (int c = tid; c < cand_total; c += BEAM_THREADS) {
      const Cand cd = ua.cand[c];
      if (!(cd.score > JB200_LOG_ZERO)) continue;
      if (first_arrival(ua.slots, cd.node, seq_no(cd.src, c - offs[cd.src]))) mark_creator(ua.bits, c);
    }
    __syncthreads();
    PROF_MARK(3);
    int ncre_a = rank_creators(ua.bits, ua.wpre, nwords, s_warp);
    if (ncre_a > MAXT) { if (tid == 0) s_overflow = 1; ncre_a = 0; }
    __syncthreads();
    PROF_MARK(4);

    // ---- A4: materialise the tokens of half A (no output probability yet) and mark their slots "exists"
    for (int c = tid; c < cand_total && ncre_a > 0; c += BEAM_THREADS) {
      const unsigned wbits = __ldcg(ua.bits + (c >> 5));
      if (!((wbits >> (c & 31)) & 1u)) continue;
      const int r = creation_rank(wbits, ua.wpre, c);
      const int node = ua.cand[c].node;
      const unsigned seqw = winner_seq(ua.slots, node);
      const int j = (int)(seqw >> SEQ_LOCAL_BITS), local = (int)(seqw & (SEQ_LOCAL - 1));
      const Cand cd = ua.cand[offs[j] + local];
      const Tok src = tl[ordl[j]];
      Tok nt; nt.node = node;
      nt.score = cd.score; nt.lscore = cd.lscore; nt.tre = src.tre; nt.cword = src.cword; nt.tre_wid = src.tre_wid;
      tn[r] = nt;
      heap[r + 1] = ((unsigned long long)(unsigned)r << 32) | __float_as_uint(nt.score);
      ua.slots.set(node, r - TOK_EXISTS, ((unsigned long long)fkey(nt.score) << 32) | 0xffffffffull);
    }
    __syncthreads();
    PROF_MARK(5);

    // ---- A5: heap select #1, replayed in full
    int ns_a;
    {
      const int need = p.beam;
      if (need >= ncre_a) {
        ns_a = ncre_a;
        for (int k = tid; k < ns_a; k += BEAM_THREADS) ordn[k] = k;
      } else {
        ns_a = need;
        if (need < ncre_a - need) select_exact<true>(ca, ncre_a, need, ordn, MAXT, p.cut_counters);
        else select_exact<false>(ca, ncre_a, need, ordn, MAXT, p.cut_counters);
        if constexpr (CHECK) check_select(p.heap_chk + (size_t)u * (MAXT + 4), ncre_a, need, tn, heap, nullptr, &s_overflow);
      }
    }
    __syncthreads();
    PROF_MARK(6);

    // ---- B1: word ends among the survivors of select #1: trellis words (save_trellis, beam.c:2209)
    //          and the cross-word sources (beam_inter_word's per-token part, beam.c:2271-2335)
    int nbits_b;
    {
      int carry_a = s_natoms, carry_w = 0;
      for (int k0 = 0; k0 < ns_a; k0 += BEAM_THREADS) {
        const int k = k0 + tid;
        int is_we = 0, is_tr = 0;
        Tok tk; NodeRec nr;
        if (k < ns_a) {
          tk = tn[ordn[k]];
          nr = p.nodes[tk.node];
          if (!(tk.score < thr) && nr.stend >= 0) { is_we = 1; is_tr = (!final && nr.stend != p.tail_silwid); }
        }
        int tot_a, tot_w;
        const int oa = block_excl_scan(is_we, s_warp, &tot_a);
        const int ow = block_excl_scan(is_tr, s_warp, &tot_w);
        if (is_we) word_end<false>(p, ua, tk, nr.stend, t - 1, t > 0, carry_a + oa, is_tr, carry_w + ow, k, 0, &s_webest, &s_overflow);
        carry_a += tot_a; carry_w += tot_w;
      }
      if (tid == 0) { s_natoms = min(carry_a, ua.atom_cap); s_E = min(carry_w, MAXW); }
      nbits_b = carry_w * p.n_isoarc + p.n_sharc;
      // carry_a > ua.atom_cap: some word ends got no atom and no ua.wend entry, and ua.wend[0..E) would hold stale entries
      if (carry_w > MAXW || nbits_b > p.maxbits || carry_a > ua.atom_cap) { if (tid == 0) s_overflow = 1; nbits_b = 0; }
    }
    if (final) { n_left = ncre_a; __syncthreads(); break; }
    nwords = (nbits_b + 31) >> 5;
    for (int w = tid; w < nwords; w += BEAM_THREADS) ua.bits[w] = 0u;
    __syncthreads();
    PROF_MARK(1);
    const int E = (nbits_b > 0) ? s_E : 0;

    // ---- B2: cross-word transitions through the isolated roots (beam.c:2336-2500), one candidate per
    //          (word end, root successor), pre-reduced per successor over the word ends in visiting order
    for (int ia = tid; ia < p.n_isoarc; ia += BEAM_THREADS) {
      const IsoCand ic = reduce_word_ends<false, true>(p, ua.wend, E, __ldg(p.iso_id + __ldg(p.isoarc_iso + ia)), __ldg(p.isoarc_a + ia));
      ua.iso[ia] = ic;
      if (ic.first_e >= 0)
        cand_atomics(ua.slots, __ldg(p.isoarc_node + ia), ic.score, seq_no(ua.wend[ic.first_e].j + 1, ia), seq_no(ua.wend[ic.e].j + 1, ia));
    }
    // ---- B3: best word end -> successors of the shared (1-gram factored) roots (beam.c:2549-2616)
    const unsigned long long webest = s_webest;
    const bool have_we = (webest != 0ull) && (nbits_b > 0);
    WEnd wbest; wbest.base = 0.0f; wbest.atom = -1; wbest.last_word = -1; wbest.transp2 = 0; wbest.j = 0; wbest.nintra = 0;
    auto shared_value = [&](int sa, float &lsc, float &v) -> bool {
      const float tmpsum = factoring_score(p, wbest, __ldg(p.sharc_shared + sa), lsc);
      if (tmpsum < thr) return false;
      v = tmpsum + __ldg(p.sharc_a + sa);
      return v > JB200_LOG_ZERO;
    };
    if (have_we) {
      wbest = ua.wend[(unsigned)(~(unsigned)(webest & 0xffffffffu))];
      for (int sa = tid; sa < p.n_sharc; sa += BEAM_THREADS) {
        float lsc, v;
        if (shared_value(sa, lsc, v)) cand_atomics(ua.slots, __ldg(p.sharc_node + sa), v, seq_no(ns_a + 1, sa), seq_no(ns_a + 1, sa));
      }
    }
    __syncthreads();
    PROF_MARK(2);

    // ---- B4: creators of half B (arrival order: word end major, then the factoring pass)
    for (int ia = tid; ia < p.n_isoarc; ia += BEAM_THREADS) {
      const IsoCand ic = ua.iso[ia];
      if (ic.first_e < 0) continue;
      if (first_arrival(ua.slots, __ldg(p.isoarc_node + ia), seq_no(ua.wend[ic.first_e].j + 1, ia)))
        mark_creator(ua.bits, ic.first_e * p.n_isoarc + ia);
    }
    if (have_we) {
      for (int sa = tid; sa < p.n_sharc; sa += BEAM_THREADS)
        if (first_arrival(ua.slots, __ldg(p.sharc_node + sa), seq_no(ns_a + 1, sa))) mark_creator(ua.bits, E * p.n_isoarc + sa);
    }
    __syncthreads();
    PROF_MARK(3);
    int ncre = ncre_a + rank_creators(ua.bits, ua.wpre, nwords, s_warp);
    if (ncre > MAXT) { if (tid == 0) s_overflow = 1; ncre = ncre_a; nbits_b = 0; }
    __syncthreads();
    PROF_MARK(4);

    // ---- B5: new tokens get the winner's content; tokens of half A that lost to a cross-word arrival
    //          are overwritten in place (propagate_token, beam.c:1901-1972)
    auto winner_content = [&](unsigned seqw, Tok &nt) {
      const int j = (int)(seqw >> SEQ_LOCAL_BITS), local = (int)(seqw & (SEQ_LOCAL - 1));
      if (j == ns_a + 1) {
        float lsc, v;
        shared_value(local, lsc, v);
        nt.score = v; nt.lscore = lsc;
        enter_from(nt, wbest, ua.araw);
      } else {
        const IsoCand ic = ua.iso[local];
        const WEnd w = ua.wend[ic.e];
        nt.score = ic.score; nt.lscore = ic.lscore;
        enter_from(nt, w, ua.araw);
      }
    };
    auto settle = [&](int node, unsigned seq_first, unsigned seq_win, int pos) {
      const int fs = __ldcg(ua.slots.fs(node));
      const unsigned seqw = winner_seq(ua.slots, node);
      if (fs < 0) {
        if (seqw != seq_win) return;
        Tok nt; nt.node = node;
        winner_content(seqw, nt);
        tn[fs + TOK_EXISTS] = nt;
      } else if ((unsigned)fs == seq_first) {
        const int r = ncre_a + creation_rank(__ldcg(ua.bits + (pos >> 5)), ua.wpre, pos);
        Tok nt; nt.node = node;
        winner_content(seqw, nt);
        tn[r] = nt;
      }
    };
    if (nbits_b > 0) {
      for (int ia = tid; ia < p.n_isoarc; ia += BEAM_THREADS) {
        const IsoCand ic = ua.iso[ia];
        if (ic.first_e < 0) continue;
        settle(__ldg(p.isoarc_node + ia), seq_no(ua.wend[ic.first_e].j + 1, ia), seq_no(ua.wend[ic.e].j + 1, ia),
               ic.first_e * p.n_isoarc + ia);
      }
      if (have_we)
        for (int sa = tid; sa < p.n_sharc; sa += BEAM_THREADS) {
          float lsc, v;
          if (shared_value(sa, lsc, v)) settle(__ldg(p.sharc_node + sa), seq_no(ns_a + 1, sa), seq_no(ns_a + 1, sa), E * p.n_isoarc + sa);
        }
    }
    __syncthreads();

    // ---- B6: output probabilities of the emitting tokens (beam.c:2930-2941); then the index array select #2
    //          starts from: select #1's arrangement with fresh scores, followed by the tokens of half B
    for (int r = tid; r < ncre; r += BEAM_THREADS) {
      const Tok tk = tn[r];
      const int out = p.nodes[tk.node].out;
      float sc = tk.score;
      if (((unsigned)out >> 28) != 0xFu) {
        sc += outprob_style(p, row, out, tk.tre_wid);
        tn[r].score = sc;
        atomicMax(&s_pmaxkey, fkey(sc));
      }
      atomicMax(&s_hmaxkey, fkey(sc));
      if (r >= ncre_a) heap[r + 1] = ((unsigned long long)(unsigned)r << 32) | __float_as_uint(sc);
    }
    __syncthreads();
    for (int h = 1 + tid; h <= ncre_a; h += BEAM_THREADS) {
      const unsigned id = (unsigned)(heap[h] >> 32);
      heap[h] = ((unsigned long long)id << 32) | __float_as_uint(tn[id].score);
    }
    __syncthreads();
    PROF_MARK(5);

    // ---- B7: heap select #2 (only its survivors' order is observable: loser cut allowed)
    const int ns_new = min(ncre, p.beam);
    if (ncre <= p.beam) {
      // tindex order = select #1's arrangement, then the new tokens
      for (int k = tid; k < ns_new; k += BEAM_THREADS) ordn[k] = (int)(heap[k + 1] >> 32);
    } else {
      // the input of select #2 cannot be rebuilt after the cut: the self-check keeps a copy
      if constexpr (CHECK) check_select(p.heap_chk + (size_t)u * (MAXT + 4), ncre, 0, nullptr, heap, nullptr, nullptr);
      beam_cut(p, ca, ncre, s_hmaxkey, tn, ua.slots, ordn, s_prof, s_tprev);
      slots_clean = true;
      if constexpr (CHECK) check_select(p.heap_chk + (size_t)u * (MAXT + 4), ncre, p.beam, nullptr, nullptr, ordn, &s_overflow);
    }
    PROF_MARK(6);
    // (s_pmaxkey starts at fkey(LOG_ZERO) here, never 0)
    if (tid == 0) { end_frame(p, ua.counts, t, ncre, ns_new, s_pmaxkey, s_ns, s_thr); s_cur = nxt; }
    tnum_prev = ncre;
    __syncthreads();
    if (ncre == 0) { stopped = t; break; }      // beam.c:3012-3015
  }

  if (!ck_final) {
    if (tid == 0) park_scalars(p, u, ua, T, s_natoms, s_overflow, s_thr, s_ns, s_cur, tnum_prev, stopped, slots_clean, s_prof, s_tprev);
    return;
  }
  const int groups = (stopped >= 0) ? stopped : T;

  {
    if (tid == 0 && T > 0) ua.group0[groups] = s_natoms;
    // leave the node slots clean for the next utterance that uses this work area
    // (only the unfinished final frame leaves any: every other frame's slots are reset by the next P0)
    SlotClear{ua.tok0 + (size_t)(s_cur ^ 1) * MAXT, n_left, ua.slots}.run(tid, BEAM_THREADS);
    __syncthreads();
  }
  finalize_utt<false>(p, u, tid, T, ua.araw, ua.newidx, ua.group0, ua.res, ua.words, s_natoms, s_overflow, s_found, s_outbase, s_prof, s_tprev);
}

// the beam kernel for a tree (grammar mode runs on normal trees only); check: the JB200_CHECK_HEAP build
using BeamKernel = void (*)(BeamParams);
static BeamKernel beam_kernel_for(const bool grammar, const bool multipath, const bool check) {
  if (multipath) return check ? beam_kernel_mp<true> : beam_kernel_mp<false>;
  if (grammar) return check ? beam_kernel<true, true> : beam_kernel<true, false>;
  return check ? beam_kernel<false, true> : beam_kernel<false, false>;
}

// ---- set-up kernels ------------------------------------------------------------------------------
__global__ void iw_table_kernel(BeamParams p, const int *iso_word, float *iw, int n_words) {
  // max_successor_prob_iw (factoring_sub.c:1049-1143) for EVERY last word, once
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n_words * p.n_iso) return;
  const int lw = (int)(idx / p.n_iso), i = (int)(idx % p.n_iso);
  const int w = iso_word[i];
  iw[(size_t)lw * p.n_iso + p.iso_id[i]] = bigram_prob(p, p.wton[lw], p.wton[w]) + p.cprob[w];
}

__global__ void fill_slots_kernel(NodeSlot *slots, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) slots[i] = NodeSlot{0ull, 0x7fffffff, 0};
}

// Streams of a DNN with a context window (splice_mfcc, realtime-1stpass.c:445-460): after a feed, stream s (block s) keeps
// the last min(keep, window length) frames of the feed's window -- what it carried plus what came in -- for the windows
// of its next feed.  Reads the old carry and writes the other buffer of the pair.
__global__ void carry_update_kernel(const SpliceSeg *__restrict__ seg, const float *__restrict__ in, const float *__restrict__ carry_old,
                                    float *__restrict__ carry_new, int keep, int fl) {
  const SpliceSeg s = seg[blockIdx.x];
  const int n = min(keep, s.n_win), k0 = s.n_win - n;
  for (int i = threadIdx.x; i < n * fl; i += blockDim.x)
    carry_new[(size_t)s.carry0 * fl + i] = splice_frame(s, k0 + i / fl, in, carry_old, fl)[i % fl];
}

}  // namespace jb200

// =============================================================================================
using namespace jb200;

// What turns a batch's or a feed's input into score rows: the scorer, the feature and score-row buffers it fills, and for
// a DNN that splices ctx input frames of fl floats into each network input (jb200_dnn_set_context) the segment table
// (pinned staging copy and device copy, max_utts + 1 entries) and, per stream, the input frames of its utterance so far
// and its last ctx - 1 of them on the device, in one of a pair of buffers (carry_cur) that a feed's update swaps.
// A decoder has its own; a group (jb200_group_*) has one for all its members.
struct RowSource {
  jb200_gmm *am = nullptr;
  jb200_dnn *dnn = nullptr;
  int dim = 0, S = 0, row_stride = 0;
  int max_utts = 0, max_frames = 0;
  float *d_feats = nullptr, *d_rows = nullptr;
  int ctx = 1, fl = 0;
  SpliceSeg *h_splice = nullptr, *d_splice = nullptr;
  float *d_carry[2] = {nullptr, nullptr}; int carry_cur = 0; size_t carry_floats = 0;
  std::vector<int> st_in;
  bool splices() const { return dnn && ctx > 1; }
};

struct jb200_decoder {
  RowSource in;
  int device = 0;
  int max_utts = 0, max_frames = 0;         // per batch: utterances, total frames
  int atoms_per_frame = 64;
  // the one home of every device pointer fixed at create; launch_beam sets only the chunk row, interim and atoms_in_place
  BeamParams P{};
  std::vector<void *> dev_allocs, host_allocs;  // device memory and pinned host memory, freed by jb200_decoder_destroy
  // read-only tables shared by all utterances (tree, LM, inter-word table, bigram memo) sit in ONE allocation
  char *arena = nullptr; size_t arena_size = 0, arena_used = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[5]{};
  // buffers the host writes and the kernel reads through P's const pointers
  int *d_frame_off = nullptr; long long *d_atom_off = nullptr;
  // host results (pinned)
  jb200_utt_result *h_results = nullptr; jb200_atom *h_atoms = nullptr; int *h_words = nullptr;
  unsigned long long *h_counter = nullptr;
  int last_n = 0, last_total_frames = 0;
  std::vector<int> h_frame_off;
  float last_ms[4] = {0, 0, 0, 0};
  size_t smem_bytes = 0;
  BeamKernel beam = nullptr;                    // beam_kernel_for the decoder's tree
  bool fetched = false;
  long long last_d2h = 0;
  int resident = 0;
  // chunked launches: descriptors (a pinned staging copy and its device copy, one row of max_utts per chunk)
  static constexpr int MAX_CHUNKS = 64;
  ChunkDesc *h_chunk = nullptr, *d_chunk = nullptr;
  // batch pipeline: scoring of time slice c+1 on its own stream beside the token passing of slice c
  cudaStream_t score_stream = nullptr;
  cudaEvent_t ev_slice[MAX_CHUNKS]{}; cudaEvent_t ev_score_begin = nullptr, ev_score_end = nullptr;
  int *h_seg = nullptr, *d_seg = nullptr;       // per slice: seg_off [max_utts+1] then seg_start [max_utts]
  std::vector<int> slice_nseg, slice_frames;
  int pipe_frames = 0;                          // frames per time slice; 0 = the pipeline is off
  int n_chunks = 1; float last_score_busy_ms = 0.0f; bool last_piped = false;
  // streams (jb200_stream_*)
  bool stream_mode = false; int st_n = 0, st_cap = 0;
  std::vector<int> st_t; std::vector<char> st_started, st_done;
  long long *h_aoff = nullptr;                  // pinned copy of the per-utterance atom offsets
  UttState *h_state = nullptr; int *h_interim_words = nullptr;
  // the group whose open stream this decoder is in (jb200_group_stream_open): its own feeds are refused meanwhile
  const jb200_group *stream_group = nullptr;
};

// from the shared-table arena when it has room, else an allocation of its own
static void *arena_take(jb200_decoder *d, size_t bytes) {
  const size_t need = (bytes + 255) & ~(size_t)255;
  if (!d->arena || d->arena_used + need > d->arena_size) return nullptr;
  void *p = d->arena + d->arena_used;
  d->arena_used += need;
  return p;
}
// Owner: a decoder or a group, which frees its dev_allocs and host_allocs when destroyed
template <typename Owner, typename Tp>
static int dev_alloc(Owner *d, size_t n, Tp **dst) {
  Tp *p = nullptr;
  JB_CUDA(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(Tp)));
  d->dev_allocs.push_back(p);
  *dst = p;
  return JB200_OK;
}
template <typename Tp>
static int dev_alloc_shared(jb200_decoder *d, size_t n, Tp **dst) {
  *dst = static_cast<Tp *>(arena_take(d, std::max<size_t>(n, 1) * sizeof(Tp)));
  return *dst ? JB200_OK : dev_alloc(d, n, dst);
}
template <typename Tp>
static int dev_upload(jb200_decoder *d, const Tp *src, size_t n, const Tp **dst) {
  Tp *p = nullptr;
  JB_RC(dev_alloc_shared(d, n, &p));
  if (n) JB_CUDA(cudaMemcpy(p, src, n * sizeof(Tp), cudaMemcpyHostToDevice));
  *dst = p;
  return JB200_OK;
}
template <typename Owner, typename Tp>
static int host_alloc(Owner *d, size_t n, Tp **dst) {
  Tp *p = nullptr;
  JB_CUDA(cudaMallocHost(&p, n * sizeof(Tp)));
  d->host_allocs.push_back(p);
  *dst = p;
  return JB200_OK;
}

// resets the node slots of utterances [u0, u0 + n_utts) on the main stream
static int reset_slots(jb200_decoder *d, int u0, int n_utts) {
  const size_t tot = (size_t)n_utts * d->P.n_nodes;
  fill_slots_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, d->stream>>>(d->P.slots + (size_t)u0 * d->P.n_nodes, tot);
  JB_LAUNCH_CHECK();
  return JB200_OK;
}

extern "C" void jb200_decoder_destroy(jb200_decoder *d) {
  if (!d) return;
  cudaSetDevice(d->device);
  for (void *p : d->dev_allocs) cudaFree(p);
  for (void *p : d->host_allocs) cudaFreeHost(p);
  for (auto &e : d->ev) if (e) cudaEventDestroy(e);
  for (auto &e : d->ev_slice) if (e) cudaEventDestroy(e);
  if (d->ev_score_begin) cudaEventDestroy(d->ev_score_begin);
  if (d->ev_score_end) cudaEventDestroy(d->ev_score_end);
  if (d->score_stream) cudaStreamDestroy(d->score_stream);
  if (d->stream) cudaStreamDestroy(d->stream);
  delete d;
}

// Multipath trees: the roots carry no output, so a cross-word transition into a root lands on the root's successors
// (self, next, arcs: the order propagation visits them, beam.c:2467-2500).  The word-begin node of the head silence is
// never entered (beam.c:2336-2342).  Calls f(list, root index, successor node, transition score) root-major, the isolated
// roots (list 0) before the shared ones (list 1), in original node ids.
template <typename F>
static void for_root_successors(const jb200_tree_desc *t, F f) {
  auto expand = [&](int list, int idx, int x) {
    if (t->self_a[x] != JB200_LOG_ZERO) f(list, idx, x, t->self_a[x]);
    if (t->next_a[x] != JB200_LOG_ZERO) f(list, idx, x + 1, t->next_a[x]);
    for (int k = t->arc_off[x]; k < t->arc_off[x + 1]; k++) f(list, idx, t->arc_to[k], t->arc_a[k]);
  };
  const int head_begin = t->wordbegin[t->head_silwid];
  for (int i = 0; i < t->n_iso; i++) if (t->iso_node[i] != head_begin) expand(0, i, t->iso_node[i]);
  for (int i = 0; i < t->n_shared; i++) expand(1, i, t->shared_node[i]);
}

// The trees the beam kernels cannot decode.  Reads the descriptor alone; a count is checked before the loops that read
// arrays of that size.
static int check_tree(const jb200_tree_desc *t) {
  const bool grammar = (t->lm_type == JB200_LM_DFA);
  if (t->lm_type != JB200_LM_NGRAM && !grammar) { set_error("unknown language-model type %d", t->lm_type); return JB200_ERR_UNSUPPORTED; }
  if (grammar) {
    if (t->multipath) { set_error("grammar mode on a multipath tree is not supported by the GPU beam"); return JB200_ERR_UNSUPPORTED; }
    if (t->n_shared != 0 || t->n_init < 1 || t->n_init > t->beam_width || !t->cp_allowed || !t->init_node || !t->init_lscore) {
      set_error("grammar mode: inconsistent descriptor (n_shared %d, n_init %d, beam %d)", t->n_shared, t->n_init, t->beam_width);
      return JB200_ERR_ARG;
    }
    for (int i = 0; i < t->n_words; i++)
      if (t->is_transparent[i]) { set_error("grammar mode: transparent words are not supported"); return JB200_ERR_UNSUPPORTED; }
  }
  if (t->n_nodes >= (1 << 28)) { set_error("lexicon tree too large"); return JB200_ERR_UNSUPPORTED; }
  // a transparent head silence would end the first word with no context word at all (last_word = -1): the reference
  // indexes wton[] / the inter-word cache with WORD_INVALID there (factoring_sub.c:1052-1056), i.e. has no defined result
  if (!grammar && (t->head_silwid < 0 || t->head_silwid >= t->n_words || t->is_transparent[t->head_silwid])) {
    set_error("the head silence word must exist and must not be transparent"); return JB200_ERR_UNSUPPORTED;
  }
  if (t->beam_width < 1 || t->beam_width > 8000) { set_error("beam width %d outside 1..8000", t->beam_width); return JB200_ERR_UNSUPPORTED; }
  for (int o = 0; o < t->n_nodes; o++) {
    const int style = t->outstyle[o];
    if (style > 3 && !(style == 255 && t->multipath)) { set_error("non-emitting node in a non-multipath tree"); return JB200_ERR_UNSUPPORTED; }
  }
  for (int i = 0; i < t->n_shared; i++)
    if (t->scid[t->shared_node[i]] >= 0) { set_error("shared root without 1-gram factoring value"); return JB200_ERR_ARG; }
  // a root, or on a multipath tree a root's successor, is numbered in the low SEQ_LOCAL_BITS of an arrival sequence number
  long long n_arcs[2] = {0, 0};
  if (t->multipath) for_root_successors(t, [&](int list, int, int, float) { n_arcs[list]++; });
  if (t->n_iso + 1024 >= (int)SEQ_LOCAL || n_arcs[0] >= SEQ_LOCAL || n_arcs[1] >= SEQ_LOCAL || t->n_shared >= (int)SEQ_LOCAL) {
    set_error("too many tree roots (%d isolated, %d shared) for the arrival-order numbering", t->n_iso, t->n_shared);
    return JB200_ERR_UNSUPPORTED;
  }
  return JB200_OK;
}

// Create, step 1: the tree, renumbered, and its tables
static int upload_tree(jb200_decoder *d, const jb200_tree_desc *t) {
  BeamParams &P = d->P;
  const bool grammar = (t->lm_type == JB200_LM_DFA);
  const int n = t->n_nodes;
  // Node numbering.  The host numbers the nodes word by word (a word's own nodes are consecutive), so the ~2400 nodes a
  // frame touches are spread over the whole tree although 85 % of them sit in its first three levels (half of a frame's
  // tokens are the roots that a word end fans out to): one 128-byte line of per-node arrival slots per token.  Node ids
  // are not observable outside the decoder, so the tree is renumbered breadth-first from the roots (roots in their list
  // order, then level by level): the slots and node records a frame touches become a few dense ranges -- 3.4x fewer
  // slot lines, 2.1x fewer node-record lines per frame on the 20k-word tree (tools/node_locality.py).  `next_a` no longer
  // leads to id+1, so the record carries the successor explicitly.
  std::vector<int> perm(n), inv(n);
  {
    std::vector<int> order; order.reserve(n);
    std::vector<char> seen(n, 0);
    auto push = [&](int x) { if (x >= 0 && x < n && !seen[x]) { seen[x] = 1; order.push_back(x); } };
    for (int i = 0; i < t->n_iso; i++) push(t->iso_node[i]);
    for (int i = 0; i < t->n_shared; i++) push(t->shared_node[i]);
    if (grammar) for (int i = 0; i < t->n_init; i++) push(t->init_node[i]);
    for (size_t q = 0; q < order.size(); q++) {
      const int x = order[q];
      if (t->next_a[x] != JB200_LOG_ZERO) push(x + 1);
      for (int k = t->arc_off[x]; k < t->arc_off[x + 1]; k++) push(t->arc_to[k]);
    }
    for (int x = 0; x < n; x++) push(x);                       // whatever the roots do not reach keeps its relative order
    for (int i = 0; i < n; i++) { perm[order[i]] = i; inv[i] = order[i]; }
  }
  auto remap = [&](const int *src, size_t cnt) { std::vector<int> v(cnt); for (size_t i = 0; i < cnt; i++) v[i] = perm[src[i]]; return v; };
  // node records and the arc lists, in the new order
  std::vector<NodeRec> nodes(n);
  std::vector<int> arc_to_n((size_t)std::max(t->n_arcs, 1)); std::vector<float> arc_a_n((size_t)std::max(t->n_arcs, 1));
  {
    int ao = 0;
    for (int i = 0; i < n; i++) {
      const int o = inv[i];
      NodeRec &r = nodes[i];
      r.self_a = t->self_a[o]; r.next_a = t->next_a[o];
      r.arc_off = ao; r.arc_n = t->arc_off[o + 1] - t->arc_off[o];
      for (int k = t->arc_off[o]; k < t->arc_off[o + 1]; k++) { arc_to_n[ao] = perm[t->arc_to[k]]; arc_a_n[ao] = t->arc_a[k]; ao++; }
      r.stend = t->stend[o]; r.scid = t->scid[o];
      const int style = t->outstyle[o];
      r.out = (style == 255) ? (int)0xF0000000u : (int)(((unsigned)style << 28) | (unsigned)(t->out_ref[o] & 0x0fffffff));
      r.next = (r.next_a != JB200_LOG_ZERO && o + 1 < n) ? perm[o + 1] : i;
    }
  }
  JB_RC(dev_upload(d, nodes.data(), nodes.size(), &P.nodes));
  JB_RC(dev_upload(d, arc_to_n.data(), (size_t)t->n_arcs, &P.arc_to));
  JB_RC(dev_upload(d, arc_a_n.data(), (size_t)t->n_arcs, &P.arc_a));
  JB_RC(dev_upload(d, t->rset_ctx, (size_t)t->n_rset * (t->n_ctx + 1), &P.rset_ctx));
  JB_RC(dev_upload(d, t->word_ctx, (size_t)t->n_words, &P.word_ctx));
  P.n_ctx = t->n_ctx;
  { const std::vector<int> v = remap(t->iso_node, (size_t)t->n_iso); JB_RC(dev_upload(d, v.data(), v.size(), &P.iso_node)); }
  JB_RC(dev_upload(d, t->iso_id, (size_t)t->n_iso, &P.iso_id));
  P.n_iso = t->n_iso;
  { const std::vector<int> v = remap(t->shared_node, (size_t)t->n_shared); JB_RC(dev_upload(d, v.data(), v.size(), &P.shared_node)); }
  {
    // check_tree: every shared root has a 1-gram factoring value
    std::vector<float> sf(std::max(t->n_shared, 1));
    for (int i = 0; i < t->n_shared; i++) sf[i] = t->fscore[-t->scid[t->shared_node[i]]];
    JB_RC(dev_upload(d, sf.data(), (size_t)t->n_shared, &P.shared_f));
  }
  P.n_shared = t->n_shared;
  P.multipath = t->multipath ? 1 : 0;
  P.head_node = grammar ? 0 : perm[t->wordbegin[t->head_silwid]]; P.n_nodes = n;
  if (grammar) {
    JB_RC(dev_upload(d, t->cp_allowed, (size_t)t->n_words * t->n_iso, &P.cp_allowed));
    { const std::vector<int> v = remap(t->init_node, (size_t)t->n_init); JB_RC(dev_upload(d, v.data(), v.size(), &P.init_node)); }
    JB_RC(dev_upload(d, t->init_lscore, (size_t)t->n_init, &P.init_lscore));
    P.n_init = t->n_init; P.penalty1 = t->penalty1;
  }
  // multipath: the successors of the isolated roots (list 0) and of the shared roots (list 1)
  std::vector<int> rs_node[2], rs_root[2]; std::vector<float> rs_a[2];
  if (t->multipath)
    for_root_successors(t, [&](int list, int idx, int x, float a) { rs_node[list].push_back(perm[x]); rs_root[list].push_back(idx); rs_a[list].push_back(a); });
  P.n_isoarc = (int)rs_node[0].size(); P.n_sharc = (int)rs_node[1].size();
  JB_RC(dev_upload(d, rs_node[0].data(), rs_node[0].size(), &P.isoarc_node));
  JB_RC(dev_upload(d, rs_root[0].data(), rs_root[0].size(), &P.isoarc_iso));
  JB_RC(dev_upload(d, rs_a[0].data(), rs_a[0].size(), &P.isoarc_a));
  JB_RC(dev_upload(d, rs_node[1].data(), rs_node[1].size(), &P.sharc_node));
  JB_RC(dev_upload(d, rs_root[1].data(), rs_root[1].size(), &P.sharc_shared));
  JB_RC(dev_upload(d, rs_a[1].data(), rs_a[1].size(), &P.sharc_a));
  return JB200_OK;
}

// Create, step 2: the LM tables and the inter-word table
static int upload_lm(jb200_decoder *d, const jb200_tree_desc *t) {
  BeamParams &P = d->P;
  const bool grammar = (t->lm_type == JB200_LM_DFA);
  JB_RC(dev_upload(d, t->wordend_a, (size_t)t->n_words, &P.wordend_a));
  JB_RC(dev_upload(d, t->is_transparent, (size_t)t->n_words, &P.is_transp));
  JB_RC(dev_upload(d, t->wton, (size_t)t->n_words, &P.wton));
  JB_RC(dev_upload(d, t->cprob, (size_t)t->n_words, &P.cprob));
  JB_RC(dev_upload(d, t->fscore, (size_t)t->n_fscore, &P.fscore));
  JB_RC(dev_upload(d, t->scword, (size_t)t->n_scword, &P.scword));
  JB_RC(dev_upload(d, t->uni_prob, (size_t)t->lm_nvocab, &P.uni_prob));
  JB_RC(dev_upload(d, t->uni_bow, (size_t)t->lm_nvocab, &P.uni_bow));
  JB_RC(dev_upload(d, t->bi_bgn, (size_t)t->lm_nvocab, &P.bi_bgn));
  JB_RC(dev_upload(d, t->bi_num, (size_t)t->lm_nvocab, &P.bi_num));
  JB_RC(dev_upload(d, t->bi_wid, (size_t)t->lm_nbigram, &P.bi_wid));
  JB_RC(dev_upload(d, t->bi_prob, (size_t)t->lm_nbigram, &P.bi_prob));
  P.lm_mode = t->lm_mode; P.lm_unk_id = t->lm_unk_id; P.lm_unk_num_log = t->lm_unk_num_log;
  P.lm_weight = t->lm_weight; P.lm_penalty = t->lm_penalty; P.lm_penalty_trans = t->lm_penalty_trans;
  P.prune_width = t->score_pruning_width;
  P.tail_silwid = t->tail_silwid; P.beam = t->beam_width;
  // cd sets come from the AM handle's descriptor: re-upload from the gmm handle is not exposed, so the
  // decoder asks the scorer for its device copies
  P.cd = gmm_cdsets(d->in.am);
  // inter-word bigram rows for every last word (the reference's iw_sc_cache, fully populated)
  const int *d_iso_word = nullptr;
  JB_RC(dev_upload(d, t->iso_word, (size_t)t->n_iso, &d_iso_word));
  float *iw = nullptr;
  JB_RC(dev_alloc_shared(d, (size_t)t->n_words * std::max(t->n_iso, 1), &iw));
  P.iw = iw;
  const long long tot = grammar ? 0 : (long long)t->n_words * t->n_iso;     // grammar mode reads cp_allowed instead
  if (tot > 0) {
    iw_table_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, d->stream>>>(P, d_iso_word, iw, t->n_words);
    JB_LAUNCH_CHECK();
  }
  return JB200_OK;
}

// Create, step 3: the sizes of the beam cut, from the beam width, the number of start tokens and the device's opt-in
// shared memory per block.  tests/test_gpu_beam_widths.py restates the heap placement rule.
// maxt: token capacity of a frame; sort_cap, qcap: see BeamParams (global heap only); smem_bytes: the kernel's dynamic share
struct CutSizing { int maxt; bool heap_global; int sort_cap, qcap; size_t smem_bytes; };
static int size_cut(int beam, int n_start, int smem_optin, CutSizing *cs) {
  // the reference starts at 2*beam+startnum tokens and grows on demand; we size once and flag overflow.  Seen on the
  // 20k-word tree: 4.6*beam at -b 800 (of which startnum = 1375 root tokens), 4.7*beam at -b 4000.  The array lives
  // in shared memory, and what it takes is lost to L1 (5*beam+startnum at -b 800 costs 30 % of the kernel's speed).
  int maxt = (std::max(4 * beam + n_start, 5 * beam) + 64 + 3) & ~3;
  // Where the heap-select array lives.  Shared memory as long as one block's share fits; a wide beam on a large tree
  // (-b 4000 on the 60k-word multipath tree creates up to 8.5 x beam tokens a frame) goes to global memory instead,
  // with room for 9 x beam + startnum tokens, and shared memory keeps only the closed form's sort area.
  const size_t offs_bytes = (size_t)(beam + 2) * 4 * 2;
  const int smem_limit = smem_optin - 2048;                 // static shared variables of the kernels
  const bool heap_global = (size_t)(maxt + 4) * 8 + offs_bytes > (size_t)smem_limit / 2;   // would leave one block per SM
  int sort_cap = 0, qcap = 0;
  if (heap_global) {
    maxt = std::min(65000, (std::max(maxt, 9 * beam + n_start) + 3) & ~3);
    sort_cap = 1024; while (sort_cap < 2 * beam && sort_cap < 16384) sort_cap <<= 1;   // candidates = beam + one histogram bin
    const size_t tail_bytes = (size_t)(beam + 2) * 8;                                 // the replay's copy of the tail slots
    if ((size_t)sort_cap * 8 + offs_bytes + tail_bytes > (size_t)smem_limit) { set_error("beam width %d needs more shared memory than the device has", beam); return JB200_ERR_UNSUPPORTED; }
    // what is left of shared memory holds the top levels of the heap during a replay (one block per SM: the replay is all
    // that matters at these beam widths)
    qcap = sort_cap;
    while ((size_t)qcap * 2 * 8 + offs_bytes + tail_bytes <= (size_t)smem_limit && qcap * 2 <= ((maxt + 4) | 1023) + 1) qcap <<= 1;
  }
  const size_t heap_bytes = heap_global ? (size_t)qcap * 8 + (size_t)(beam + 2) * 8 : (size_t)(maxt + 4) * 8;
  *cs = CutSizing{maxt, heap_global, sort_cap, qcap, heap_bytes + offs_bytes};
  return JB200_OK;
}

// Create, step 4: the per-utterance work areas, the batch buffers, the pipeline's stream and events, the kernel set-up
static int alloc_work(jb200_decoder *d, const jb200_tree_desc *t, const CutSizing &cs) {
  BeamParams &P = d->P;
  const int mu = d->max_utts, mf = d->max_frames, maxt = cs.maxt, MC = jb200_decoder::MAX_CHUNKS;
  P.sort_cap = cs.sort_cap; P.qcap = cs.qcap;
  if (cs.heap_global) JB_RC(dev_alloc(d, (size_t)mu * (maxt + 4), &P.heap_g));
  P.maxt = maxt; P.maxc = 4 * maxt; P.maxw = t->beam_width + 1;
  JB_RC(dev_alloc(d, (size_t)mu * 2 * maxt, &P.tok));
  JB_RC(dev_alloc(d, (size_t)mu * 2 * maxt, &P.order));
  JB_RC(dev_alloc(d, (size_t)mu * P.n_nodes, &P.slots));
  JB_RC(dev_alloc(d, (size_t)mu * P.maxc, &P.cand));
  JB_RC(dev_alloc(d, (size_t)mu * P.maxc, &P.candb));
  JB_RC(dev_alloc(d, (size_t)mu * (t->beam_width + 2), &P.surv));
  const int n_isoent = std::max(std::max(t->n_iso, P.n_isoarc), 1);
  JB_RC(dev_alloc(d, (size_t)mu * n_isoent, &P.iso));
  JB_RC(dev_alloc(d, (size_t)mu * P.maxw, &P.wend));
  P.maxbits = (P.maxc + std::min(P.maxw, 256) * n_isoent + std::max(t->n_shared, P.n_sharc) + 63) & ~31;
  JB_RC(dev_alloc(d, (size_t)mu * (P.maxbits >> 5), &P.bitmask));
  JB_RC(dev_alloc(d, (size_t)mu * (P.maxbits >> 5), &P.wordpre));
  JB_RC(dev_alloc(d, CUT_SLOTS, &P.cut_counters));
  JB_CUDA(cudaMemset(P.cut_counters, 0, CUT_SLOTS * sizeof(unsigned long long)));
  // JB200_CHECK_HEAP=1: check every cut against the plain sequential replay
  const bool check_heap = getenv("JB200_CHECK_HEAP") && atoi(getenv("JB200_CHECK_HEAP"));
  if (check_heap && P.multipath) JB_RC(dev_alloc(d, (size_t)mu * (maxt + 4), &P.heap_chk));
  if (P.lmc_bits > 0) {
    JB_RC(dev_alloc_shared(d, (size_t)1 << P.lmc_bits, &P.lmc));
    JB_CUDA(cudaMemsetAsync(P.lmc, 0xff, sizeof(unsigned long long) << P.lmc_bits, d->stream));
  }
  JB_RC(reset_slots(d, 0, mu));
  P.atoms_out_cap = (long long)mf * d->atoms_per_frame + (long long)mu * 64;
  const size_t atoms_cap = (size_t)P.atoms_out_cap;
  JB_RC(dev_alloc(d, atoms_cap, &P.atoms_raw));
  JB_RC(dev_alloc(d, atoms_cap, &P.newidx));
  JB_RC(dev_alloc(d, (size_t)mf + mu + 8, &P.group0));
  JB_RC(dev_alloc(d, (size_t)mf * 2 + 8, &P.counts));
  JB_RC(dev_alloc(d, atoms_cap, &P.atoms_out));
  JB_RC(dev_alloc(d, 1, &P.atom_counter));
  JB_RC(dev_alloc(d, (size_t)mu, &P.results));
  JB_RC(dev_alloc(d, (size_t)mu * MAX_WORDS, &P.words));
  JB_RC(dev_alloc(d, (size_t)mu * 8, &P.prof));
  JB_RC(dev_alloc(d, (size_t)mu + 1, &d->d_frame_off));
  JB_RC(dev_alloc(d, (size_t)mu + 1, &d->d_atom_off));
  JB_RC(dev_alloc(d, (size_t)mf * d->in.dim, &d->in.d_feats));
  JB_RC(dev_alloc(d, (size_t)mf * P.row_stride, &d->in.d_rows));
  JB_RC(host_alloc(d, (size_t)mu, &d->h_results));
  JB_RC(host_alloc(d, atoms_cap, &d->h_atoms));
  JB_RC(host_alloc(d, (size_t)mu * MAX_WORDS, &d->h_words));
  JB_RC(host_alloc(d, 1, &d->h_counter));
  JB_RC(dev_alloc(d, (size_t)MC * mu, &d->d_chunk));
  JB_RC(host_alloc(d, (size_t)MC * mu, &d->h_chunk));
  JB_RC(dev_alloc(d, (size_t)mu, &P.state));
  JB_CUDA(cudaMemset(P.state, 0, sizeof(UttState) * (size_t)mu));
  JB_RC(dev_alloc(d, (size_t)mu * MAX_WORDS, &P.interim_words));
  JB_RC(dev_alloc(d, (size_t)MC * (2 * mu + 1), &d->d_seg));
  JB_RC(host_alloc(d, (size_t)MC * (2 * mu + 1), &d->h_seg));
  JB_RC(host_alloc(d, (size_t)mu + 1, &d->h_aoff));
  JB_RC(host_alloc(d, (size_t)mu, &d->h_state));
  JB_RC(host_alloc(d, (size_t)mu * MAX_WORDS, &d->h_interim_words));
  P.rows = d->in.d_rows; P.frame_off = d->d_frame_off; P.atom_off = d->d_atom_off; P.chunk = d->d_chunk;
  // the scoring stream of the batch pipeline gets the higher priority: its thread blocks take the room the token-passing
  // kernel leaves on every SM as soon as it is free
  int lo = 0, hi = 0;
  JB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  JB_CUDA(cudaStreamCreateWithPriority(&d->score_stream, cudaStreamNonBlocking, hi));
  for (auto &e : d->ev_slice) JB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  JB_CUDA(cudaEventCreate(&d->ev_score_begin)); JB_CUDA(cudaEventCreate(&d->ev_score_end));
  if (const char *e = getenv("JB200_PIPE_FRAMES")) d->pipe_frames = std::max(0, atoi(e));
  d->smem_bytes = cs.smem_bytes;
  d->beam = beam_kernel_for(t->lm_type == JB200_LM_DFA, P.multipath, check_heap);
  const void *kern = (const void *)d->beam;
  // the limit belongs to the kernel, which decoders of other beam widths share: only ever raise it
  cudaFuncAttributes fa;
  JB_CUDA(cudaFuncGetAttributes(&fa, kern));
  if ((size_t)fa.maxDynamicSharedSizeBytes < d->smem_bytes)
    JB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d->smem_bytes));
  int per_sm = 0, sms = 0;
  JB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, BEAM_THREADS, d->smem_bytes));
  JB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, d->device));
  d->resident = per_sm * sms;
  JB_CUDA(cudaStreamSynchronize(d->stream));
  return JB200_OK;
}

// the device half of jb200_decoder_create, on a checked tree
static int build_decoder(jb200_decoder *d, const jb200_tree_desc *t, jb200_gmm *am, int max_utts, int max_frames) {
  d->in.am = am; d->device = gmm_device(am); d->in.dim = gmm_dim(am); d->in.S = jb200_gmm_n_states(am);
  d->in.row_stride = d->P.row_stride = (d->in.S + 3) & ~3;
  d->max_utts = d->in.max_utts = max_utts; d->max_frames = d->in.max_frames = max_frames;
  if (const char *e = getenv("JB200_ATOMS_PER_FRAME")) d->atoms_per_frame = std::max(4, atoi(e));
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
  for (auto &e : d->ev) JB_CUDA(cudaEventCreate(&e));
  // bigram-factoring memo, 2^21 entries: keys are (word id, successor slot) packed 16+16, so it needs both below 65535
  d->P.lmc_bits = (t->n_words >= 65535 || t->n_scword >= 65535) ? 0 : 21;
  // shared read-only tables: nodes 32 B, arcs 8 B, context table, inter-word table, bigram memo, LM arrays (+ slack)
  const size_t est = (size_t)t->n_nodes * 32 + (size_t)t->n_arcs * 8 * 3 + (size_t)t->n_rset * (t->n_ctx + 1) * 4 + (size_t)t->n_words * 32 +
                     (size_t)t->n_words * std::max(t->n_iso, 1) * (t->lm_type == JB200_LM_DFA ? 1 : 4) + ((size_t)8 << d->P.lmc_bits) +
                     (size_t)t->lm_nvocab * 16 + (size_t)t->lm_nbigram * 8 + (size_t)(t->n_iso + t->n_shared + t->n_fscore + t->n_scword) * 16 + (4u << 20);
  if (cudaMalloc(&d->arena, est) == cudaSuccess) { d->arena_size = est; d->dev_allocs.push_back(d->arena); }
  else { d->arena = nullptr; cudaGetLastError(); }
  JB_RC(upload_tree(d, t));
  JB_RC(upload_lm(d, t));
  int smem_optin = 0;
  JB_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, d->device));
  CutSizing cs;
  JB_RC(size_cut(t->beam_width, t->n_start, smem_optin, &cs));
  return alloc_work(d, t, cs);
}

extern "C" int jb200_decoder_create(const jb200_tree_desc *t, jb200_gmm *am, int max_utts, int max_frames, jb200_decoder **out) {
  if (!t || !out || max_utts < 1 || max_frames < 1) { set_error("jb200_decoder_create: bad argument"); return JB200_ERR_ARG; }
  JB_RC(check_tree(t));
  if (!am) { set_error("jb200_decoder_create: no acoustic model"); return JB200_ERR_ARG; }
  jb200_decoder *d = new jb200_decoder();
  const int rc = build_decoder(d, t, am, max_utts, max_frames);
  if (rc) { jb200_decoder_destroy(d); return rc; }
  *out = d;
  return JB200_OK;
}

// Lays out n_utts utterances: frame_off (n_utts + 1 entries) becomes h_frame_off, and an utterance of T frames gets room
// for T * atoms_per_frame + 64 atoms from h_aoff[u] on.  Both go to the device on the main stream.
static int layout_utts(jb200_decoder *d, const int32_t *frame_off, int n_utts) {
  d->h_aoff[0] = 0;
  for (int u = 0; u < n_utts; u++) {
    const int T = frame_off[u + 1] - frame_off[u];
    if (T < 0 || T > 32767) { set_error("utterance %d has %d frames (trellis times are 16-bit in the reference)", u, T); return JB200_ERR_ARG; }
    d->h_aoff[u + 1] = d->h_aoff[u] + (long long)T * d->atoms_per_frame + 64;
  }
  d->h_frame_off.assign(frame_off, frame_off + n_utts + 1);
  JB_CUDA(cudaMemcpyAsync(d->d_frame_off, d->h_frame_off.data(), sizeof(int) * (n_utts + 1), cudaMemcpyHostToDevice, d->stream));
  JB_CUDA(cudaMemcpyAsync(d->d_atom_off, d->h_aoff, sizeof(long long) * (n_utts + 1), cudaMemcpyHostToDevice, d->stream));
  return JB200_OK;
}

// Cut a batch into time slices.  One slice (the whole utterance per launch) unless the pipeline is on: then slice c holds
// frames [c*F, (c+1)*F) of every utterance, scored by its own launch on the scoring stream (a gather over the segment
// list) while the beam kernel works on slice c-1.  Fills the staging copies of the chunk descriptors and segment lists.
static void plan_slices(jb200_decoder *d, const int32_t *frame_off, int n_utts, bool allow_pipe) {
  int maxT = 0;
  for (int u = 0; u < n_utts; u++) maxT = std::max(maxT, frame_off[u + 1] - frame_off[u]);
  int F = (allow_pipe && !d->in.dnn && d->pipe_frames > 0) ? d->pipe_frames : 0;
  int nch = 1;
  if (F > 0) {
    nch = (maxT + F - 1) / F;
    if (nch > jb200_decoder::MAX_CHUNKS) { F = (maxT + jb200_decoder::MAX_CHUNKS - 1) / jb200_decoder::MAX_CHUNKS; nch = (maxT + F - 1) / F; }
    if (nch < 2) { nch = 1; F = 0; }
  }
  d->n_chunks = nch; d->last_piped = (F > 0);
  d->slice_nseg.assign(nch, 0); d->slice_frames.assign(nch, 0);
  const int mu = d->max_utts, segw = 2 * mu + 1;
  for (int c = 0; c < nch; c++) {
    ChunkDesc *cd = d->h_chunk + (size_t)c * mu;
    int *so = d->h_seg + (size_t)c * segw, *ss = so + mu + 1;     // seg_off [mu+1], seg_start [mu]
    int nseg = 0, lf = 0;
    for (int u = 0; u < n_utts; u++) {
      const int T = frame_off[u + 1] - frame_off[u];
      ChunkDesc k;
      k.row_base = frame_off[u];
      if (F == 0) { k.t0 = 0; k.t1 = T; k.flags = CHUNK_FIRST | CHUNK_FINAL; }
      else {
        k.t0 = std::min(c * F, T); k.t1 = std::min((c + 1) * F, T);
        const bool past = (c > 0) && (c * F >= T);             // the utterance ended in an earlier slice
        const bool last = ((c + 1) * F >= T);
        k.flags = past ? CHUNK_SKIP : ((c == 0 ? CHUNK_FIRST : 0) | (last ? CHUNK_FINAL : 0));
        if (!past && k.t1 > k.t0) { so[nseg] = lf; ss[nseg] = frame_off[u] + k.t0; nseg++; lf += k.t1 - k.t0; }
      }
      cd[u] = k;
    }
    so[nseg] = lf;
    d->slice_nseg[c] = nseg; d->slice_frames[c] = lf;
  }
}

// a batch of n_utts utterances whose decoded frames start at frame_off fits the capacity of s
static int check_batch(const RowSource &s, const int32_t *frame_off, int n_utts) {
  if (!frame_off || n_utts < 1) { set_error("decode: bad argument"); return JB200_ERR_ARG; }
  if (n_utts > s.max_utts) { set_error("batch of %d utterances exceeds decoder capacity %d", n_utts, s.max_utts); return JB200_ERR_CAPACITY; }
  const int total = frame_off[n_utts] - frame_off[0];
  if (frame_off[0] != 0) { set_error("frame_off[0] must be 0"); return JB200_ERR_ARG; }
  if (total > s.max_frames) { set_error("batch of %d frames exceeds decoder capacity %d", total, s.max_frames); return JB200_ERR_CAPACITY; }
  return JB200_OK;
}

static int prepare_batch(jb200_decoder *d, const int32_t *frame_off, int n_utts, bool allow_pipe) {
  if (!d) { set_error("decode: bad argument"); return JB200_ERR_ARG; }
  JB_RC(check_batch(d->in, frame_off, n_utts));
  const int total = frame_off[n_utts];
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaStreamSynchronize(d->stream));   // the staging buffers below may still feed the previous batch's copies
  JB_RC(layout_utts(d, frame_off, n_utts));
  d->stream_mode = false; d->stream_group = nullptr;
  plan_slices(d, frame_off, n_utts, allow_pipe);
  const int mu = d->max_utts;
  JB_CUDA(cudaMemcpyAsync(d->d_chunk, d->h_chunk, sizeof(ChunkDesc) * (size_t)d->n_chunks * mu, cudaMemcpyHostToDevice, d->stream));
  if (d->last_piped)
    JB_CUDA(cudaMemcpyAsync(d->d_seg, d->h_seg, sizeof(int) * (size_t)d->n_chunks * (2 * mu + 1), cudaMemcpyHostToDevice, d->stream));
  JB_CUDA(cudaMemsetAsync(d->P.atom_counter, 0, sizeof(unsigned long long), d->stream));
  JB_CUDA(cudaStreamSynchronize(d->stream));   // h_frame_off is a std::vector (pageable)
  d->last_n = n_utts; d->last_total_frames = total; d->fetched = false;
  return JB200_OK;
}

// the beam kernel over chunk chunk_index of n_utts utterances; rows: a group's score rows instead of the decoder's own
static int launch_beam(jb200_decoder *d, int n_utts, int chunk_index, int interim = 0, const float *rows = nullptr) {
  BeamParams P = d->P;
  if (rows) P.rows = rows;
  P.chunk = d->d_chunk + (size_t)chunk_index * d->max_utts;
  P.interim = interim; P.atoms_in_place = d->stream_mode ? 1 : 0;
  d->beam<<<n_utts, BEAM_THREADS, d->smem_bytes, d->stream>>>(P);
  JB_LAUNCH_CHECK();
  return JB200_OK;
}

// scores T frames of device features into the source's score rows, on stream st; a splicing DNN reads its input rows
// through sm
static int score_frames(RowSource &s, cudaStream_t st, const float *d_feats, int T, const SpliceMap &sm = SpliceMap()) {
  return s.dnn ? dnn_forward_device(s.dnn, d_feats, T, s.d_rows, s.row_stride, st, sm)
               : gmm_launch_states(s.am, d_feats, T, s.d_rows, s.row_stride, st, nullptr, nullptr, 0);
}

// scoring of a prepared batch's features at d_feats, time slice by time slice on the scoring stream, beside the token
// passing of the slices on the main stream; ev[1] has been recorded on the main stream
static int run_pipeline(jb200_decoder *d, const float *d_feats, int n_utts) {
  // every slice's scoring is queued on the scoring stream at once (it only depends on the features), the beam kernel of
  // slice c waits for the scores of slice c alone
  const int mu = d->max_utts, segw = 2 * mu + 1;
  JB_CUDA(cudaStreamWaitEvent(d->score_stream, d->ev[1], 0));
  JB_CUDA(cudaEventRecord(d->ev_score_begin, d->score_stream));
  for (int c = 0; c < d->n_chunks; c++) {
    const int *ds = d->d_seg + (size_t)c * segw;
    JB_RC(gmm_launch_states(d->in.am, d_feats, d->slice_frames[c], d->in.d_rows, d->P.row_stride, d->score_stream, ds, ds + mu + 1, d->slice_nseg[c]));
    JB_CUDA(cudaEventRecord(d->ev_slice[c], d->score_stream));
  }
  JB_CUDA(cudaEventRecord(d->ev_score_end, d->score_stream));
  for (int c = 0; c < d->n_chunks; c++) {
    JB_CUDA(cudaStreamWaitEvent(d->stream, d->ev_slice[c], 0));
    if (c == 0) JB_CUDA(cudaEventRecord(d->ev[2], d->stream));       // "scoring" = what the beam had to wait for
    JB_RC(launch_beam(d, n_utts, c));
  }
  return JB200_OK;
}

// The phase times of the last batch: ev[0..4] bracket the upload, the scoring, the beam and the copy of the results.
// The last is 0 when the results were not fetched.
static void read_timing(jb200_decoder *d, bool fetched) {
  for (int i = 0; i < 3; i++) cudaEventElapsedTime(&d->last_ms[i], d->ev[i], d->ev[i + 1]);
  d->last_ms[3] = 0.0f;
  if (fetched) cudaEventElapsedTime(&d->last_ms[3], d->ev[3], d->ev[4]);
  if (d->last_piped) cudaEventElapsedTime(&d->last_score_busy_ms, d->ev_score_begin, d->ev_score_end);
}

extern "C" int jb200_decoder_fetch(jb200_decoder *d) {
  if (!d) { set_error("null decoder"); return JB200_ERR_ARG; }
  if (d->fetched) return JB200_OK;
  const BeamParams &P = d->P;
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaEventRecord(d->ev[3], d->stream));
  JB_CUDA(cudaMemcpyAsync(d->h_counter, P.atom_counter, sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
  JB_CUDA(cudaMemcpyAsync(d->h_results, P.results, sizeof(jb200_utt_result) * d->last_n, cudaMemcpyDeviceToHost, d->stream));
  JB_CUDA(cudaMemcpyAsync(d->h_words, P.words, sizeof(int) * (size_t)d->last_n * MAX_WORDS, cudaMemcpyDeviceToHost, d->stream));
  JB_CUDA(cudaStreamSynchronize(d->stream));
  long long na = (long long)*d->h_counter;
  if (na > P.atoms_out_cap) na = P.atoms_out_cap;
  if (na > 0) JB_CUDA(cudaMemcpyAsync(d->h_atoms, P.atoms_out, sizeof(jb200_atom) * (size_t)na, cudaMemcpyDeviceToHost, d->stream));
  JB_CUDA(cudaEventRecord(d->ev[4], d->stream));
  JB_CUDA(cudaStreamSynchronize(d->stream));
  read_timing(d, true);
  d->last_d2h = (long long)sizeof(unsigned long long) + (long long)sizeof(jb200_utt_result) * d->last_n +
                (long long)sizeof(int) * d->last_n * MAX_WORDS + (long long)sizeof(jb200_atom) * na;
  d->fetched = true;
  return JB200_OK;
}

extern "C" int jb200_decoder_sync_timing(jb200_decoder *d) {
  if (!d) { set_error("null decoder"); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaEventSynchronize(d->ev[3]));
  read_timing(d, false);
  return JB200_OK;
}

extern "C" int jb200_decoder_phase_cycles(jb200_decoder *d, int64_t *cycles, int n_utts) {
  if (!d || !cycles || n_utts < 1 || n_utts > d->last_n) { set_error("bad argument"); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaMemcpy(cycles, d->P.prof, sizeof(long long) * 8 * (size_t)n_utts, cudaMemcpyDeviceToHost));
  return JB200_OK;
}

// a row source's splice set-up for input frames fl wide, ctx to a network input: with ctx > 1 the segment table and the
// carry of max_utts streams
template <typename Owner>
static int reserve_splice(Owner *o, RowSource &s, int ctx, int fl) {
  if (ctx > 1) {
    if (!s.d_splice) {
      JB_RC(dev_alloc(o, (size_t)s.max_utts + 1, &s.d_splice));
      JB_RC(host_alloc(o, (size_t)s.max_utts + 1, &s.h_splice));
    }
    const size_t carry = (size_t)s.max_utts * (ctx - 1) * fl;
    if (carry > s.carry_floats) {
      for (auto &c : s.d_carry) JB_RC(dev_alloc(o, carry, &c));
      s.carry_floats = carry;
    }
  }
  s.ctx = ctx; s.fl = fl;
  return JB200_OK;
}

extern "C" int jb200_decoder_attach_dnn(jb200_decoder *d, jb200_dnn *dnn) {
  if (!d || !dnn) { set_error("null argument"); return JB200_ERR_ARG; }
  if (jb200_dnn_out_dim(dnn) != d->in.S) { set_error("DNN has %d outputs but the HMM set has %d states", jb200_dnn_out_dim(dnn), d->in.S); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(d->device));
  const int dim = jb200_dnn_in_dim(dnn);
  if (dim != d->in.dim) {
    // the feature buffer was sized for the AM's dimension; re-size it for the DNN's input width
    float *nf = nullptr;
    JB_RC(dev_alloc(d, (size_t)d->max_frames * dim, &nf));
    d->in.d_feats = nf; d->in.dim = dim;
  }
  // input frames of a splicing DNN are dim / ctx wide: max_frames network inputs' worth of them fit in d_feats as it is
  const int ctx = dnn_fix_context(dnn);
  JB_RC(reserve_splice(d, d->in, ctx, dim / ctx));
  d->in.dnn = dnn;
  return JB200_OK;
}

// copies the beam-cut counters [first, first + n) to out
static int read_cut_counters(jb200_decoder *d, CutCounter first, int n, int64_t *out) {
  if (!d || !out) { set_error("bad argument"); return JB200_ERR_ARG; }
  unsigned long long v[CUT_SLOTS];
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaMemcpy(v, d->P.cut_counters + first, sizeof(v[0]) * n, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; i++) out[i] = (int64_t)v[i];
  return JB200_OK;
}

extern "C" int64_t jb200_decoder_misspeculations(jb200_decoder *d) {
  int64_t v = 0;
  return read_cut_counters(d, CUT_SEQ_FALLBACKS, 1, &v) == JB200_OK ? v : -1;
}

extern "C" int jb200_decoder_heap_stats(jb200_decoder *d, int64_t out[3]) {
  return read_cut_counters(d, CUT_SEQ_FALLBACKS, 3, out);     // fall-backs, replay ticks, extractions replayed
}

extern "C" int jb200_decoder_select_stats(jb200_decoder *d, int64_t out[2]) {
  return read_cut_counters(d, CUT_UPWARD, 2, out);            // upward selects, of which closed form
}

extern "C" int64_t jb200_decoder_relocated_selects(jb200_decoder *d) {
  int64_t v = 0;
  return read_cut_counters(d, CUT_RELOCATED, 1, &v) == JB200_OK ? v : -1;
}

extern "C" int jb200_decoder_cut_placement(jb200_decoder *d, int64_t out[3]) {
  if (!d || !out) { set_error("bad argument"); return JB200_ERR_ARG; }
  JB_RC(read_cut_counters(d, CUT_GLOBAL_WHOLE, 2, out + 1));  // whole-heap copies, top-and-tail copies
  out[0] = d->P.heap_g ? 1 : 0;
  return JB200_OK;
}

extern "C" int64_t jb200_decoder_last_d2h_bytes(const jb200_decoder *d) { return d ? d->last_d2h : 0; }
extern "C" int jb200_decoder_resident_utts(const jb200_decoder *d) { return d ? d->resident : 0; }

// What a batch call hands in: features on the device, features on the host, or score rows on the host
enum BatchInput { FEATS_DEVICE, FEATS_HOST, SCORES_HOST };

// A batch for a splicing DNN: frame_off counts input frames, and utterance u of N_u of them decodes
// max(0, N_u - ctx + 1) frames (an input shorter than the window decodes none, Julius' "input too short",
// wav2mfcc.c:132-135).  rows_off gets the offsets of the decoded frames.
static int splice_rows(const RowSource &s, bool host_feats, const int32_t *frame_off, int n_utts, std::vector<int32_t> &rows_off) {
  if (!frame_off || n_utts < 1) { set_error("decode: bad argument"); return JB200_ERR_ARG; }
  if (frame_off[0] != 0) { set_error("frame_off[0] must be 0"); return JB200_ERR_ARG; }
  rows_off.assign(n_utts + 1, 0);
  for (int u = 0; u < n_utts; u++) {
    const int N = frame_off[u + 1] - frame_off[u];
    if (N < 0) { set_error("utterance %d has %d input frames", u, N); return JB200_ERR_ARG; }
    rows_off[u + 1] = rows_off[u] + std::max(0, N - s.ctx + 1);
  }
  if (host_feats && (long long)frame_off[n_utts] * s.fl > (long long)s.max_frames * s.dim) {
    set_error("batch of %d input frames exceeds decoder capacity %d", frame_off[n_utts], s.max_frames * s.ctx);
    return JB200_ERR_CAPACITY;
  }
  return JB200_OK;
}

// Getting a batch's rows, step 1, on the host: *rows gets the offsets of the decoded frames, which are frame_off unless
// a splicing DNN takes features (then they are kept in rows_off).
static int batch_rows_off(const RowSource &s, BatchInput in, const float *x, const int32_t *frame_off, int n_utts,
                          std::vector<int32_t> &rows_off, const int32_t **rows) {
  if (in != FEATS_DEVICE && !x) { set_error(in == SCORES_HOST ? "null scores" : "null feats"); return JB200_ERR_ARG; }
  *rows = frame_off;
  if (in != SCORES_HOST && s.splices()) {
    JB_RC(splice_rows(s, in == FEATS_HOST, frame_off, n_utts, rows_off));
    *rows = rows_off.data();
  }
  return JB200_OK;
}

// Getting a batch's rows, step 2, on stream st once the batch is laid out: uploads what the call hands in, records ev_in,
// and with score scores the features into s.d_rows.  *d_x gets the features on the device (for the batch pipeline, which
// scores them itself).  The staging segment table must be free: st has no copy from it pending.
static int batch_rows(RowSource &s, cudaStream_t st, BatchInput in, const float *x, const int32_t *frame_off, const int32_t *rows,
                      int n_utts, cudaEvent_t ev_in, bool score, const float **d_x) {
  const bool splice = in != SCORES_HOST && s.splices();
  const int total = rows[n_utts];
  SpliceMap sm;
  if (splice) {
    // utterance u's decoded frames read the windows of its own input frames
    for (int u = 0; u <= n_utts; u++)
      s.h_splice[u] = SpliceSeg{rows[u], frame_off[u], 0, 0, u < n_utts ? frame_off[u + 1] - frame_off[u] : 0};
    JB_CUDA(cudaMemcpyAsync(s.d_splice, s.h_splice, sizeof(SpliceSeg) * (n_utts + 1), cudaMemcpyHostToDevice, st));
    sm.seg = s.d_splice; sm.nseg = n_utts;
  }
  if (in == FEATS_HOST) {
    const size_t n = splice ? (size_t)frame_off[n_utts] * s.fl : (size_t)total * s.dim;
    JB_CUDA(cudaMemcpyAsync(s.d_feats, x, sizeof(float) * n, cudaMemcpyHostToDevice, st));
    x = s.d_feats;
  }
  if (in == SCORES_HOST)
    JB_CUDA(cudaMemcpy2DAsync(s.d_rows, sizeof(float) * s.row_stride, x, sizeof(float) * s.S, sizeof(float) * s.S, total,
                              cudaMemcpyHostToDevice, st));
  JB_CUDA(cudaEventRecord(ev_in, st));
  *d_x = x;
  if (score && in != SCORES_HOST) JB_RC(score_frames(s, st, x, total, sm));
  return JB200_OK;
}

// One batch, ev[0..3] around the upload, the scoring and the beam.  The host variants fetch the results; for device
// features that is left to jb200_decoder_fetch.  Score rows are never pipelined.
static int decode_batch(jb200_decoder *d, BatchInput in, const float *x, const int32_t *frame_off, int n_utts) {
  if (!d) { set_error("decode: bad argument"); return JB200_ERR_ARG; }
  std::vector<int32_t> rows_off;
  const int32_t *rows = nullptr;
  JB_RC(batch_rows_off(d->in, in, x, frame_off, n_utts, rows_off, &rows));
  JB_RC(prepare_batch(d, rows, n_utts, in != SCORES_HOST));
  JB_CUDA(cudaEventRecord(d->ev[0], d->stream));
  const float *d_x = nullptr;
  JB_RC(batch_rows(d->in, d->stream, in, x, frame_off, rows, n_utts, d->ev[1], !d->last_piped, &d_x));
  if (d->last_piped) {
    JB_RC(run_pipeline(d, d_x, n_utts));
  } else {
    JB_CUDA(cudaEventRecord(d->ev[2], d->stream));
    JB_RC(launch_beam(d, n_utts, 0));
  }
  if (in != FEATS_DEVICE) return jb200_decoder_fetch(d);
  JB_CUDA(cudaEventRecord(d->ev[3], d->stream));
  return JB200_OK;
}

extern "C" int jb200_decode_batch_device(jb200_decoder *d, const float *d_feats, const int32_t *frame_off, int n_utts) {
  return decode_batch(d, FEATS_DEVICE, d_feats, frame_off, n_utts);
}

extern "C" int jb200_decode_batch_host(jb200_decoder *d, const float *feats, const int32_t *frame_off, int n_utts) {
  return decode_batch(d, FEATS_HOST, feats, frame_off, n_utts);
}

extern "C" int jb200_decode_batch_scores_host(jb200_decoder *d, const float *scores, const int32_t *frame_off, int n_utts) {
  return decode_batch(d, SCORES_HOST, scores, frame_off, n_utts);
}

// ---- frame-synchronous operation (streams) -----------------------------------------------------------------------
extern "C" int jb200_stream_open(jb200_decoder *d, int n_streams) {
  if (!d || n_streams < 1) { set_error("jb200_stream_open: bad argument"); return JB200_ERR_ARG; }
  if (n_streams > d->max_utts) { set_error("%d streams exceed decoder capacity %d", n_streams, d->max_utts); return JB200_ERR_CAPACITY; }
  JB_CUDA(cudaSetDevice(d->device));
  JB_CUDA(cudaStreamSynchronize(d->stream));
  // a stream that was abandoned before its last frame has left node slots behind: wipe those work areas
  if (d->stream_mode)
    for (int u = 0; u < d->st_n; u++) if (d->st_started[u] && !d->st_done[u]) JB_RC(reset_slots(d, u, 1));
  const int cap = std::min(d->max_frames / n_streams, 32767);
  if (cap < 1) { set_error("decoder capacity of %d frames is too small for %d streams", d->max_frames, n_streams); return JB200_ERR_CAPACITY; }
  d->stream_mode = true; d->stream_group = nullptr; d->st_n = n_streams; d->st_cap = cap;
  d->st_t.assign(n_streams, 0); d->st_started.assign(n_streams, 0); d->st_done.assign(n_streams, 0); d->in.st_in.assign(n_streams, 0);
  std::vector<int32_t> frame_off(n_streams + 1);
  for (int u = 0; u <= n_streams; u++) frame_off[u] = u * cap;
  JB_RC(layout_utts(d, frame_off.data(), n_streams));
  JB_CUDA(cudaStreamSynchronize(d->stream));
  d->last_n = n_streams; d->n_chunks = 1; d->last_piped = false; d->fetched = true;
  return JB200_OK;
}

// Advancing the beams of a feed, step 1: the beam launch over the rows of the rows[s] new decoded frames of every stream,
// packed stream-major (rows: a group's score rows instead of the decoder's own), and the copies of what the feed
// returns.  *launched = false when no stream had anything to do.
static int stream_launch(jb200_decoder *d, const int32_t *rows, const uint8_t *last, int want_interim, const float *d_rows, bool *launched) {
  int pack = 0;
  bool any = false, fin_any = false;
  for (int u = 0; u < d->st_n; u++) {
    ChunkDesc k; k.t0 = d->st_t[u]; k.t1 = k.t0 + rows[u]; k.row_base = pack - k.t0; k.flags = 0;
    const bool fin = last && last[u];
    if (d->st_done[u] || (rows[u] == 0 && !fin)) k.flags = CHUNK_SKIP;
    else {
      if (!d->st_started[u]) k.flags |= CHUNK_FIRST;
      if (fin) k.flags |= CHUNK_FINAL;
      any = true; fin_any |= fin;
    }
    d->h_chunk[u] = k;
    pack += rows[u];
  }
  *launched = any;
  if (!any) return JB200_OK;
  const BeamParams &P = d->P;
  JB_CUDA(cudaMemcpyAsync(d->d_chunk, d->h_chunk, sizeof(ChunkDesc) * (size_t)d->st_n, cudaMemcpyHostToDevice, d->stream));
  JB_RC(launch_beam(d, d->st_n, 0, want_interim, d_rows));
  // results of the streams that ended; interim state of the others
  if (fin_any) {
    JB_CUDA(cudaMemcpyAsync(d->h_results, P.results, sizeof(jb200_utt_result) * d->st_n, cudaMemcpyDeviceToHost, d->stream));
    JB_CUDA(cudaMemcpyAsync(d->h_words, P.words, sizeof(int) * (size_t)d->st_n * MAX_WORDS, cudaMemcpyDeviceToHost, d->stream));
  }
  JB_CUDA(cudaMemcpyAsync(d->h_state, P.state, sizeof(UttState) * (size_t)d->st_n, cudaMemcpyDeviceToHost, d->stream));
  if (want_interim)
    JB_CUDA(cudaMemcpyAsync(d->h_interim_words, P.interim_words, sizeof(int) * (size_t)d->st_n * MAX_WORDS, cudaMemcpyDeviceToHost, d->stream));
  return JB200_OK;
}

// Advancing the beams of a feed, step 2, after a launch: waits for it, moves the streams on and fetches the atoms of the
// streams that ended
static int stream_collect(jb200_decoder *d) {
  const BeamParams &P = d->P;
  JB_CUDA(cudaStreamSynchronize(d->stream));
  d->last_d2h = 0;
  for (int u = 0; u < d->st_n; u++) {
    const int fl = d->h_chunk[u].flags;
    if (fl & CHUNK_SKIP) continue;
    d->st_started[u] = 1; d->st_t[u] = d->h_chunk[u].t1;
    if (fl & CHUNK_FINAL) {
      d->st_done[u] = 1;
      const int na = d->h_results[u].n_atoms;
      if (na > 0) JB_CUDA(cudaMemcpyAsync(d->h_atoms + d->h_aoff[u], P.atoms_out + d->h_aoff[u], sizeof(jb200_atom) * (size_t)na, cudaMemcpyDeviceToHost, d->stream));
      d->last_d2h += (long long)sizeof(jb200_atom) * na + (long long)sizeof(jb200_utt_result) + (long long)sizeof(int) * MAX_WORDS;
    }
  }
  JB_CUDA(cudaStreamSynchronize(d->stream));
  return JB200_OK;
}

// Getting a feed's rows, step 1: rows[s], the frames stream s decodes from its n_new[s] new ones.  For a splicing DNN the
// features are input frames: stream s's window is the last min(ctx - 1, have) frames it was fed before (have = its input
// frames so far) followed by its n_new[s] new ones, which give max(0, have + n_new[s] - ctx + 1) - max(0, have - ctx + 1)
// decoded frames (splice_mfcc: nothing until ctx frames have arrived, then one per frame).
static int feed_rows(const RowSource &s, bool scores, const int32_t *n_new, int n, std::vector<int32_t> &rows) {
  const bool splice = !scores && s.splices();
  rows.assign(n, 0);
  for (int u = 0; u < n; u++) {
    if (n_new[u] < 0) { set_error("stream %d: negative frame count", u); return JB200_ERR_ARG; }
    rows[u] = splice ? std::max(0, s.st_in[u] + n_new[u] - s.ctx + 1) - std::max(0, s.st_in[u] - s.ctx + 1) : n_new[u];
  }
  return JB200_OK;
}

// a decoder's streams can take rows[s] more frames each: none has ended, none goes past the per-stream capacity
static int check_feed(const jb200_decoder *d, const int32_t *n_new, const int32_t *rows) {
  for (int u = 0; u < d->st_n; u++) {
    if (d->st_done[u] && n_new[u] > 0) { set_error("stream %d has ended; restart it before feeding more frames", u); return JB200_ERR_ARG; }
    if (d->st_t[u] + rows[u] > d->st_cap) { set_error("stream %d: %d frames exceed the per-stream capacity %d", u, d->st_t[u] + rows[u], d->st_cap); return JB200_ERR_CAPACITY; }
  }
  return JB200_OK;
}

// Getting a feed's rows, step 2: the feed fits the buffers of s
static int feed_totals(const RowSource &s, bool scores, const float *x, const int32_t *n_new, const int32_t *rows, int n) {
  long long tot = 0, tot_rows = 0;
  for (int u = 0; u < n; u++) { tot += n_new[u]; tot_rows += rows[u]; }
  if (tot_rows > s.max_frames) { set_error("%lld new frames exceed decoder capacity %d", tot_rows, s.max_frames); return JB200_ERR_CAPACITY; }
  if (!scores && s.splices() && tot * s.fl > (long long)s.max_frames * s.dim) {
    set_error("%lld new input frames exceed decoder capacity %d", tot, s.max_frames * s.ctx);
    return JB200_ERR_CAPACITY;
  }
  if (tot > 0 && !x) { set_error(scores ? "null scores" : "null feats"); return JB200_ERR_ARG; }
  return JB200_OK;
}

// Getting a feed's rows, step 3, on stream st: uploads the new frames of every stream, packed stream-major, as features or
// as score rows, and scores the features into s.d_rows; a splicing DNN's streams move their carry on.
// ev_in (may be null) is recorded once the input is on the device.
static int feed_score(RowSource &s, cudaStream_t st, bool scores, const float *x, const int32_t *n_new, const int32_t *rows, int n,
                      cudaEvent_t ev_in) {
  int tot = 0, tot_rows = 0;
  for (int u = 0; u < n; u++) { tot += n_new[u]; tot_rows += rows[u]; }
  if (tot == 0) {
    if (ev_in) JB_CUDA(cudaEventRecord(ev_in, st));
    return JB200_OK;
  }
  if (scores) {
    JB_CUDA(cudaMemcpy2DAsync(s.d_rows, sizeof(float) * s.row_stride, x, sizeof(float) * s.S, sizeof(float) * s.S, tot, cudaMemcpyHostToDevice, st));
    if (ev_in) JB_CUDA(cudaEventRecord(ev_in, st));
  } else if (!s.splices()) {
    JB_CUDA(cudaMemcpyAsync(s.d_feats, x, sizeof(float) * (size_t)tot * s.dim, cudaMemcpyHostToDevice, st));
    if (ev_in) JB_CUDA(cudaEventRecord(ev_in, st));
    JB_RC(score_frames(s, st, s.d_feats, tot));
  } else {
    JB_CUDA(cudaStreamSynchronize(st));   // the staging segment table may still feed the last feed's copy
    int pack_in = 0, pack_rows = 0;
    for (int u = 0; u < n; u++) {
      const int have = std::min(s.ctx - 1, s.st_in[u]);
      s.h_splice[u] = SpliceSeg{pack_rows, pack_in, u * (s.ctx - 1), have, have + n_new[u]};
      pack_in += n_new[u]; pack_rows += rows[u];
    }
    s.h_splice[n] = SpliceSeg{pack_rows, pack_in, 0, 0, 0};
    JB_CUDA(cudaMemcpyAsync(s.d_splice, s.h_splice, sizeof(SpliceSeg) * (n + 1), cudaMemcpyHostToDevice, st));
    JB_CUDA(cudaMemcpyAsync(s.d_feats, x, sizeof(float) * (size_t)tot * s.fl, cudaMemcpyHostToDevice, st));
    if (ev_in) JB_CUDA(cudaEventRecord(ev_in, st));
    SpliceMap sm;
    sm.seg = s.d_splice; sm.nseg = n; sm.carry = s.d_carry[s.carry_cur];
    JB_RC(score_frames(s, st, s.d_feats, tot_rows, sm));
    // after the scoring has read the carry, in stream order: the new carry goes to the other buffer
    carry_update_kernel<<<n, 128, 0, st>>>(s.d_splice, s.d_feats, s.d_carry[s.carry_cur], s.d_carry[s.carry_cur ^ 1], s.ctx - 1, s.fl);
    JB_LAUNCH_CHECK();
    s.carry_cur ^= 1;
    for (int u = 0; u < n; u++) s.st_in[u] += n_new[u];
  }
  return JB200_OK;
}

// jb200_stream_feed_host / _scores_host: the new frames of every stream, packed stream-major, as features or as score rows
static int stream_feed(jb200_decoder *d, bool scores, const float *x, const int32_t *n_new, const uint8_t *last, int want_interim) {
  if (!d || !n_new) { set_error("jb200_stream_feed: bad argument"); return JB200_ERR_ARG; }
  if (!d->stream_mode) { set_error("jb200_stream_feed: call jb200_stream_open first"); return JB200_ERR_ARG; }
  if (d->stream_group) { set_error("jb200_stream_feed: the decoder is in an open group stream; feed the group"); return JB200_ERR_ARG; }
  std::vector<int32_t> rows;                    // decoded frames of each stream in this feed
  JB_RC(feed_rows(d->in, scores, n_new, d->st_n, rows));
  JB_RC(check_feed(d, n_new, rows.data()));
  JB_RC(feed_totals(d->in, scores, x, n_new, rows.data(), d->st_n));
  JB_CUDA(cudaSetDevice(d->device));
  JB_RC(feed_score(d->in, d->stream, scores, x, n_new, rows.data(), d->st_n, nullptr));
  bool launched = false;
  JB_RC(stream_launch(d, rows.data(), last, want_interim, nullptr, &launched));
  return launched ? stream_collect(d) : JB200_OK;
}

extern "C" int jb200_stream_feed_host(jb200_decoder *d, const float *feats, const int32_t *n_new, const uint8_t *last, int want_interim) {
  return stream_feed(d, false, feats, n_new, last, want_interim);
}

extern "C" int jb200_stream_feed_scores_host(jb200_decoder *d, const float *scores, const int32_t *n_new, const uint8_t *last, int want_interim) {
  return stream_feed(d, true, scores, n_new, last, want_interim);
}

extern "C" int jb200_stream_restart(jb200_decoder *d, int stream) {
  if (!d || !d->stream_mode || stream < 0 || stream >= d->st_n) { set_error("jb200_stream_restart: bad argument"); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(d->device));
  if (d->st_started[stream] && !d->st_done[stream]) {
    JB_RC(reset_slots(d, stream, 1));
    JB_CUDA(cudaStreamSynchronize(d->stream));
  }
  d->st_t[stream] = 0; d->st_started[stream] = 0; d->st_done[stream] = 0; d->in.st_in[stream] = 0;
  return JB200_OK;
}

extern "C" int jb200_stream_status(jb200_decoder *d, int stream, int32_t *frames_done, int32_t *alive, int32_t *ended) {
  if (!d || !d->stream_mode || stream < 0 || stream >= d->st_n) { set_error("jb200_stream_status: bad argument"); return JB200_ERR_ARG; }
  if (frames_done) *frames_done = d->st_t[stream];
  if (alive) *alive = (!d->st_started[stream] || d->st_done[stream]) ? 1 : (d->h_state[stream].stopped < 0);
  if (ended) *ended = d->st_done[stream];
  return JB200_OK;
}

extern "C" int jb200_stream_partial(jb200_decoder *d, int stream, int32_t *words, int max_words, int32_t *n_words, float *score, int32_t *frame) {
  if (!d || !d->stream_mode || stream < 0 || stream >= d->st_n || !n_words) { set_error("jb200_stream_partial: bad argument"); return JB200_ERR_ARG; }
  if (!d->st_started[stream] || d->st_done[stream]) { *n_words = 0; if (score) *score = JB200_LOG_ZERO; if (frame) *frame = -1; return JB200_OK; }
  const UttState &st = d->h_state[stream];
  const int n = std::min(st.interim_nwords, std::max(max_words, 0));
  for (int i = 0; i < n && words; i++) words[i] = d->h_interim_words[(size_t)stream * MAX_WORDS + i];
  *n_words = words ? n : st.interim_nwords;
  if (score) *score = st.interim_score;
  if (frame) *frame = st.interim_frame;
  return JB200_OK;
}

extern "C" int jb200_stream_result(jb200_decoder *d, int stream, const jb200_utt_result **utt, const jb200_atom **atoms, const int32_t **words) {
  if (!d || !d->stream_mode || stream < 0 || stream >= d->st_n) { set_error("jb200_stream_result: bad argument"); return JB200_ERR_ARG; }
  if (!d->st_done[stream]) { set_error("stream %d has not ended", stream); return JB200_ERR_ARG; }
  if (utt) *utt = d->h_results + stream;
  if (atoms) *atoms = d->h_atoms;        // index with utt->atom_offset, as for a batch
  if (words) *words = d->h_words;        // index with utt->word_offset
  return JB200_OK;
}

extern "C" int jb200_decoder_pipeline_info(jb200_decoder *d, int32_t *n_slices, float *score_busy_ms) {
  if (!d) { set_error("null decoder"); return JB200_ERR_ARG; }
  if (n_slices) *n_slices = d->last_piped ? d->n_chunks : 1;
  if (score_busy_ms) *score_busy_ms = d->last_piped ? d->last_score_busy_ms : 0.0f;
  return JB200_OK;
}

extern "C" int jb200_decoder_set_pipeline(jb200_decoder *d, int frames_per_slice) {
  if (!d || frames_per_slice < 0) { set_error("jb200_decoder_set_pipeline: bad argument"); return JB200_ERR_ARG; }
  d->pipe_frames = frames_per_slice;
  return JB200_OK;
}

extern "C" int jb200_decoder_results(jb200_decoder *d, const jb200_utt_result **utts, const jb200_atom **atoms, const int32_t **words) {
  if (!d) { set_error("null decoder"); return JB200_ERR_ARG; }
  if (!d->fetched) { int rc = jb200_decoder_fetch(d); if (rc) return rc; }
  if (utts) *utts = d->h_results;
  if (atoms) *atoms = d->h_atoms;
  if (words) *words = d->h_words;
  return JB200_OK;
}

extern "C" int jb200_decoder_last_timing(jb200_decoder *d, float ms[4]) {
  if (!d || !ms) { set_error("bad argument"); return JB200_ERR_ARG; }
  for (int i = 0; i < 4; i++) ms[i] = d->last_ms[i];
  return JB200_OK;
}

extern "C" int jb200_decoder_frame_counts(jb200_decoder *d, int u, int32_t *counts, int max_frames) {
  if (!d || !counts || u < 0 || u >= d->last_n) { set_error("bad argument"); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(d->device));
  const int f0 = d->h_frame_off[u], T = d->h_frame_off[u + 1] - f0;
  const int n = T < max_frames ? T : max_frames;
  JB_CUDA(cudaMemcpy(counts, d->P.counts + (size_t)f0 * 2, sizeof(int) * 2 * n, cudaMemcpyDeviceToHost));
  return JB200_OK;
}

// ---- decoder groups (jb200_group_*): recognition instances on one acoustic model score each input once -------------
struct jb200_group {
  std::vector<jb200_decoder *> m;
  std::vector<char> active;
  std::vector<cudaEvent_t> beam_done;           // per member: its last beam over the group's rows, on its own stream
  int device = 0;
  RowSource in;                                 // the group's features, score rows and splice state
  std::vector<void *> dev_allocs, host_allocs;  // freed by jb200_group_destroy
  cudaStream_t stream = nullptr;
  // ev[0..4]: upload begins, input on the device, scored, every member's beam done, results copied back
  cudaEvent_t ev[5]{};
  bool timed = false, fetched = false;
  bool st_open = false; int st_n = 0;
};

extern "C" void jb200_group_destroy(jb200_group *g) {
  if (!g) return;
  cudaSetDevice(g->device);
  // the members' beams may still read the group's rows
  for (jb200_decoder *d : g->m) {
    cudaStreamSynchronize(d->stream);
    if (d->stream_group == g) d->stream_group = nullptr;
  }
  if (g->stream) cudaStreamSynchronize(g->stream);
  for (void *p : g->dev_allocs) cudaFree(p);
  for (void *p : g->host_allocs) cudaFreeHost(p);
  for (auto &e : g->ev) if (e) cudaEventDestroy(e);
  for (auto &e : g->beam_done) if (e) cudaEventDestroy(e);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
}

// the device half of jb200_group_create
static int build_group(jb200_group *g) {
  JB_CUDA(cudaSetDevice(g->device));
  JB_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
  for (auto &e : g->ev) JB_CUDA(cudaEventCreate(&e));
  for (auto &e : g->beam_done) JB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  RowSource &s = g->in;
  JB_RC(dev_alloc(g, (size_t)s.max_frames * s.dim, &s.d_feats));
  JB_RC(dev_alloc(g, (size_t)s.max_frames * s.row_stride, &s.d_rows));
  return reserve_splice(g, s, g->m[0]->in.ctx, g->m[0]->in.fl);
}

extern "C" int jb200_group_create(jb200_decoder *const *members, int n_members, jb200_group **out) {
  if (!members || !out || n_members < 1 || n_members > JB200_GROUP_MAX) {
    set_error("jb200_group_create: 1 to %d members", JB200_GROUP_MAX); return JB200_ERR_ARG;
  }
  const jb200_decoder *d0 = members[0];
  for (int i = 0; i < n_members; i++) {
    const jb200_decoder *d = members[i];
    if (!d) { set_error("jb200_group_create: member %d is null", i); return JB200_ERR_ARG; }
    for (int j = 0; j < i; j++)
      if (members[j] == d) { set_error("jb200_group_create: members %d and %d are the same decoder", j, i); return JB200_ERR_ARG; }
    if (d->in.am != d0->in.am || d->device != d0->device) {
      set_error("jb200_group_create: member %d uses another acoustic model than member 0", i); return JB200_ERR_ARG;
    }
    if (d->in.dnn != d0->in.dnn) { set_error("jb200_group_create: member %d has another DNN than member 0", i); return JB200_ERR_ARG; }
  }
  jb200_group *g = new jb200_group();
  g->m.assign(members, members + n_members);
  g->active.assign(n_members, 1);
  g->beam_done.assign(n_members, nullptr);
  g->device = d0->device;
  RowSource &s = g->in;
  s.am = d0->in.am; s.dnn = d0->in.dnn; s.dim = d0->in.dim; s.S = d0->in.S; s.row_stride = d0->in.row_stride;
  s.max_utts = d0->max_utts; s.max_frames = d0->max_frames;
  for (const jb200_decoder *d : g->m) { s.max_utts = std::min(s.max_utts, d->max_utts); s.max_frames = std::min(s.max_frames, d->max_frames); }
  const int rc = build_group(g);
  if (rc) { jb200_group_destroy(g); return rc; }
  *out = g;
  return JB200_OK;
}

extern "C" int jb200_group_set_active(jb200_group *g, int member, int active) {
  if (!g || member < 0 || member >= (int)g->m.size()) { set_error("jb200_group_set_active: bad argument"); return JB200_ERR_ARG; }
  // a stream that missed feeds, or got feeds its member did not, cannot go on: the change waits for the utterances' ends
  const jb200_decoder *d = g->m[member];
  if (g->st_open && (g->active[member] != 0) != (active != 0) && d->stream_group == g)
    for (int u = 0; u < d->st_n; u++)
      if (d->st_started[u] && !d->st_done[u]) {
        set_error("jb200_group_set_active: member %d is inside an utterance on stream %d; end or restart it first", member, u);
        return JB200_ERR_ARG;
      }
  g->active[member] = active ? 1 : 0;
  return JB200_OK;
}

// The start of a group call, once it has been checked: the group's stream waits (on the device) until no member's beam
// of an earlier call still reads the rows, then ev[0]
static int group_begin(jb200_group *g) {
  JB_CUDA(cudaSetDevice(g->device));
  for (cudaEvent_t e : g->beam_done) JB_CUDA(cudaStreamWaitEvent(g->stream, e, 0));
  JB_CUDA(cudaEventRecord(g->ev[0], g->stream));
  g->timed = true; g->fetched = false;
  return JB200_OK;
}

// Once the rows are scored (ev[2] on the group's stream): every active member's beam waits for them on its own stream.
// launch(i) launches member i's beam and tells whether it did; ev[3] follows the last of them.
template <typename Launch>
static int group_beams(jb200_group *g, Launch launch) {
  JB_CUDA(cudaEventRecord(g->ev[2], g->stream));
  for (size_t i = 0; i < g->m.size(); i++) {
    if (!g->active[i]) continue;
    jb200_decoder *d = g->m[i];
    JB_CUDA(cudaStreamWaitEvent(d->stream, g->ev[2], 0));
    JB_RC(launch(i));
    JB_CUDA(cudaEventRecord(g->beam_done[i], d->stream));
    JB_CUDA(cudaStreamWaitEvent(g->stream, g->beam_done[i], 0));
  }
  JB_CUDA(cudaEventRecord(g->ev[3], g->stream));
  return JB200_OK;
}

// ev[4] after the results of the active members have been copied back
static int group_fetched(jb200_group *g) {
  JB_CUDA(cudaEventRecord(g->ev[4], g->stream));
  g->fetched = true;
  return JB200_OK;
}

static int group_batch(jb200_group *g, BatchInput in, const float *x, const int32_t *frame_off, int n_utts) {
  if (!g) { set_error("null group"); return JB200_ERR_ARG; }
  RowSource &s = g->in;
  std::vector<int32_t> rows_off;
  const int32_t *rows = nullptr;
  JB_RC(batch_rows_off(s, in, x, frame_off, n_utts, rows_off, &rows));
  JB_RC(check_batch(s, rows, n_utts));          // the group's capacity is the smallest member's
  for (jb200_decoder *d : g->m) if (d->stream_group == g) d->stream_group = nullptr;
  g->st_open = false;
  for (size_t i = 0; i < g->m.size(); i++) if (g->active[i]) JB_RC(prepare_batch(g->m[i], rows, n_utts, false));
  if (rows != frame_off) {
    JB_CUDA(cudaSetDevice(g->device));
    JB_CUDA(cudaStreamSynchronize(g->stream));  // the staging segment table may still feed the last call's copy
  }
  JB_RC(group_begin(g));
  const float *d_x = nullptr;
  JB_RC(batch_rows(s, g->stream, in, x, frame_off, rows, n_utts, g->ev[1], true, &d_x));
  JB_RC(group_beams(g, [&](size_t i) {
    // the member's own timing: no upload or scoring of its own, then its beam
    jb200_decoder *d = g->m[i];
    for (int k = 0; k < 3; k++) JB_CUDA(cudaEventRecord(d->ev[k], d->stream));
    JB_RC(launch_beam(d, n_utts, 0, 0, s.d_rows));
    if (in == FEATS_DEVICE) JB_CUDA(cudaEventRecord(d->ev[3], d->stream));
    return JB200_OK;
  }));
  if (in == FEATS_DEVICE) return JB200_OK;
  for (size_t i = 0; i < g->m.size(); i++) if (g->active[i]) JB_RC(jb200_decoder_fetch(g->m[i]));
  return group_fetched(g);
}

extern "C" int jb200_group_decode_batch_host(jb200_group *g, const float *feats, const int32_t *frame_off, int n_utts) {
  return group_batch(g, FEATS_HOST, feats, frame_off, n_utts);
}

extern "C" int jb200_group_decode_batch_device(jb200_group *g, const float *d_feats, const int32_t *frame_off, int n_utts) {
  return group_batch(g, FEATS_DEVICE, d_feats, frame_off, n_utts);
}

extern "C" int jb200_group_decode_batch_scores_host(jb200_group *g, const float *scores, const int32_t *frame_off, int n_utts) {
  return group_batch(g, SCORES_HOST, scores, frame_off, n_utts);
}

extern "C" int jb200_group_stream_open(jb200_group *g, int n_streams) {
  if (!g || n_streams < 1) { set_error("jb200_group_stream_open: bad argument"); return JB200_ERR_ARG; }
  if (n_streams > g->in.max_utts) { set_error("%d streams exceed group capacity %d", n_streams, g->in.max_utts); return JB200_ERR_CAPACITY; }
  g->st_open = false;
  for (jb200_decoder *d : g->m) {
    JB_RC(jb200_stream_open(d, n_streams));
    d->stream_group = g;
  }
  g->in.st_in.assign(n_streams, 0);
  g->st_open = true; g->st_n = n_streams;
  return JB200_OK;
}

extern "C" int jb200_group_stream_restart(jb200_group *g, int stream) {
  if (!g || !g->st_open || stream < 0 || stream >= g->st_n) { set_error("jb200_group_stream_restart: bad argument"); return JB200_ERR_ARG; }
  for (size_t i = 0; i < g->m.size(); i++)
    if (g->active[i] && g->m[i]->stream_group == g) JB_RC(jb200_stream_restart(g->m[i], stream));
  g->in.st_in[stream] = 0;
  return JB200_OK;
}

static int group_feed(jb200_group *g, bool scores, const float *x, const int32_t *n_new, const uint8_t *last, int want_interim) {
  if (!g || !n_new) { set_error("jb200_group_stream_feed: bad argument"); return JB200_ERR_ARG; }
  if (!g->st_open) { set_error("jb200_group_stream_feed: call jb200_group_stream_open first"); return JB200_ERR_ARG; }
  for (size_t i = 0; i < g->m.size(); i++) {
    const jb200_decoder *d = g->m[i];
    if (g->active[i] && (d->stream_group != g || !d->stream_mode)) {
      set_error("jb200_group_stream_feed: member %zu has left the group's stream", i); return JB200_ERR_ARG;
    }
  }
  RowSource &s = g->in;
  std::vector<int32_t> rows;
  JB_RC(feed_rows(s, scores, n_new, g->st_n, rows));
  for (size_t i = 0; i < g->m.size(); i++) if (g->active[i]) JB_RC(check_feed(g->m[i], n_new, rows.data()));
  JB_RC(feed_totals(s, scores, x, n_new, rows.data(), g->st_n));
  JB_RC(group_begin(g));
  JB_RC(feed_score(s, g->stream, scores, x, n_new, rows.data(), g->st_n, g->ev[1]));
  std::vector<char> launched(g->m.size(), 0);
  JB_RC(group_beams(g, [&](size_t i) {
    bool l = false;
    JB_RC(stream_launch(g->m[i], rows.data(), last, want_interim, s.d_rows, &l));
    launched[i] = l;
    return JB200_OK;
  }));
  for (size_t i = 0; i < g->m.size(); i++) if (launched[i]) JB_RC(stream_collect(g->m[i]));
  return group_fetched(g);
}

extern "C" int jb200_group_stream_feed_host(jb200_group *g, const float *feats, const int32_t *n_new, const uint8_t *last, int want_interim) {
  return group_feed(g, false, feats, n_new, last, want_interim);
}

extern "C" int jb200_group_stream_feed_scores_host(jb200_group *g, const float *scores, const int32_t *n_new, const uint8_t *last, int want_interim) {
  return group_feed(g, true, scores, n_new, last, want_interim);
}

extern "C" int jb200_group_last_timing(jb200_group *g, float ms[4]) {
  if (!g || !ms) { set_error("bad argument"); return JB200_ERR_ARG; }
  for (int i = 0; i < 4; i++) ms[i] = 0.0f;
  if (!g->timed) return JB200_OK;
  JB_CUDA(cudaSetDevice(g->device));
  JB_CUDA(cudaEventSynchronize(g->ev[3]));
  for (int i = 0; i < 3; i++) JB_CUDA(cudaEventElapsedTime(&ms[i], g->ev[i], g->ev[i + 1]));
  if (g->fetched) {
    JB_CUDA(cudaEventSynchronize(g->ev[4]));
    JB_CUDA(cudaEventElapsedTime(&ms[3], g->ev[3], g->ev[4]));
  }
  return JB200_OK;
}
