#define _GNU_SOURCE
/* oracle/restate/beam.c -- TEST INFRASTRUCTURE (CPU restatement, see oracle.h).
 *
 * Frame-synchronous token passing on the flattened lexicon tree, restating
 *   get_back_trellis_init / init_nodescore   libjulius/src/beam.c:1825-1922, 1552-1665
 *   get_back_trellis_proceed (NORMAL MODE)   beam.c:2663-3019
 *   propagate_token                          beam.c:1945-1978
 *   beam_intra_word(_core)                   beam.c:2004-2177
 *   save_trellis                             beam.c:2209-2247
 *   beam_inter_word                          beam.c:2271-2517
 *   beam_inter_word_factoring                beam.c:2549-2616
 *   sort_token_upward/downward/no_order      beam.c:1342-1520   (heap select; order matters on ties)
 *   get_back_trellis_end / finalize_1st_pass beam.c:3052-3162
 *   find_1pass_result / trace_backptr        beam.c:253-301, 372-512
 *   outprob_style                            libjulius/src/outprob_style.c:354-494 (context table form)
 *   max_successor_prob(_iw)                  libjulius/src/factoring_sub.c:942-1143
 *   bi_prob_*                                libsent/src/ngram/ngram_access.c:249-466
 *   bt_relocate_rw / bt_sort_rw              libjulius/src/backtrellis.c:218-267, 438-478
 * for the stock "fast" build switches (UNIGRAM_FACTORING, LOWMEM2, PASS1_IWCD,
 * SCORE_PRUNING, no WPAIR/WORD_GRAPH), N-gram LM; both the NORMAL (:2838-2894) and the MULTIPATH
 * (:2752-2828, forced by -multipath or needed by the HMM topology) branches.
 * Sequential, same visiting order, same fp32 expression order.
 */
#include <math.h>
#include "oracle.h"

float oracle_cdset_one(const jb200_gmm_desc *g, const float *strow, int c, float *nbest_work);

typedef struct {
  int last_tre;       /* atom index, -1 = bos */
  int last_cword;     /* -1 = WORD_INVALID */
  float last_lscore;
  float score;
  int node;
} Tok;

typedef struct {
  const jb200_tree_desc *t;
  const jb200_gmm_desc *g;
  const float *st; int T, S;
  Tok *tlist[2]; int *tindex[2]; int tnum[2]; int maxtnum;
  int *token;              /* [n_nodes] -> token id in tn, -1 */
  int tn, tl, n_start, n_end;
  float wordend_best_score; int wordend_best_node, wordend_best_tre, wordend_best_last_cword;
  float score_pruning_threshold, score_pruning_max;
  /* trellis (creation order) */
  oracle_atom *atoms; int natoms, maxatoms;
  /* per-frame cdset memo */
  float *cdval; int *cdstamp; float *nbest_work;
  /* iw rows memo per last word */
  float *iwrow; int iwrow_word;
} Beam;

/* ---- LM ---------------------------------------------------------------------------- */
static int search_bigram(const jb200_tree_desc *t, int w_context, int w) {
  int left, right, mid;
  if ((left = t->bi_bgn[w_context]) < 0) return -1;
  right = left + t->bi_num[w_context] - 1;
  while (left < right) {
    mid = (left + right) / 2;
    if (t->bi_wid[mid] < w) left = mid + 1; else right = mid;
  }
  return (t->bi_wid[left] == w) ? left : -1;
}

static float bigram_prob(const jb200_tree_desc *t, int w1, int w2) {
  int n2; float prob;
  switch (t->lm_mode) {
    case JB200_BI_NORMAL:
    case JB200_BI_ADDITIONAL_OLDBIN:
      if ((n2 = search_bigram(t, w1, w2)) >= 0) prob = t->bi_prob[n2];
      else prob = t->uni_bow[w1] + t->uni_prob[w2];
      break;
    case JB200_BI_ADDITIONAL:
      if ((n2 = search_bigram(t, w2, w1)) >= 0) prob = t->bi_prob[n2];
      else prob = t->uni_bow[w1] + t->uni_prob[w2];
      break;
    default: /* JB200_BI_COMPUTE */
      if ((n2 = search_bigram(t, w2, w1)) >= 0) prob = t->bi_prob[n2];
      else prob = t->uni_bow[w2] + t->uni_prob[w1];
      prob = prob + t->uni_prob[w2] - t->uni_prob[w1];
      break;
  }
  if (w2 != t->lm_unk_id) return prob;
  return prob - t->lm_unk_num_log;
}

static float max_successor_prob(const jb200_tree_desc *t, int lastword, int node) {
  int scid, w;
  if (lastword < 0) return 0.0;
  scid = t->scid[node];
  if (scid < 0) return t->fscore[-scid];
  w = t->scword[scid];
  return bigram_prob(t, t->wton[lastword], t->wton[w]) + t->cprob[w];
}

static const float *max_successor_prob_iw(Beam *b, int lastword) {
  const jb200_tree_desc *t = b->t;
  int i;
  if (b->iwrow_word == lastword) return b->iwrow;
  for (i = 0; i < t->n_iso; i++) {
    int w = t->iso_word[i];
    b->iwrow[t->iso_id[i]] = bigram_prob(t, t->wton[lastword], t->wton[w]) + t->cprob[w];
  }
  b->iwrow_word = lastword;
  return b->iwrow;
}

/* ---- acoustic ------------------------------------------------------------------------ */
static float cdset(Beam *b, int c, int t) {
  if (b->cdstamp[c] != t) {
    b->cdval[c] = oracle_cdset_one(b->g, b->st + (size_t)t * b->S, c, b->nbest_work);
    b->cdstamp[c] = t;
  }
  return b->cdval[c];
}

static float outprob_style(Beam *b, int node, int last_wid, int t) {
  const jb200_tree_desc *tr = b->t;
  int ref = tr->out_ref[node];
  switch (tr->outstyle[node]) {
    case JB200_AS_STATE: return b->st[(size_t)t * b->S + ref];
    case JB200_AS_LSET:  return cdset(b, ref, t);
    default: {
      int col = (last_wid < 0) ? tr->n_ctx : tr->word_ctx[last_wid];
      int r = tr->rset_ctx[(size_t)ref * (tr->n_ctx + 1) + col];
      if (r >= 0) return b->st[(size_t)t * b->S + r];
      return cdset(b, -r - 1, t);
    }
  }
}

/* ---- tokens -------------------------------------------------------------------------- */
static void expand_tlist(Beam *b) {
  int k;
  b->maxtnum *= 2;
  for (k = 0; k < 2; k++) {
    b->tlist[k] = (Tok *)realloc(b->tlist[k], sizeof(Tok) * b->maxtnum);
    b->tindex[k] = (int *)realloc(b->tindex[k], sizeof(int) * b->maxtnum);
  }
}

static int create_token(Beam *b) {
  int tn = b->tn, newid = b->tnum[tn];
  b->tnum[tn]++;
  while (b->tnum[tn] >= b->maxtnum) expand_tlist(b);
  b->tindex[tn][newid] = newid;
  return newid;
}

static void propagate_token(Beam *b, int next_node, float next_score, int last_tre, int last_cword, float last_lscore) {
  Tok *tknext; int id;
  if (next_score <= JB200_LOG_ZERO) return;
  if ((id = b->token[next_node]) != -1) {
    tknext = &b->tlist[b->tn][id];
    if (tknext->score < next_score) {
      tknext->last_tre = last_tre; tknext->last_cword = last_cword;
      tknext->last_lscore = last_lscore; tknext->score = next_score;
    }
  } else {
    id = create_token(b);
    tknext = &b->tlist[b->tn][id];
    tknext->last_tre = last_tre; tknext->last_cword = last_cword;
    tknext->last_lscore = last_lscore; tknext->score = next_score;
    b->token[next_node] = id; tknext->node = next_node;
  }
}

static int atom_wid(const Beam *b, int tre) { return tre < 0 ? -1 : b->atoms[tre].wid; }
static int atom_endtime(const Beam *b, int tre) { return tre < 0 ? -1 : b->atoms[tre].endtime; }

/* ---- heap select (beam.c:1342-1520) ------------------------------------------------ */
#define SD(A) tindex_local[(A)-1]
#define SVAL(A) (tlist_local[tindex_local[(A)-1]].score)
#define STVAL (tlist_local[s].score)

static void sort_token_upward(Beam *b, int neednum, int totalnum) {
  int n, root, child, parent, s;
  Tok *tlist_local = b->tlist[b->tn]; int *tindex_local = b->tindex[b->tn];
  for (root = totalnum / 2; root >= 1; root--) {
    s = SD(root); parent = root;
    while ((child = parent * 2) <= totalnum) {
      if (child < totalnum && SVAL(child) < SVAL(child + 1)) child++;
      if (STVAL >= SVAL(child)) break;
      SD(parent) = SD(child); parent = child;
    }
    SD(parent) = s;
  }
  n = totalnum;
  while (n > totalnum - neednum) {
    s = SD(n); SD(n) = SD(1); n--; parent = 1;
    while ((child = parent * 2) <= n) {
      if (child < n && SVAL(child) < SVAL(child + 1)) child++;
      if (STVAL >= SVAL(child)) break;
      SD(parent) = SD(child); parent = child;
    }
    SD(parent) = s;
  }
}

static void sort_token_downward(Beam *b, int neednum, int totalnum) {
  int n, root, child, parent, s;
  Tok *tlist_local = b->tlist[b->tn]; int *tindex_local = b->tindex[b->tn];
  for (root = totalnum / 2; root >= 1; root--) {
    s = SD(root); parent = root;
    while ((child = parent * 2) <= totalnum) {
      if (child < totalnum && SVAL(child) > SVAL(child + 1)) child++;
      if (STVAL <= SVAL(child)) break;
      SD(parent) = SD(child); parent = child;
    }
    SD(parent) = s;
  }
  n = totalnum;
  while (n > totalnum - neednum) {
    s = SD(n); SD(n) = SD(1); n--; parent = 1;
    while ((child = parent * 2) <= n) {
      if (child < n && SVAL(child) > SVAL(child + 1)) child++;
      if (STVAL <= SVAL(child)) break;
      SD(parent) = SD(child); parent = child;
    }
    SD(parent) = s;
  }
}

/* test tooling: oracle_set_heap_dump(path) makes every beam cut append (totalnum, neednum, scores in token-index
   order) to a file, so that tools/beamcut.cpp and the heap micro-benchmarks run on the selects of a real decode */
static FILE *heap_dump_fp = NULL;
void oracle_set_heap_dump(const char *path) {
  if (heap_dump_fp) { fclose(heap_dump_fp); heap_dump_fp = NULL; }
  if (path && path[0]) heap_dump_fp = fopen(path, "wb");
}

/* test tooling: oracle_set_node_dump(path) appends (totalnum, node ids of the frame's tokens in creation order) at
   every beam cut -- the per-frame node working set, for tools/node_locality.py */
static FILE *node_dump_fp = NULL;
void oracle_set_node_dump(const char *path) {
  if (node_dump_fp) { fclose(node_dump_fp); node_dump_fp = NULL; }
  if (path && path[0]) node_dump_fp = fopen(path, "wb");
}

static void sort_token_no_order(Beam *b, int neednum, int *start, int *end) {
  int totalnum = b->tnum[b->tn], restnum = totalnum - neednum;
  if (node_dump_fp) {
    int i;
    fwrite(&totalnum, sizeof(int), 1, node_dump_fp);
    for (i = 0; i < totalnum; i++) fwrite(&b->tlist[b->tn][i].node, sizeof(int), 1, node_dump_fp);
  }
  if (heap_dump_fp && neednum < totalnum) {
    int hdr[2] = { totalnum, neednum }, i;
    fwrite(hdr, sizeof(int), 2, heap_dump_fp);
    for (i = 0; i < totalnum; i++) fwrite(&b->tlist[b->tn][b->tindex[b->tn][i]].score, sizeof(float), 1, heap_dump_fp);
  }
  if (neednum >= totalnum) { *start = 0; *end = totalnum - 1; }
  else if (neednum < restnum) { sort_token_upward(b, neednum, totalnum); *start = totalnum - neednum; *end = totalnum - 1; }
  else { sort_token_downward(b, restnum, totalnum); *start = 0; *end = neednum - 1; }
}

/* ---- expansion ----------------------------------------------------------------------- */
static void beam_intra_word_core(Beam *b, const Tok *tk, int next_node, float next_a) {
  const jb200_tree_desc *t = b->t;
  int node = tk->node;
  float tmpsum, ngram_score_cache;
  tmpsum = tk->score + next_a;
  ngram_score_cache = JB200_LOG_ZERO;
  if (next_node != node) {
    if (t->scid[next_node] != 0) {
      ngram_score_cache = max_successor_prob(t, tk->last_cword, next_node) * t->lm_weight + t->lm_penalty;
      tmpsum -= tk->last_lscore;
      tmpsum += ngram_score_cache;
    }
  }
  if (ngram_score_cache == JB200_LOG_ZERO) ngram_score_cache = tk->last_lscore;
  propagate_token(b, next_node, tmpsum, tk->last_tre, tk->last_cword, ngram_score_cache);
}

static void beam_intra_word(Beam *b, int j) {
  const jb200_tree_desc *t = b->t;
  /* NOTE: take a copy; tlist[tl] is never reallocated inside a frame in a way that
     changes its content, the copy only protects against realloc moving it */
  Tok tk = b->tlist[b->tl][b->tindex[b->tl][j]];
  int node = tk.node, k;
  if (t->self_a[node] != JB200_LOG_ZERO) beam_intra_word_core(b, &tk, node, t->self_a[node]);
  if (t->next_a[node] != JB200_LOG_ZERO) beam_intra_word_core(b, &tk, node + 1, t->next_a[node]);
  for (k = t->arc_off[node]; k < t->arc_off[node + 1]; k++) beam_intra_word_core(b, &tk, t->arc_to[k], t->arc_a[k]);
}

static int save_trellis(Beam *b, const Tok *tk, int t) {
  oracle_atom *a;
  if (b->natoms == b->maxatoms) {
    b->maxatoms *= 2;
    b->atoms = (oracle_atom *)realloc(b->atoms, sizeof(oracle_atom) * b->maxatoms);
  }
  a = &b->atoms[b->natoms];
  a->wid = b->t->stend[tk->node];
  a->backscore = tk->score;
  a->begintime = atom_endtime(b, tk->last_tre) + 1;
  a->endtime = t - 1;
  a->last = tk->last_tre;
  a->lscore = tk->last_lscore;
  return b->natoms++;
}

/* multipath: the root node has no output, go one step further (beam.c:2467-2500, :2584-2605) */
static void propagate_from_root(Beam *b, int root, float tmpsum, int tre, int last_word, float lsc) {
  const jb200_tree_desc *t = b->t;
  int k;
  if (t->self_a[root] != JB200_LOG_ZERO) propagate_token(b, root, tmpsum + t->self_a[root], tre, last_word, lsc);
  if (t->next_a[root] != JB200_LOG_ZERO) propagate_token(b, root + 1, tmpsum + t->next_a[root], tre, last_word, lsc);
  for (k = t->arc_off[root]; k < t->arc_off[root + 1]; k++) propagate_token(b, t->arc_to[k], tmpsum + t->arc_a[k], tre, last_word, lsc);
}

/* grammar mode: every root, gated by the category pair of (ending word, root's word); the language score is the
 * insertion penalty (beam.c:2404-2411, :2444-2450; CLASS_NGRAM adds cprob[last_word]) */
static void beam_inter_word_dfa(Beam *b, const Tok *tk, int tre) {
  const jb200_tree_desc *t = b->t;
  int node = tk->node, sword = t->stend[node], i, last_word;
  float tmpsum, ngram_score_cache;
  last_word = t->is_transparent[sword] ? tk->last_cword : sword;
  for (i = 0; i < t->n_iso; i++) {
    int next_node = t->iso_node[i];
    if (!t->cp_allowed[(size_t)sword * t->n_iso + t->iso_id[i]]) continue;
    tmpsum = tk->score;
    if (!t->multipath) tmpsum += t->wordend_a[sword];
    ngram_score_cache = t->penalty1;
    ngram_score_cache += t->cprob[last_word];
    tmpsum += ngram_score_cache;
    if (t->multipath) propagate_from_root(b, next_node, tmpsum, tre, last_word, ngram_score_cache);
    else propagate_token(b, next_node, tmpsum, tre, last_word, ngram_score_cache);
  }
}

static void beam_inter_word(Beam *b, const Tok *tk, int tre) {
  const jb200_tree_desc *t = b->t;
  int node = tk->node, sword = t->stend[node], i, last_word;
  float tmpprob, tmpsum, ngram_score_cache;
  const float *iwparray;
  int transp_s;
  if (t->lm_type == JB200_LM_DFA) { beam_inter_word_dfa(b, tk, tre); return; }
  transp_s = t->is_transparent[sword];
  last_word = transp_s ? tk->last_cword : sword;
  if (sword == t->tail_silwid) return;
  tmpprob = tk->score;
  if (!t->multipath) tmpprob += t->wordend_a[sword];
  if (b->wordend_best_score < tmpprob) {
    b->wordend_best_score = tmpprob; b->wordend_best_node = node;
    b->wordend_best_tre = tre; b->wordend_best_last_cword = tk->last_cword;
  }
  iwparray = max_successor_prob_iw(b, transp_s ? tk->last_cword : sword);
  for (i = 0; i < t->n_iso; i++) {
    int next_node = t->iso_node[i];
    if (t->multipath && t->wordbegin[t->head_silwid] == next_node) continue;   /* beam.c:2337-2342 */
    tmpprob = iwparray[t->iso_id[i]];
    tmpsum = tk->score;
    if (!t->multipath) tmpsum += t->wordend_a[sword];
    ngram_score_cache = tmpprob * t->lm_weight + t->lm_penalty;
    tmpsum += ngram_score_cache;
    if (transp_s && tk->last_cword >= 0 && t->is_transparent[tk->last_cword]) tmpsum += t->lm_penalty_trans;
    if (t->multipath) propagate_from_root(b, next_node, tmpsum, tre, last_word, ngram_score_cache);
    else propagate_token(b, next_node, tmpsum, tre, last_word, ngram_score_cache);
  }
}

static void beam_inter_word_factoring(Beam *b) {
  const jb200_tree_desc *t = b->t;
  int node = b->wordend_best_node, sword = t->stend[node], i, last_word;
  float tmpprob, tmpsum, ngram_score_cache;
  int transp_s = t->is_transparent[sword];
  last_word = transp_s ? b->wordend_best_last_cword : sword;
  for (i = 0; i < t->n_shared; i++) {
    int next_node = t->shared_node[i];
    tmpprob = t->fscore[-t->scid[next_node]];
    ngram_score_cache = tmpprob * t->lm_weight + t->lm_penalty;
    tmpsum = b->wordend_best_score;
    tmpsum += ngram_score_cache;
    if (transp_s && b->wordend_best_last_cword >= 0 && t->is_transparent[b->wordend_best_last_cword]) tmpsum += t->lm_penalty_trans;
    if (tmpsum < b->score_pruning_threshold) continue;
    if (t->multipath) propagate_from_root(b, next_node, tmpsum, b->wordend_best_tre, last_word, ngram_score_cache);
    else propagate_token(b, next_node, tmpsum, b->wordend_best_tre, last_word, ngram_score_cache);
  }
}

/* ---- frames -------------------------------------------------------------------------- */
static void init_frame0(Beam *b) {
  const jb200_tree_desc *t = b->t;
  int node, newid; Tok *nw;
  b->tn = 0; b->tl = 1;
  b->tnum[0] = b->tnum[1] = 0;
  if (t->lm_type == JB200_LM_DFA) {
    /* init_nodescore, grammar branch (beam.c:1669-1760): one token per sentence-initial word (duplicates of a
     * shared first node were dropped when the list was made), in the reference's creation order */
    int i;
    for (i = 0; i < t->n_init; i++) {
      node = t->init_node[i];
      newid = create_token(b);
      nw = &b->tlist[b->tn][newid];
      nw->last_tre = -1; nw->last_cword = -1;       /* the bos atom: wid = WORD_INVALID */
      nw->last_lscore = t->init_lscore[i];
      if (t->multipath) nw->score = nw->last_lscore;
      else nw->score = outprob_style(b, node, -1, 0) + nw->last_lscore;
      b->token[node] = newid; nw->node = node;
    }
    sort_token_no_order(b, t->beam_width, &b->n_start, &b->n_end);
    b->score_pruning_threshold = JB200_LOG_ZERO;
    return;
  }
  newid = create_token(b);
  nw = &b->tlist[b->tn][newid];
  node = t->wordbegin[t->head_silwid];      /* offset[beginword][0] */
  if (t->scid[node] != 0) nw->last_lscore = max_successor_prob(t, -1, node);
  else nw->last_lscore = 0.0;
  nw->last_lscore = nw->last_lscore * t->lm_weight + t->lm_penalty;
  nw->last_tre = -1; nw->last_cword = -1;
  if (t->multipath) nw->score = nw->last_lscore;      /* beam.c:1654-1656: the word-begin node has no output */
  else nw->score = outprob_style(b, node, -1, 0) + nw->last_lscore;
  b->token[node] = newid; nw->node = node;
  sort_token_no_order(b, t->beam_width, &b->n_start, &b->n_end);
  b->score_pruning_threshold = JB200_LOG_ZERO;
}

static int proceed(Beam *b, int t) {
  const jb200_tree_desc *tr = b->t;
  int j, tl, tn;
  b->tl = b->tn; b->tn = (b->tn == 0) ? 1 : 0;
  tl = b->tl; tn = b->tn;
  b->wordend_best_score = JB200_LOG_ZERO;
  for (j = 0; j < b->tnum[tl]; j++) b->token[b->tlist[tl][j].node] = -1;     /* clear_tokens */

  for (j = b->n_start; j <= b->n_end; j++) {
    Tok tk = b->tlist[tl][b->tindex[tl][j]];
    if (tk.score <= JB200_LOG_ZERO) continue;
    if (tk.score < b->score_pruning_threshold) continue;
    beam_intra_word(b, j);
    if (tr->stend[tk.node] >= 0) {
      int tre = save_trellis(b, &tk, t);
      beam_inter_word(b, &tk, tre);
    }
  }
  if (b->wordend_best_score > JB200_LOG_ZERO) beam_inter_word_factoring(b);

  b->score_pruning_max = JB200_LOG_ZERO;
  for (j = 0; j < b->tnum[tn]; j++) {
    Tok *tk = &b->tlist[tn][b->tindex[tn][j]];
    tk->score += outprob_style(b, tk->node, atom_wid(b, tk->last_tre), t);
    if (b->score_pruning_max < tk->score) b->score_pruning_max = tk->score;
  }
  if (tr->score_pruning_width >= 0.0) b->score_pruning_threshold = b->score_pruning_max - tr->score_pruning_width;
  else b->score_pruning_threshold = JB200_LOG_ZERO;

  b->tnum[tl] = 0;                                                           /* clear_tlist */
  sort_token_no_order(b, tr->beam_width, &b->n_start, &b->n_end);
  return b->tnum[tn] != 0;
}

/* MULTIPATH MODE, beam.c:2752-2828 + :2935-2941 */
static int proceed_multipath(Beam *b, int t, int final) {
  const jb200_tree_desc *tr = b->t;
  int j, tl, tn;
  b->tl = b->tn; b->tn = (b->tn == 0) ? 1 : 0;
  tl = b->tl; tn = b->tn;
  b->wordend_best_score = JB200_LOG_ZERO;
  for (j = 0; j < b->tnum[tl]; j++) b->token[b->tlist[tl][j].node] = -1;
  for (j = b->n_start; j <= b->n_end; j++) {
    Tok tk = b->tlist[tl][b->tindex[tl][j]];
    if (tk.score <= JB200_LOG_ZERO) continue;
    if (tk.score < b->score_pruning_threshold) continue;
    beam_intra_word(b, j);
  }
  sort_token_no_order(b, tr->beam_width, &b->n_start, &b->n_end);
  for (j = b->n_start; j <= b->n_end; j++) {
    Tok tk = b->tlist[tn][b->tindex[tn][j]];
    if (tk.score < b->score_pruning_threshold) continue;
    if (tr->stend[tk.node] >= 0) {
      int tre = save_trellis(b, &tk, t);
      if (final) continue;
      beam_inter_word(b, &tk, tre);
    }
  }
  if (b->wordend_best_score > JB200_LOG_ZERO) beam_inter_word_factoring(b);
  b->score_pruning_max = JB200_LOG_ZERO;
  if (!final) {
    for (j = 0; j < b->tnum[tn]; j++) {
      Tok *tk = &b->tlist[tn][b->tindex[tn][j]];
      if (tr->outstyle[tk->node] == 255) continue;
      tk->score += outprob_style(b, tk->node, atom_wid(b, tk->last_tre), t);
      if (b->score_pruning_max < tk->score) b->score_pruning_max = tk->score;
    }
  }
  if (tr->score_pruning_width >= 0.0) b->score_pruning_threshold = b->score_pruning_max - tr->score_pruning_width;
  else b->score_pruning_threshold = JB200_LOG_ZERO;
  b->tnum[tl] = 0;
  sort_token_no_order(b, tr->beam_width, &b->n_start, &b->n_end);
  return b->tnum[tn] != 0;
}

static int cmp_atom_idx(const void *pa, const void *pb, void *ctx) {
  const oracle_atom *a = (const oracle_atom *)ctx;
  int x = *(const int *)pa, y = *(const int *)pb;
  if (a[x].endtime != a[y].endtime) return a[x].endtime - a[y].endtime;
  return a[x].wid - a[y].wid;
}

int oracle_beam_decode(const jb200_tree_desc *t, const jb200_gmm_desc *g,
                       const float *st, int T, int S,
                       oracle_atom *atoms_out, int max_atoms,
                       int *best_words, int *n_best, float *best_score, int *status,
                       int *trace_counts) {
  Beam b; int f, i, j, k, framelen, C = g ? g->n_cdsets : 0;
  int *order, *newidx, nkeep;
  memset(&b, 0, sizeof(b));
  b.t = t; b.g = g; b.st = st; b.T = T; b.S = S;
  b.maxtnum = t->beam_width * 2 + t->n_start + 16;
  for (k = 0; k < 2; k++) {
    b.tlist[k] = (Tok *)malloc(sizeof(Tok) * b.maxtnum);
    b.tindex[k] = (int *)malloc(sizeof(int) * b.maxtnum);
  }
  b.token = (int *)malloc(sizeof(int) * t->n_nodes);
  for (i = 0; i < t->n_nodes; i++) b.token[i] = -1;
  b.maxatoms = 4096; b.atoms = (oracle_atom *)malloc(sizeof(oracle_atom) * b.maxatoms);
  b.cdval = (float *)malloc(sizeof(float) * (C + 1));
  b.cdstamp = (int *)malloc(sizeof(int) * (C + 1));
  for (i = 0; i <= C; i++) b.cdstamp[i] = -1;
  b.nbest_work = (float *)malloc(sizeof(float) * ((g ? g->iwcd_nbest : 0) + 4));
  b.iwrow = (float *)malloc(sizeof(float) * (t->n_iso + 1));
  b.iwrow_word = -2;

  *status = 0; *n_best = 0; *best_score = 0.0f;
  framelen = T;
  if (T > 0) {
    init_frame0(&b);
    if (t->multipath) proceed_multipath(&b, 0, 0);            /* pass1.c:239-242 */
    if (trace_counts) { trace_counts[0] = b.tnum[b.tn]; trace_counts[1] = b.n_end - b.n_start + 1; }
    for (f = 1; f < T; f++) {
      int alive = t->multipath ? proceed_multipath(&b, f, 0) : proceed(&b, f);
      if (trace_counts) { trace_counts[2 * f] = b.tnum[b.tn]; trace_counts[2 * f + 1] = b.n_end - b.n_start + 1; }
      if (!alive) { framelen = f; break; }   /* pass1.c:242-245: search terminated */
    }
    if (t->multipath) {
      /* get_back_trellis_end, multipath version (beam.c:3066-3072): only arcs to word ends */
      proceed_multipath(&b, T, 1);
    } else {
      /* get_back_trellis_end (normal version), beam.c:3076-3086 */
      b.tl = b.tn; b.tn = (b.tn == 0) ? 1 : 0;
      for (j = b.n_start; j <= b.n_end; j++) {
        Tok *tk = &b.tlist[b.tl][b.tindex[b.tl][j]];
        if (t->stend[tk->node] >= 0) save_trellis(&b, tk, T);
      }
    }
  }

  /* finalize_1st_pass: relocate by end frame, sort by word id (backtrellis.c:218-267,438-478) */
  order = (int *)malloc(sizeof(int) * (b.natoms + 1));
  newidx = (int *)malloc(sizeof(int) * (b.natoms + 1));
  nkeep = 0;
  for (i = 0; i < b.natoms; i++) { newidx[i] = -1; if (b.atoms[i].endtime < framelen) order[nkeep++] = i; }
  qsort_r(order, nkeep, sizeof(int), cmp_atom_idx, b.atoms);
  for (i = 0; i < nkeep; i++) newidx[order[i]] = i;
  if (nkeep > max_atoms) { nkeep = -3; goto done; }
  for (i = 0; i < nkeep; i++) {
    atoms_out[i] = b.atoms[order[i]];
    atoms_out[i].last = (atoms_out[i].last < 0) ? -1 : newidx[atoms_out[i].last];
  }

  /* find_1pass_result (LM_PROB, no segmentation): best </s> atom on the last frame that has one */
  {
    int last_time, found = -1;
    for (last_time = framelen - 1; last_time >= 0 && found < 0; last_time--) {
      float maxscore = JB200_LOG_ZERO;
      for (i = 0; i < nkeep; i++) {
        if (atoms_out[i].endtime != last_time) continue;
        if (t->lm_type == JB200_LM_DFA) {
          /* grammar mode (beam.c:435-458): the best atom of the last frame that holds any */
          if (maxscore < atoms_out[i].backscore) { maxscore = atoms_out[i].backscore; found = i; }
          continue;
        }
        if (atoms_out[i].wid == t->tail_silwid && maxscore < atoms_out[i].backscore) { maxscore = atoms_out[i].backscore; found = i; break; }
      }
    }
    if (nkeep == 0 || found < 0) { *status = -1; }
    else {
      /* trace_backptr: the reference returns the sequence in normal order */
      int tmp[150], n = 0, a = found;
      tmp[n++] = atoms_out[a].wid;
      while (atoms_out[a].begintime > 0) {
        a = atoms_out[a].last;
        if (a < 0 || n >= 150) break;
        tmp[n++] = atoms_out[a].wid;
      }
      for (i = 0; i < n; i++) best_words[i] = tmp[n - i - 1];
      *n_best = n; *best_score = atoms_out[found].backscore;
    }
  }
done:
  for (k = 0; k < 2; k++) { free(b.tlist[k]); free(b.tindex[k]); }
  free(b.token); free(b.atoms); free(b.cdval); free(b.cdstamp); free(b.nbest_work); free(b.iwrow);
  free(order); free(newidx);
  return nkeep;
}
