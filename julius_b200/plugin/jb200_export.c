/* jb200_export.c -- Julius plugin (.jpi): flattens the live engine's models for the GPU path.
 *
 * Boundary (SURVEY.md 8b): a .jpi is a shared object found through -plugindir
 * (libjulius/src/plugin.c:139-227).  This one exports
 *     initialize / get_plugin_info          (plugin.c:184-210)
 *     startup(Recog*)                       (plugin.c:374-395, called last in j_final_fusion, m_fusion.c:1453)
 * At startup every model is loaded and the lexicon tree is built, so the hook
 * walks the reference's pointer graphs ONCE and writes them out as the plain
 * arrays of include/jb200_model.h:
 *     HTK_HMM_INFO (states, mixtures, inverted variances)      -> gmm.*
 *     CD_State_Set pseudo-phone sets                           -> am.cd_*
 *     DNNData                                                  -> dnn.*
 *     WCHMM_INFO (tree nodes, arcs, roots, factoring values)   -> tree.*
 *     RC_INFO / LRC_INFO context resolution (outprob_style.c:385-486),
 *       tabulated per left-context centre phone                -> tree.rset_ctx / word_ctx
 *     NGRAM_INFO 1-/2-gram tables (ngram_access.c:249-466)     -> tree.uni_* / tree.bi_*
 *     search parameters (beam width, LM weight/penalty)        -> tree.*
 * With JB200_EXPORT=<path> in the environment the blob is written to that
 * file ("JB2M" container); the in-process GPU attach lives in jb200_plugin.c.
 *
 * Every refusal is made by check_am / check_recog before anything is allocated or added to the blob.  After them a
 * build step can fail only by running out of memory; each step frees what it allocated on every exit.
 *
 * This file reads reference structures only through their public headers; it
 * contains no reference code.
 */
#include <julius/juliuslib.h>
#include "jb200_model.h"

#define PLUGIN_TITLE "jb200 model flattener (GPU acoustic scoring + pass-1 beam)"

static int oom(void) { jlog("ERROR: jb200: out of memory\n"); return -1; }

/* ---------------------------------------------------------------- tiny pointer map */
typedef struct { const void **k; int *v; int cap, n; } PMap;
static void pm_free(PMap *m) { free(m->k); free(m->v); m->k = NULL; m->v = NULL; }
static int pm_init(PMap *m, int cap) {
  int c = 64; while (c < cap * 2) c <<= 1;
  m->cap = c; m->n = 0;
  m->k = (const void **)calloc((size_t)c, sizeof(void *));
  m->v = (int *)calloc((size_t)c, sizeof(int));
  if (m->k != NULL && m->v != NULL) return 0;
  pm_free(m);
  return -1;
}
static int pm_slot(const PMap *m, const void *p) {
  size_t h = ((size_t)p >> 3) * 0x9E3779B97F4A7C15ull;
  int i = (int)(h >> 20) & (m->cap - 1);
  while (m->k[i] != NULL && m->k[i] != p) i = (i + 1) & (m->cap - 1);
  return i;
}
static int pm_grow(PMap *m) {
  PMap n; int i;
  if (pm_init(&n, m->cap) != 0) return -1;
  for (i = 0; i < m->cap; i++) if (m->k[i]) { int s = pm_slot(&n, m->k[i]); n.k[s] = m->k[i]; n.v[s] = m->v[i]; n.n++; }
  pm_free(m); *m = n;
  return 0;
}
/* returns existing id or assigns next id (= current count); -1 when out of memory */
static int pm_intern(PMap *m, const void *p, int *is_new) {
  int s;
  if (m->n * 2 >= m->cap && pm_grow(m) != 0) return -1;
  s = pm_slot(m, p);
  if (m->k[s] == p) { *is_new = 0; return m->v[s]; }
  m->k[s] = p; m->v[s] = m->n; *is_new = 1;
  return m->n++;
}

/* growable int vector; -1, and the vector unchanged, when out of memory */
typedef struct { int *d; int n, cap; } IVec;
static int iv_push(IVec *v, int x) {
  if (v->n == v->cap) {
    int cap = v->cap ? v->cap * 2 : 1024, *d = (int *)realloc(v->d, sizeof(int) * cap);
    if (d == NULL) return -1;
    v->d = d; v->cap = cap;
  }
  v->d[v->n++] = x;
  return 0;
}

/* ---------------------------------------------------------------- cd-set registry */
/* failed: an allocation failed; nothing is registered after that, and jb200_flatten reports it once at the end */
typedef struct { PMap map; IVec off; IVec states; int failed; } CdReg;

static int cd_intern(CdReg *r, CD_State_Set *cs) {
  int is_new, id, i;
  if (r->failed || (id = pm_intern(&r->map, cs, &is_new)) < 0) { r->failed = 1; return 0; }
  if (is_new) {
    for (i = 0; i < cs->num; i++) r->failed |= iv_push(&r->states, cs->s[i]->id) != 0;
    r->failed |= iv_push(&r->off, r->states.n) != 0;
  }
  return id;
}

/* ---------------------------------------------------------------- refusals */
static int check_am(PROCESS_AM *am) {
  HTK_HMM_INFO *hi;
  HTK_HMM_State *st;
  if (am == NULL) { jlog("ERROR: jb200: no acoustic model\n"); return -1; }
  if (am->dnn != NULL) {
    if (am->dnn->hnum + 1 > JB200_DNN_MAX_LAYERS) { jlog("ERROR: jb200: too many DNN layers\n"); return -1; }
    return 0;
  }
  hi = am->hmminfo;
  if (hi->opt.stream_info.num != 1) { jlog("ERROR: jb200: multi-stream AM is not supported\n"); return -1; }
  /* Tied-mixture (codebook) states are flattened into ordinary states: the mixture list of a <TMIX> state is its
   * codebook's densities with the state's own weights.  That IS what calc_tied_mix computes for -gprune none and
   * safe (calc_tied_mix.c:161-248: codebook scores once per frame, + weight[id], addlog_array in list order;
   * gprune_none lists ids in order, gprune_safe the N best sorted by score -- exactly what calc_mix does for a
   * private mixture).  The true beam/heuristic pruning of codebooks seeds itself with the previous frame's best
   * ids (calc_tied_mix.c:193-200), i.e. depends on which frames the search happened to evaluate: refused. */
  if (hi->is_tied_mixture &&
      (am->config->gprune_method == GPRUNE_SEL_BEAM || am->config->gprune_method == GPRUNE_SEL_HEURISTIC)) {
    jlog("ERROR: jb200: tied-mixture AM with history-dependent Gaussian pruning; use -gprune none or -gprune safe\n");
    return -1;
  }
  if (!hi->variance_inversed) { jlog("ERROR: jb200: variances are expected to be inverted at this point\n"); return -1; }
  for (st = hi->ststart; st; st = st->next)
    if (st->id < 0 || st->id >= hi->totalstatenum) { jlog("ERROR: jb200: state id out of range\n"); return -1; }
  return 0;
}

/* -userlm (wchmm.h:274-276): pass 1 reads the LM through two host function pointers.  They cannot be called from the
 * device, so the 2-gram side is tabulated once -- a dense table over the dictionary, flatten_userlm -- which bounds the
 * vocabulary this mode supports */
static int check_userlm(WCHMM_INFO *w) {
  WORD_INFO *wi = w->winfo;
  const char *e = getenv("JB200_USERLM_MAXWORDS");
  const int lim = (e != NULL && atoi(e) > 0) ? atoi(e) : 8192, V = wi->num;
  int i, dup = 0;
  if (w->bi_prob_user == NULL) { jlog("ERROR: jb200: -userlm without a registered 2-gram function\n"); return -1; }
  if (w->ngram != NULL) {
    /* the host caches these values per N-gram entry of the last word (factoring_sub.c:951-957,966: last_nword), so
     * with two dictionary words on one entry what it returns depends on which of them asked first */
    unsigned char *seen = (unsigned char *)calloc((size_t)w->ngram->max_word_num + 1, 1);
    if (seen == NULL) return oom();
    for (i = 0; i < V && !dup; i++) { dup = seen[wi->wton[i]]; seen[wi->wton[i]] = 1; }
    free(seen);
    if (dup) { jlog("ERROR: jb200: -userlm with several dictionary words on one N-gram entry is not supported\n"); return -1; }
  }
  if (V > lim) { jlog("ERROR: jb200: -userlm is tabulated densely and supports up to %d words (JB200_USERLM_MAXWORDS), the dictionary has %d\n", lim, V); return -1; }
  return 0;
}

static int check_recog(RecogProcess *r) {
  WCHMM_INFO *w = r->wchmm;
  int i, stid, niso = 0;
  if (w->lmtype == LM_DFA) {
    /* grammar mode: category tree + category-pair constraint only (beam.c:2404-2455) */
    if (w->lmvar != LM_DFA_GRAMMAR || !w->category_tree || w->dfa == NULL) {
      jlog("ERROR: jb200: grammar mode needs a category tree over a DFA grammar (isolated-word mode is not supported)\n");
      return -1;
    }
    if (w->dfa_forward != NULL) { jlog("ERROR: jb200: forward-DFA state tracking (.dfa.forward) is not supported\n"); return -1; }
  } else {
    if (w->lmtype != LM_PROB || (w->ngram == NULL && w->lmvar != LM_NGRAM_USER)) { jlog("ERROR: jb200: lexicon tree without a language model\n"); return -1; }
    if (w->category_tree) { jlog("ERROR: jb200: category tree with an N-gram is not supported\n"); return -1; }
    if (w->lmvar == LM_NGRAM_USER && check_userlm(w) != 0) return -1;
  }
  for (i = 0; i < w->n; i++) {
    const int s = w->outstyle[i];
    if (w->state[i].out.state != NULL && s != AS_STATE && s != AS_LSET && s != AS_RSET && s != AS_LRSET) {
      jlog("ERROR: jb200: unknown outstyle\n");
      return -1;
    }
  }
  if (w->lmtype == LM_DFA) return 0;
  /* in the order flatten_roots visits them */
  for (stid = w->startnum - 1; stid >= 0; stid--) {
    if (w->start2isolate[stid] == -1) continue;
    if (w->state[w->startnode[stid]].scid <= 0) { jlog("ERROR: jb200: isolated root without successor word\n"); return -1; }
    niso++;
  }
  if (niso != w->isolatenum) { jlog("ERROR: jb200: isolatenum mismatch\n"); return -1; }
  if (w->lmvar != LM_NGRAM_USER && w->ngram->d[1].is24bit) { jlog("ERROR: jb200: 24-bit 2-gram index is not supported\n"); return -1; }
  return 0;
}

/* ---------------------------------------------------------------- AM: GMM */
static int gmm_densities(HTK_HMM_INFO *hi, HTK_HMM_State **byid, const int *off, jb200_blob *b) {
  const int S = hi->totalstatenum, D = hi->opt.vec_size, G = off[S];
  float *mean = (float *)calloc((size_t)G * D, sizeof(float)), *ivar = (float *)calloc((size_t)G * D, sizeof(float));
  float *gconst = (float *)calloc((size_t)G, sizeof(float)), *lnw = (float *)calloc((size_t)G, sizeof(float));
  unsigned char *valid = (unsigned char *)calloc((size_t)G, 1);
  int i, d, m, rc = 0;
  if (!mean || !ivar || !gconst || !lnw || !valid) rc = oom();
  for (i = 0; i < S && rc == 0; i++) {
    HTK_HMM_PDF *p;
    if (!byid[i]) continue;
    p = byid[i]->pdf[0];
    for (m = 0; m < p->mix_num; m++) {
      HTK_HMM_Dens *dn = p->tmix ? ((GCODEBOOK *)p->b)->d[m] : p->b[m];
      int g = off[i] + m;
      lnw[g] = p->bweight[m];
      if (dn == NULL) { valid[g] = 0; continue; }
      valid[g] = 1;
      gconst[g] = dn->gconst;
      for (d = 0; d < D; d++) { mean[(size_t)g * D + d] = dn->mean[d]; ivar[(size_t)g * D + d] = dn->var->vec[d]; }
    }
  }
  if (rc == 0) {
    jb200_blob_add(b, "gmm.mean", JB200_F32, (int64_t)G * D, mean);
    jb200_blob_add(b, "gmm.ivar", JB200_F32, (int64_t)G * D, ivar);
    jb200_blob_add(b, "gmm.gconst", JB200_F32, G, gconst);
    jb200_blob_add(b, "gmm.lnweight", JB200_F32, G, lnw);
    jb200_blob_add(b, "gmm.valid", JB200_U8, G, valid);
  }
  free(mean); free(ivar); free(gconst); free(lnw); free(valid);
  return rc;
}

static int flatten_gmm(PROCESS_AM *am, jb200_blob *b) {
  HTK_HMM_INFO *hi = am->hmminfo;
  const int S = hi->totalstatenum;
  HTK_HMM_State *st, **byid = (HTK_HMM_State **)calloc((size_t)S, sizeof(void *));
  int *off = (int *)malloc(sizeof(int) * (S + 1)), i, rc, meth;
  if (byid == NULL || off == NULL) rc = oom();
  else {
    for (st = hi->ststart; st; st = st->next) byid[st->id] = st;
    off[0] = 0;
    for (i = 0; i < S; i++) off[i + 1] = off[i] + (byid[i] ? byid[i]->pdf[0]->mix_num : 0);
    switch (am->config->gprune_method) {
      case GPRUNE_SEL_SAFE: meth = JB200_GPRUNE_SAFE; break;
      case GPRUNE_SEL_HEURISTIC: meth = JB200_GPRUNE_HEU; break;
      case GPRUNE_SEL_BEAM: meth = JB200_GPRUNE_BEAM; break;
      default: meth = JB200_GPRUNE_NONE; break;
    }
    jb200_blob_add_i(b, "gmm.n_states", S);
    jb200_blob_add_i(b, "gmm.dim", hi->opt.vec_size);
    jb200_blob_add_i(b, "gmm.n_gauss", off[S]);
    jb200_blob_add_i(b, "gmm.max_mix", hi->maxmixturenum);
    jb200_blob_add_i(b, "gmm.gprune_method", meth);
    jb200_blob_add_i(b, "gmm.gprune_num", am->hmmwrk.OP_gprune_num);
    jb200_blob_add(b, "gmm.state_off", JB200_I32, S + 1, off);
    rc = gmm_densities(hi, byid, off, b);
  }
  free(byid); free(off);
  return rc;
}

/* ---------------------------------------------------------------- AM: DNN */
static void flatten_dnn(PROCESS_AM *am, jb200_blob *b) {
  DNNData *dnn = am->dnn;
  int i, L = dnn->hnum + 1;
  char nm[48];
  jb200_blob_add_i(b, "dnn.n_layers", L);
  jb200_blob_add_i(b, "dnn.in_dim", dnn->inputnodenum);
  jb200_blob_add_i(b, "dnn.out_dim", dnn->outputnodenum);
  for (i = 0; i < L; i++) {
    DNNLayer *l = (i < dnn->hnum) ? &dnn->h[i] : &dnn->o;
    snprintf(nm, sizeof(nm), "dnn.l%d.in", i);  jb200_blob_add_i(b, nm, l->in);
    snprintf(nm, sizeof(nm), "dnn.l%d.out", i); jb200_blob_add_i(b, nm, l->out);
    snprintf(nm, sizeof(nm), "dnn.l%d.w", i);   jb200_blob_add(b, nm, JB200_F32, (int64_t)l->in * l->out, l->w);
    snprintf(nm, sizeof(nm), "dnn.l%d.b", i);   jb200_blob_add(b, nm, JB200_F32, l->out, l->b);
  }
  jb200_blob_add(b, "dnn.state_prior", JB200_F32, dnn->state_prior_num, dnn->state_prior);
  /* the state id space is still the HMM's */
  jb200_blob_add_i(b, "gmm.n_states", am->hmminfo->totalstatenum);
}

/* ---------------------------------------------------------------- tree: arcs, node outputs, roots, words */
static int word_begin(const WCHMM_INFO *w, int wd) { return w->hmminfo->multipath ? w->wordbegin[wd] : w->offset[wd][0]; }

/* class N-gram: the in-class log probability of word wd */
static LOGPROB word_cprob(const WORD_INFO *wi, int wd) {
#ifdef CLASS_NGRAM
  return wi->cprob[wd];
#else
  (void)wi; (void)wd;
  return 0.0f;
#endif
}

/* A_CELL2 lists, kept in the order beam_intra_word walks them (beam.c:2172-2176) */
static int flatten_arcs(WCHMM_INFO *w, jb200_blob *b) {
  const int n = w->n;
  int *off = (int *)malloc(sizeof(int) * (n + 1)), *to, i, j, k, narc = 0, rc = 0;
  float *a;
  A_CELL2 *ac;
  if (off == NULL) return oom();
  for (i = 0; i < n; i++) {
    off[i] = narc;
    for (ac = w->ac[i]; ac; ac = ac->next) narc += ac->n;
  }
  off[n] = narc;
  to = (int *)malloc(sizeof(int) * (narc + 1));
  a = (float *)malloc(sizeof(float) * (narc + 1));
  if (to == NULL || a == NULL) rc = oom();
  else {
    for (i = 0, k = 0; i < n; i++)
      for (ac = w->ac[i]; ac; ac = ac->next) for (j = 0; j < ac->n; j++) { to[k] = ac->arc[j]; a[k] = ac->a[j]; k++; }
    jb200_blob_add_i(b, "tree.n_arcs", narc);
    jb200_blob_add(b, "tree.arc_off", JB200_I32, n + 1, off);
    jb200_blob_add(b, "tree.arc_to", JB200_I32, narc, to);
    jb200_blob_add(b, "tree.arc_a", JB200_F32, narc, a);
  }
  free(off); free(to); free(a);
  return rc;
}

/* context class of an RSET / LRSET node */
typedef struct { HMM_Logical *hmm; int loc, style, cat; } RKey;

/* outstyle and out_ref of node i; an RSET / LRSET node refers to its context class, added to keys on first use */
static void node_output(WCHMM_INFO *w, CdReg *cd, int i, RKey *keys, int *nr, unsigned char *style, int *ref) {
  RKey k = {NULL, 0, 0, -1};
  int j;
  if (w->state[i].out.state == NULL) { *style = 255; *ref = -1; return; }
  switch (w->outstyle[i]) {
    case AS_STATE: *style = JB200_AS_STATE; *ref = w->state[i].out.state->id; return;
    case AS_LSET:  *style = JB200_AS_LSET;  *ref = cd_intern(cd, w->state[i].out.lset); return;
    case AS_RSET:  k.hmm = w->state[i].out.rset->hmm; k.loc = w->state[i].out.rset->state_loc; k.style = JB200_AS_RSET; break;
    default:       /* AS_LRSET: check_recog refused any other style */
      k.hmm = w->state[i].out.lrset->hmm; k.loc = w->state[i].out.lrset->state_loc; k.style = JB200_AS_LRSET;
      if (w->category_tree) k.cat = (int)w->state[i].out.lrset->category;     /* category-indexed cd sets, outprob_style.c:448-459 */
  }
  for (j = 0; j < *nr; j++) if (keys[j].hmm == k.hmm && keys[j].loc == k.loc && keys[j].style == k.style && keys[j].cat == k.cat) break;
  if (j == *nr) keys[(*nr)++] = k;
  *style = (unsigned char)k.style; *ref = j;
}

/* outprob_style()'s resolution of class k after a word whose last phone has centre phone lc (NULL: no such word):
 * a state id, or -(cd-set id)-1 */
static int rset_ref(WCHMM_INFO *w, CdReg *cd, const RKey *k, char *lc) {
  HTK_HMM_INFO *hi = w->hmminfo;
  HMM_Logical *h = k->hmm, *o;
  CD_Set *lcd = NULL;
  char buf[MAX_HMMNAME_LEN];
  if (k->style == JB200_AS_RSET) {
    /* outprob_style.c:385-436 */
    if (lc != NULL && (o = get_left_context_HMM(h, lc, hi)) != NULL) h = o;
  } else if (w->category_tree) {
    /* outprob_style.c:437-486, category-indexed cd sets (outprob_style.c:448-459) */
    o = lc != NULL ? get_left_context_HMM(h, lc, hi) : NULL;
    lcd = lcdset_lookup_with_category(w, o != NULL ? o : h, (WORD_ID)k->cat);
  } else {
    /* outprob_style.c:437-486 */
    strcpy(buf, h->name);
    if (lc != NULL) add_left_context(buf, lc);
    lcd = lcdset_lookup_by_hmmname(hi, buf);
  }
  if (lcd != NULL) return -cd_intern(cd, &lcd->stateset[k->loc]) - 1;
  if (h->is_pseudo) return -cd_intern(cd, &h->body.pseudo->stateset[k->loc]) - 1;
  return h->body.defined->s[k->loc]->id;
}

static int ctx_lookup(char **names, int n, const char *s) {
  int i;
  for (i = 0; i < n; i++) if (strcmp(names[i], s) == 0) return i;
  return -1;
}

/* per-node arrays, the context classes and the rset_ctx / word_ctx tables; the context columns are the centre phones
 * of the words' last phones (cdhmm.c:129-160), plus one for "no word" */
static int flatten_outputs(WCHMM_INFO *w, CdReg *cd, jb200_blob *b) {
  WORD_INFO *wi = w->winfo;
  const int n = w->n, V = wi->num;
  char **names = (char **)calloc((size_t)V, sizeof(char *)), buf[MAX_HMMNAME_LEN];
  int *word_ctx = (int *)malloc(sizeof(int) * V), *stend = (int *)malloc(sizeof(int) * n);
  int *scid = (int *)malloc(sizeof(int) * n), *out_ref = (int *)malloc(sizeof(int) * n), *tab = NULL;
  unsigned char *outstyle = (unsigned char *)malloc((size_t)n);
  RKey *keys = (RKey *)malloc(sizeof(RKey) * n);
  int nctx = 0, nr = 0, i, c, rc = 0;
  if (!names || !word_ctx || !stend || !scid || !out_ref || !outstyle || !keys) rc = oom();
  for (i = 0; i < V && rc == 0; i++) {
    center_name(wi->wseq[i][wi->wlen[i] - 1]->name, buf);
    if ((word_ctx[i] = ctx_lookup(names, nctx, buf)) >= 0) continue;
    if ((names[nctx] = strdup(buf)) == NULL) rc = oom();
    word_ctx[i] = nctx++;
  }
  for (i = 0; i < n && rc == 0; i++) {
    stend[i] = (w->stend[i] == WORD_INVALID) ? -1 : (int)w->stend[i];
    scid[i] = (w->lmtype == LM_DFA) ? 0 : w->state[i].scid;      /* no factoring inside a category tree (beam.c:2028) */
    node_output(w, cd, i, keys, &nr, &outstyle[i], &out_ref[i]);
  }
  if (rc == 0 && (tab = (int *)malloc(sizeof(int) * (size_t)(nr ? nr : 1) * (nctx + 1))) == NULL) rc = oom();
  if (rc == 0) {
    for (i = 0; i < nr; i++)
      for (c = 0; c <= nctx; c++) tab[(size_t)i * (nctx + 1) + c] = rset_ref(w, cd, &keys[i], c < nctx ? names[c] : NULL);
    jb200_blob_add_i(b, "tree.n_rset", nr);
    jb200_blob_add_i(b, "tree.n_ctx", nctx);
    jb200_blob_add(b, "tree.rset_ctx", JB200_I32, (int64_t)nr * (nctx + 1), tab);
    jb200_blob_add(b, "tree.stend", JB200_I32, n, stend);
    jb200_blob_add(b, "tree.scid", JB200_I32, n, scid);
    jb200_blob_add(b, "tree.outstyle", JB200_U8, n, outstyle);
    jb200_blob_add(b, "tree.out_ref", JB200_I32, n, out_ref);
    jb200_blob_add(b, "tree.word_ctx", JB200_I32, V, word_ctx);
  }
  for (i = 0; i < nctx; i++) free(names[i]);
  free(names); free(word_ctx); free(stend); free(scid); free(out_ref); free(outstyle); free(keys); free(tab);
  return rc;
}

/* roots in visiting order stid = startnum-1 .. 0 (beam.c:2334, :2565) */
static int flatten_roots(WCHMM_INFO *w, jb200_blob *b) {
  const int ns = w->startnum;
  int *node = (int *)malloc(sizeof(int) * (ns + 1)), *word = (int *)malloc(sizeof(int) * (ns + 1));
  int *id = (int *)malloc(sizeof(int) * (ns + 1)), *shared = (int *)malloc(sizeof(int) * (ns + 1));
  int niso = 0, nsh = 0, stid, rc = 0;
  if (!node || !word || !id || !shared) rc = oom();
  for (stid = ns - 1; stid >= 0 && rc == 0; stid--) {
    const int nd = w->startnode[stid];
    if (w->lmtype == LM_DFA) {
      /* grammar mode: every root takes cross-word arrivals, gated by the category pair (beam.c:2404-2411) */
      node[niso] = nd; id[niso] = stid; word[niso++] = (int)w->start2wid[stid];
    } else if (w->start2isolate[stid] == -1) shared[nsh++] = nd;
    else { node[niso] = nd; id[niso] = w->start2isolate[stid]; word[niso++] = (int)w->scword[w->state[nd].scid]; }
  }
  if (rc == 0) {
    jb200_blob_add_i(b, "tree.n_iso", niso);
    jb200_blob_add_i(b, "tree.n_shared", nsh);
    jb200_blob_add(b, "tree.iso_node", JB200_I32, niso, node);
    jb200_blob_add(b, "tree.iso_word", JB200_I32, niso, word);
    jb200_blob_add(b, "tree.iso_id", JB200_I32, niso, id);
    jb200_blob_add(b, "tree.shared_node", JB200_I32, nsh, shared);
  }
  free(node); free(word); free(id); free(shared);
  return rc;
}

static int flatten_words(WCHMM_INFO *w, jb200_blob *b) {
  WORD_INFO *wi = w->winfo;
  const int V = wi->num, multipath = w->hmminfo->multipath, user = w->lmtype != LM_DFA && w->lmvar == LM_NGRAM_USER;
  float *wea = (float *)malloc(sizeof(float) * V), *cprob = (float *)malloc(sizeof(float) * V);
  int *wend = (int *)malloc(sizeof(int) * V), *wbeg = (int *)malloc(sizeof(int) * V), *wton = (int *)malloc(sizeof(int) * V);
  unsigned char *tr = (unsigned char *)malloc((size_t)V);
  int i, rc = 0;
  if (!wea || !cprob || !wend || !wbeg || !wton || !tr) rc = oom();
  else {
    for (i = 0; i < V; i++) {
      wea[i] = multipath ? 0.0f : w->wordend_a[i];
      wend[i] = w->wordend[i];
      wbeg[i] = word_begin(w, i);
      tr[i] = wi->is_transparent[i] ? 1 : 0;
      /* -userlm: the tabulated values of flatten_userlm are indexed by dictionary word and already final */
      wton[i] = user ? i : (int)wi->wton[i];
      cprob[i] = user ? 0.0f : word_cprob(wi, i);
    }
    jb200_blob_add(b, "tree.wordend_a", JB200_F32, V, wea);
    jb200_blob_add(b, "tree.wordend", JB200_I32, V, wend);
    jb200_blob_add(b, "tree.wordbegin", JB200_I32, V, wbeg);
    jb200_blob_add(b, "tree.wton", JB200_I32, V, wton);
    jb200_blob_add(b, "tree.is_transparent", JB200_U8, V, tr);
    jb200_blob_add(b, "tree.cprob", JB200_F32, V, cprob);
  }
  free(wea); free(cprob); free(wend); free(wbeg); free(wton); free(tr);
  return rc;
}

/* ---------------------------------------------------------------- tree: language model */
/* sentence-initial words and their nodes, in the order init_nodescore creates their tokens -> count */
static int init_words(RecogProcess *r, int *iw, int *in) {
  WCHMM_INFO *w = r->wchmm;
  DFA_INFO *dfa = w->dfa;
  MULTIGRAM *m;
  int t, x, y, ni = 0;
  for (m = r->lm->grammars; m; m = m->next) {
    if (!m->active) continue;
    for (t = m->cate_begin; t < m->cate_begin + m->dfa->term_num; t++) {
      if (!dfa_cp_begin(dfa, t)) continue;
      for (x = 0; x < dfa->term.wnum[t]; x++) {
        const int wd = (int)dfa->term.tw[t][x], node = word_begin(w, wd);
        for (y = 0; y < ni && in[y] != node; y++) ;
        if (y < ni) continue;     /* node_exist_token, beam.c:1719 */
        iw[ni] = wd; in[ni++] = node;
      }
    }
  }
  return ni;
}

/* grammar mode: category-pair table, sentence-initial words, penalty (beam.c:1669-1760, :2444-2450) */
static int flatten_grammar(RecogProcess *r, jb200_blob *b) {
  WCHMM_INFO *w = r->wchmm;
  WORD_INFO *wi = w->winfo;
  const int V = wi->num, ns = w->startnum;
  unsigned char *cp = (unsigned char *)malloc((size_t)V * (ns ? ns : 1));
  int *iw = (int *)malloc(sizeof(int) * V), *in = (int *)malloc(sizeof(int) * V), ni, i, k, rc = 0;
  float *il = (float *)malloc(sizeof(float) * V);
  if (!cp || !iw || !in || !il) rc = oom();
  else {
    for (i = 0; i < V; i++)
      for (k = 0; k < ns; k++) cp[(size_t)i * ns + k] = dfa_cp(w->dfa, (int)wi->wton[i], (int)wi->wton[w->start2wid[k]]) ? 1 : 0;
    ni = init_words(r, iw, in);
    for (i = 0; i < ni; i++) il[i] = r->config->lmp.penalty1 + word_cprob(wi, iw[i]);
    jb200_blob_add_i(b, "tree.lm_type", JB200_LM_DFA);
    jb200_blob_add_i(b, "tree.n_init", ni);
    jb200_blob_add_f(b, "tree.penalty1", r->config->lmp.penalty1);
    jb200_blob_add(b, "tree.init_word", JB200_I32, ni, iw);
    jb200_blob_add(b, "tree.init_node", JB200_I32, ni, in);
    jb200_blob_add(b, "tree.init_lscore", JB200_F32, ni, il);
    jb200_blob_add(b, "tree.cp_allowed", JB200_U8, (int64_t)V * ns, cp);
    /* the N-gram side of the descriptor stays empty */
    jb200_blob_add_i(b, "tree.n_fscore", 0); jb200_blob_add_i(b, "tree.n_scword", 0);
    jb200_blob_add(b, "tree.fscore", JB200_F32, 0, NULL); jb200_blob_add(b, "tree.scword", JB200_I32, 0, NULL);
    jb200_blob_add_i(b, "tree.lm_nvocab", 0); jb200_blob_add_i(b, "tree.lm_nbigram", 0);
    jb200_blob_add_i(b, "tree.lm_mode", 0); jb200_blob_add_i(b, "tree.lm_unk_id", -1);
    jb200_blob_add_f(b, "tree.lm_unk_num_log", 0.0f);
    jb200_blob_add(b, "tree.uni_prob", JB200_F32, 0, NULL); jb200_blob_add(b, "tree.uni_bow", JB200_F32, 0, NULL);
    jb200_blob_add(b, "tree.bi_bgn", JB200_I32, 0, NULL); jb200_blob_add(b, "tree.bi_num", JB200_I32, 0, NULL);
    jb200_blob_add(b, "tree.bi_wid", JB200_I32, 0, NULL); jb200_blob_add(b, "tree.bi_prob", JB200_F32, 0, NULL);
  }
  free(cp); free(iw); free(in); free(il);
  return rc;
}

/* factoring values: 1-gram (fscore) and successor-word (scword) tables */
static int flatten_factoring(WCHMM_INFO *w, jb200_blob *b) {
  int *scw = (int *)calloc((size_t)w->scnum + 1, sizeof(int)), i;
  if (scw == NULL) return oom();
  for (i = 1; i < w->scnum; i++) scw[i] = (int)w->scword[i];
  jb200_blob_add_i(b, "tree.n_fscore", w->fsnum);
  jb200_blob_add_i(b, "tree.n_scword", w->scnum);
  jb200_blob_add(b, "tree.fscore", JB200_F32, w->fsnum, w->fscore);
  jb200_blob_add(b, "tree.scword", JB200_I32, w->scnum, scw);
  free(scw);
  return 0;
}

/* the 1-/2-gram tables bi_prob_*() reads (ngram_access.c:249-466) */
static int flatten_ngram(NGRAM_INFO *ng, jb200_blob *b) {
  NGRAM_TUPLE_INFO *t1 = &ng->d[0], *t2 = &ng->d[1];
  const int Vn = ng->max_word_num;
  int *bgn = (int *)malloc(sizeof(int) * Vn), *num = (int *)malloc(sizeof(int) * Vn);
  int *bwid = (int *)malloc(sizeof(int) * (t2->totalnum + 1)), mode, i, rc = 0;
  const float *bow, *biprob;
  if (!bgn || !num || !bwid) rc = oom();
  else {
    if (ng->bigram_index_reversed) { mode = JB200_BI_ADDITIONAL_OLDBIN; bow = ng->bo_wt_1; biprob = ng->p_2; }
    else if (ng->dir == DIR_LR)    { mode = JB200_BI_NORMAL;            bow = t1->bo_wt;   biprob = t2->prob; }
    else if (ng->bo_wt_1 != NULL)  { mode = JB200_BI_ADDITIONAL;        bow = ng->bo_wt_1; biprob = ng->p_2; }
    else                           { mode = JB200_BI_COMPUTE;           bow = t1->bo_wt;   biprob = t2->prob; }
    for (i = 0; i < Vn; i++) {
      bgn[i] = (t2->bgn[i] == NNID_INVALID) ? -1 : (int)t2->bgn[i];
      num[i] = (int)t2->num[i];
    }
    for (i = 0; i < (int)t2->totalnum; i++) bwid[i] = (int)t2->nnid2wid[i];
    jb200_blob_add_i(b, "tree.lm_nvocab", Vn);
    jb200_blob_add_i(b, "tree.lm_nbigram", (int)t2->totalnum);
    jb200_blob_add_i(b, "tree.lm_mode", mode);
    jb200_blob_add_i(b, "tree.lm_unk_id", (ng->unk_id == WORD_INVALID) ? -1 : (int)ng->unk_id);
    jb200_blob_add_f(b, "tree.lm_unk_num_log", ng->unk_num_log);
    jb200_blob_add(b, "tree.uni_prob", JB200_F32, Vn, t1->prob);
    jb200_blob_add(b, "tree.uni_bow", JB200_F32, Vn, bow);
    jb200_blob_add(b, "tree.bi_bgn", JB200_I32, Vn, bgn);
    jb200_blob_add(b, "tree.bi_num", JB200_I32, Vn, num);
    jb200_blob_add(b, "tree.bi_wid", JB200_I32, (int64_t)t2->totalnum, bwid);
    jb200_blob_add(b, "tree.bi_prob", JB200_F32, (int64_t)t2->totalnum, biprob);
  }
  free(bgn); free(num); free(bwid);
  return rc;
}

/* User-defined LM.  What pass 1 asks of it (factoring_sub.c:963-981 for a node with one successor word, :1118-1128 for
 * the isolated roots) is  g(lw, w) = bi_prob_user(winfo, lw, w, ngram 2-gram(lw, w) + cprob[w])  with LOG_ZERO in place
 * of the N-gram term when no N-gram is loaded; the 1-gram factoring values (wchmm->fscore) went through uni_prob_user
 * when the host built the tree (wchmm.c:1497,1626).  g is tabulated as a DENSE 2-gram over the dictionary itself: every
 * row holds all V words, so the device's binary search always hits and returns the entry unchanged. */
static int flatten_userlm(WCHMM_INFO *w, jb200_blob *b) {
  WORD_INFO *wi = w->winfo;
  NGRAM_INFO *ng = w->ngram;
  const int V = wi->num;
  const int64_t VV = (int64_t)V * V;
  float *g = (float *)malloc(sizeof(float) * (size_t)VV), *zf = (float *)calloc((size_t)V, sizeof(float));
  int *bw = (int *)malloc(sizeof(int) * (size_t)VV), *bgn = (int *)malloc(sizeof(int) * V), *num = (int *)malloc(sizeof(int) * V);
  int a, c, rc = 0;
  if (!g || !zf || !bw || !bgn || !num) { jlog("ERROR: jb200: out of memory tabulating the user LM\n"); rc = -1; }
  for (a = 0; a < V && rc == 0; a++) {
    bgn[a] = a * V; num[a] = V;
    for (c = 0; c < V; c++) {
      LOGPROB p;
      if (ng != NULL) p = (*(ng->bigram_prob))(ng, wi->wton[a], wi->wton[c]) + word_cprob(wi, c);
      else p = LOG_ZERO;
      g[(size_t)a * V + c] = (*(w->bi_prob_user))(wi, (WORD_ID)a, (WORD_ID)c, p);
      bw[(size_t)a * V + c] = c;
    }
  }
  if (rc == 0) {
    jb200_blob_add_i(b, "tree.lm_nvocab", V);
    jb200_blob_add_i(b, "tree.lm_nbigram", (int)VV);
    jb200_blob_add_i(b, "tree.lm_mode", JB200_BI_NORMAL);
    jb200_blob_add_i(b, "tree.lm_unk_id", -1);
    jb200_blob_add_f(b, "tree.lm_unk_num_log", 0.0f);
    jb200_blob_add(b, "tree.uni_prob", JB200_F32, V, zf);
    jb200_blob_add(b, "tree.uni_bow", JB200_F32, V, zf);
    jb200_blob_add(b, "tree.bi_bgn", JB200_I32, V, bgn);
    jb200_blob_add(b, "tree.bi_num", JB200_I32, V, num);
    jb200_blob_add(b, "tree.bi_wid", JB200_I32, VV, bw);
    jb200_blob_add(b, "tree.bi_prob", JB200_F32, VV, g);
    jb200_blob_add_i(b, "tree.lm_user", 1);
  }
  free(g); free(zf); free(bw); free(bgn); free(num);
  return rc;
}

/* ---------------------------------------------------------------- tree */
static int flatten_tree(RecogProcess *r, CdReg *cd, jb200_blob *b) {
  WCHMM_INFO *w = r->wchmm;
  WORD_INFO *wi = w->winfo;
  const int is_dfa = (w->lmtype == LM_DFA);
  if (flatten_arcs(w, b) != 0 || flatten_outputs(w, cd, b) != 0 || flatten_roots(w, b) != 0 || flatten_words(w, b) != 0)
    return -1;
  if (is_dfa ? flatten_grammar(r, b) != 0
             : (flatten_factoring(w, b) != 0 || (w->lmvar == LM_NGRAM_USER ? flatten_userlm(w, b) : flatten_ngram(w->ngram, b)) != 0))
    return -1;
  jb200_blob_add_i(b, "tree.n_nodes", w->n);
  jb200_blob_add_i(b, "tree.n_words", wi->num);
  jb200_blob_add_i(b, "tree.n_start", w->startnum);
  jb200_blob_add_i(b, "tree.head_silwid", (is_dfa || wi->head_silwid == WORD_INVALID) ? -1 : (int)wi->head_silwid);
  jb200_blob_add_i(b, "tree.tail_silwid", (is_dfa || wi->tail_silwid == WORD_INVALID) ? -1 : (int)wi->tail_silwid);
  jb200_blob_add_i(b, "tree.multipath", w->hmminfo->multipath ? 1 : 0);
  jb200_blob_add_i(b, "tree.beam_width", r->trellis_beam_width);
  jb200_blob_add_f(b, "tree.lm_weight", r->config->lmp.lm_weight);
  jb200_blob_add_f(b, "tree.lm_penalty", r->config->lmp.lm_penalty);
  jb200_blob_add_f(b, "tree.lm_penalty_trans", r->pass1.lm_penalty_trans);   /* FSBeam copy, what beam.c:2441 reads */
  jb200_blob_add_f(b, "tree.score_pruning_width", r->config->pass1.score_pruning_width);
  jb200_blob_add(b, "tree.self_a", JB200_F32, w->n, w->self_a);
  jb200_blob_add(b, "tree.next_a", JB200_F32, w->n, w->next_a);
  return 0;
}

/* ---------------------------------------------------------------- entry: build the blob */
int jb200_flatten(PROCESS_AM *am, RecogProcess *r, jb200_blob *b) {
  const int tree = r != NULL && r->wchmm != NULL;
  CdReg cd;
  int rc, meth;

  if (check_am(am) != 0 || (tree && check_recog(r) != 0)) return -1;
  memset(&cd, 0, sizeof(cd));
  if (pm_init(&cd.map, 4096) != 0 || iv_push(&cd.off, 0) != 0) rc = oom();
  else if (am->dnn != NULL) { flatten_dnn(am, b); rc = 0; }
  else rc = flatten_gmm(am, b);
  if (rc == 0 && tree) rc = flatten_tree(r, &cd, b);
  if (rc == 0) {
    switch (am->hmminfo->cdset_method) {
      case IWCD_MAX: meth = JB200_IWCD_MAX; break;
      case IWCD_AVG: meth = JB200_IWCD_AVG; break;
      default: meth = JB200_IWCD_NBEST; break;
    }
    jb200_blob_add_i(b, "am.iwcd_method", meth);
    jb200_blob_add_i(b, "am.iwcd_nbest", am->hmminfo->cdmax_num);
    jb200_blob_add_i(b, "am.n_cdsets", cd.map.n);
    jb200_blob_add_i(b, "am.n_cdset_states", cd.states.n);
    jb200_blob_add(b, "am.cd_off", JB200_I32, cd.off.n, cd.off.d);
    jb200_blob_add(b, "am.cd_states", JB200_I32, cd.states.n, cd.states.d);
    if (cd.failed || b->failed) rc = oom();
  }
  pm_free(&cd.map); free(cd.off.d); free(cd.states.d);
  return rc;
}

int jb200_flatten_recog(Recog *recog, jb200_blob *b) {
  if (recog->amlist && (recog->amlist->next != NULL || (recog->process_list && recog->process_list->next != NULL)))
    jlog("WARNING: jb200: several AM/SR instances; only the first is flattened\n");
  return jb200_flatten(recog->amlist, recog->process_list, b);
}

/* ---------------------------------------------------------------- plugin ABI */
#ifndef JB200_NO_PLUGIN_ENTRY
int initialize(void) { return 0; }

int get_plugin_info(int opcode, char *buf, int buflen) {
  switch (opcode) {
    case 0: strncpy(buf, PLUGIN_TITLE, buflen); break;
  }
  return 0;
}

extern int jb200_attach(Recog *recog, jb200_blob *b);     /* jb200_attach.c */

int startup(void *data) {
  Recog *recog = (Recog *)data;
  const char *path = getenv("JB200_EXPORT");
  const char *attach = getenv("JB200_ATTACH");
  jb200_blob *b;
  int rc;
  const int want_attach = attach != NULL && (atoi(attach) != 0 || strcmp(attach, "calcmix") == 0);
  if (path == NULL && !want_attach) return 0;
  b = (jb200_blob *)malloc(sizeof(jb200_blob));
  if (b == NULL) return oom();
  jb200_blob_init(b);
  rc = jb200_flatten_recog(recog, b);
  if (rc == 0 && path != NULL) {
    rc = jb200_blob_save(b, path);
    if (rc == 0) jlog("STAT: jb200: flattened model written to %s (%d arrays)\n", path, b->n);
    else jlog("ERROR: jb200: cannot write %s\n", path);
  }
  if (rc == 0 && want_attach) return jb200_attach(recog, b);   /* keeps the blob alive */
  jb200_blob_free(b);
  free(b);
  return rc;
}
#endif /* JB200_NO_PLUGIN_ENTRY */
