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
 * This file reads reference structures only through their public headers; it
 * contains no reference code.
 */
#include <julius/juliuslib.h>
#include "jb200_model.h"

#define PLUGIN_TITLE "jb200 model flattener (GPU acoustic scoring + pass-1 beam)"

/* ---------------------------------------------------------------- tiny pointer map */
typedef struct { const void **k; int *v; int cap, n; } PMap;
static void pm_init(PMap *m, int cap) {
  int c = 64; while (c < cap * 2) c <<= 1;
  m->cap = c; m->n = 0;
  m->k = (const void **)calloc((size_t)c, sizeof(void *));
  m->v = (int *)calloc((size_t)c, sizeof(int));
}
static void pm_free(PMap *m) { free(m->k); free(m->v); }
static int pm_slot(const PMap *m, const void *p) {
  size_t h = ((size_t)p >> 3) * 0x9E3779B97F4A7C15ull;
  int i = (int)(h >> 20) & (m->cap - 1);
  while (m->k[i] != NULL && m->k[i] != p) i = (i + 1) & (m->cap - 1);
  return i;
}
static void pm_grow(PMap *m) {
  PMap n; int i;
  pm_init(&n, m->cap);
  for (i = 0; i < m->cap; i++) if (m->k[i]) { int s = pm_slot(&n, m->k[i]); n.k[s] = m->k[i]; n.v[s] = m->v[i]; n.n++; }
  pm_free(m); *m = n;
}
/* returns existing id or assigns next id (= current count) */
static int pm_intern(PMap *m, const void *p, int *is_new) {
  int s;
  if (m->n * 2 >= m->cap) pm_grow(m);
  s = pm_slot(m, p);
  if (m->k[s] == p) { if (is_new) *is_new = 0; return m->v[s]; }
  m->k[s] = p; m->v[s] = m->n; if (is_new) *is_new = 1;
  return m->n++;
}

/* growable int vector */
typedef struct { int *d; int n, cap; } IVec;
static void iv_push(IVec *v, int x) {
  if (v->n == v->cap) { v->cap = v->cap ? v->cap * 2 : 1024; v->d = (int *)realloc(v->d, sizeof(int) * v->cap); }
  v->d[v->n++] = x;
}

/* ---------------------------------------------------------------- cd-set registry */
typedef struct { PMap map; IVec off; IVec states; } CdReg;

static int cd_intern(CdReg *r, CD_State_Set *cs) {
  int is_new, id, i;
  id = pm_intern(&r->map, cs, &is_new);
  if (is_new) {
    for (i = 0; i < cs->num; i++) iv_push(&r->states, cs->s[i]->id);
    iv_push(&r->off, r->states.n);
  }
  return id;
}

/* ---------------------------------------------------------------- AM: GMM */
static int flatten_gmm(PROCESS_AM *am, jb200_blob *b) {
  HTK_HMM_INFO *hi = am->hmminfo;
  HTK_HMM_State *st;
  int S = hi->totalstatenum, D = hi->opt.vec_size, G = 0, i, d, m;
  int *off;
  float *mean, *ivar, *gconst, *lnw;
  unsigned char *valid;
  HTK_HMM_State **byid;

  if (hi->opt.stream_info.num != 1) { jlog("ERROR: jb200: multi-stream AM is not supported\n"); return -1; }
  if (hi->is_tied_mixture) {
    /* Tied-mixture (codebook) states are flattened into ordinary states: the mixture list of a <TMIX> state is its
     * codebook's densities with the state's own weights.  That IS what calc_tied_mix computes for -gprune none and
     * safe (calc_tied_mix.c:161-248: codebook scores once per frame, + weight[id], addlog_array in list order;
     * gprune_none lists ids in order, gprune_safe the N best sorted by score -- exactly what calc_mix does for a
     * private mixture).  The true beam/heuristic pruning of codebooks seeds itself with the previous frame's best
     * ids (calc_tied_mix.c:193-200), i.e. depends on which frames the search happened to evaluate: refused. */
    if (am->config->gprune_method == GPRUNE_SEL_BEAM || am->config->gprune_method == GPRUNE_SEL_HEURISTIC) {
      jlog("ERROR: jb200: tied-mixture AM with history-dependent Gaussian pruning; use -gprune none or -gprune safe\n");
      return -1;
    }
  }
  if (!hi->variance_inversed) { jlog("ERROR: jb200: variances are expected to be inverted at this point\n"); return -1; }
  byid = (HTK_HMM_State **)calloc((size_t)S, sizeof(void *));
  for (st = hi->ststart; st; st = st->next) {
    if (st->id < 0 || st->id >= S) { jlog("ERROR: jb200: state id out of range\n"); return -1; }
    byid[st->id] = st;
  }
  off = (int *)malloc(sizeof(int) * (S + 1));
  off[0] = 0;
  for (i = 0; i < S; i++) off[i + 1] = off[i] + (byid[i] ? byid[i]->pdf[0]->mix_num : 0);
  G = off[S];
  mean = (float *)calloc((size_t)G * D, sizeof(float));
  ivar = (float *)calloc((size_t)G * D, sizeof(float));
  gconst = (float *)calloc((size_t)G, sizeof(float));
  lnw = (float *)calloc((size_t)G, sizeof(float));
  valid = (unsigned char *)calloc((size_t)G, 1);
  for (i = 0; i < S; i++) {
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
  jb200_blob_add_i(b, "gmm.n_states", S);
  jb200_blob_add_i(b, "gmm.dim", D);
  jb200_blob_add_i(b, "gmm.n_gauss", G);
  jb200_blob_add_i(b, "gmm.max_mix", hi->maxmixturenum);
  {
    int meth = JB200_GPRUNE_NONE;
    switch (am->config->gprune_method) {
      case GPRUNE_SEL_SAFE: meth = JB200_GPRUNE_SAFE; break;
      case GPRUNE_SEL_HEURISTIC: meth = JB200_GPRUNE_HEU; break;
      case GPRUNE_SEL_BEAM: meth = JB200_GPRUNE_BEAM; break;
      default: meth = JB200_GPRUNE_NONE; break;
    }
    jb200_blob_add_i(b, "gmm.gprune_method", meth);
    jb200_blob_add_i(b, "gmm.gprune_num", am->hmmwrk.OP_gprune_num);
  }
  jb200_blob_add(b, "gmm.state_off", JB200_I32, S + 1, off);
  jb200_blob_add(b, "gmm.mean", JB200_F32, (int64_t)G * D, mean);
  jb200_blob_add(b, "gmm.ivar", JB200_F32, (int64_t)G * D, ivar);
  jb200_blob_add(b, "gmm.gconst", JB200_F32, G, gconst);
  jb200_blob_add(b, "gmm.lnweight", JB200_F32, G, lnw);
  jb200_blob_add(b, "gmm.valid", JB200_U8, G, valid);
  free(byid); free(off); free(mean); free(ivar); free(gconst); free(lnw); free(valid);
  return 0;
}

/* ---------------------------------------------------------------- AM: DNN */
static int flatten_dnn(PROCESS_AM *am, jb200_blob *b) {
  DNNData *dnn = am->dnn;
  int i, L = dnn->hnum + 1;
  char nm[48];
  if (L > JB200_DNN_MAX_LAYERS) { jlog("ERROR: jb200: too many DNN layers\n"); return -1; }
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
  return 0;
}

/* ---------------------------------------------------------------- tree + LM */
static int ctx_lookup(char **names, int n, const char *s) {
  int i;
  for (i = 0; i < n; i++) if (strcmp(names[i], s) == 0) return i;
  return -1;
}

static int flatten_tree(RecogProcess *r, CdReg *cd, jb200_blob *b) {
  WCHMM_INFO *w = r->wchmm;
  WORD_INFO *wi = w->winfo;
  HTK_HMM_INFO *hi = w->hmminfo;
  NGRAM_INFO *ng = w->ngram;
  int n = w->n, V = wi->num, i, k, narc = 0;
  int *arc_off, *arc_to, *stend, *scid, *out_ref;
  float *arc_a;
  unsigned char *outstyle;
  /* context classes */
  typedef struct { HMM_Logical *hmm; int loc; int style; int cat; } RKey;
  RKey *rkeys = NULL; int nr = 0, rcap = 0;
  char **ctxnames; int nctx = 0;
  int *word_ctx;
  char buf[MAX_HMMNAME_LEN], rbuf[MAX_HMMNAME_LEN];

  const int is_dfa = (w->lmtype == LM_DFA);
  if (is_dfa) {
    /* grammar mode: category tree + category-pair constraint only (beam.c:2404-2455) */
    if (w->lmvar != LM_DFA_GRAMMAR || !w->category_tree || w->dfa == NULL) {
      jlog("ERROR: jb200: grammar mode needs a category tree over a DFA grammar (isolated-word mode is not supported)\n");
      return -1;
    }
    if (w->dfa_forward != NULL) { jlog("ERROR: jb200: forward-DFA state tracking (.dfa.forward) is not supported\n"); return -1; }
  } else {
    if (w->lmtype != LM_PROB || (ng == NULL && w->lmvar != LM_NGRAM_USER)) { jlog("ERROR: jb200: lexicon tree without a language model\n"); return -1; }
    if (w->category_tree) { jlog("ERROR: jb200: category tree with an N-gram is not supported\n"); return -1; }
    if (w->lmvar == LM_NGRAM_USER) {
      /* -userlm (wchmm.h:274-276): pass 1 reads the LM through two host function pointers.  They cannot be called from
       * the device, so the 2-gram side is tabulated once -- a dense table over the dictionary, see below -- which bounds
       * the vocabulary this mode supports */
      const char *e = getenv("JB200_USERLM_MAXWORDS");
      const int lim = (e != NULL && atoi(e) > 0) ? atoi(e) : 8192;
      if (w->bi_prob_user == NULL) { jlog("ERROR: jb200: -userlm without a registered 2-gram function\n"); return -1; }
      if (ng != NULL) {
        /* the host caches these values per N-gram entry of the last word (factoring_sub.c:951-957,966: last_nword), so
         * with two dictionary words on one entry what it returns depends on which of them asked first */
        unsigned char *seen = (unsigned char *)calloc((size_t)ng->max_word_num + 1, 1);
        int dup = 0;
        for (i = 0; i < V && seen != NULL; i++) { if (seen[wi->wton[i]]) dup = 1; seen[wi->wton[i]] = 1; }
        free(seen);
        if (dup) { jlog("ERROR: jb200: -userlm with several dictionary words on one N-gram entry is not supported\n"); return -1; }
      }
      if (V > lim) { jlog("ERROR: jb200: -userlm is tabulated densely and supports up to %d words (JB200_USERLM_MAXWORDS), the dictionary has %d\n", lim, V); return -1; }
    }
  }

  /* ---- arcs (A_CELL2 lists, kept in the order beam_intra_word walks them, beam.c:2172-2176) */
  arc_off = (int *)malloc(sizeof(int) * (n + 1));
  for (i = 0; i < n; i++) {
    A_CELL2 *ac;
    arc_off[i] = narc;
    for (ac = w->ac[i]; ac; ac = ac->next) narc += ac->n;
  }
  arc_off[n] = narc;
  arc_to = (int *)malloc(sizeof(int) * (narc + 1));
  arc_a = (float *)malloc(sizeof(float) * (narc + 1));
  for (i = 0, k = 0; i < n; i++) {
    A_CELL2 *ac; int j;
    for (ac = w->ac[i]; ac; ac = ac->next) for (j = 0; j < ac->n; j++) { arc_to[k] = ac->arc[j]; arc_a[k] = ac->a[j]; k++; }
  }

  /* ---- left-context columns: centre phone of every word's last phone (cdhmm.c:129-160) */
  ctxnames = (char **)malloc(sizeof(char *) * (hi->basephone.num + 16));
  word_ctx = (int *)malloc(sizeof(int) * V);
  for (i = 0; i < V; i++) {
    int c;
    center_name(wi->wseq[i][wi->wlen[i] - 1]->name, buf);
    c = ctx_lookup(ctxnames, nctx, buf);
    if (c < 0) { ctxnames[nctx] = strdup(buf); c = nctx++; }
    word_ctx[i] = c;
  }

  /* ---- per node output reference */
  stend = (int *)malloc(sizeof(int) * n);
  scid = (int *)malloc(sizeof(int) * n);
  out_ref = (int *)malloc(sizeof(int) * n);
  outstyle = (unsigned char *)malloc((size_t)n);
  for (i = 0; i < n; i++) {
    stend[i] = (w->stend[i] == WORD_INVALID) ? -1 : (int)w->stend[i];
    scid[i] = is_dfa ? 0 : w->state[i].scid;      /* no factoring inside a category tree (beam.c:2028) */
    if (w->state[i].out.state == NULL) { outstyle[i] = 255; out_ref[i] = -1; continue; }
    switch (w->outstyle[i]) {
      case AS_STATE: outstyle[i] = JB200_AS_STATE; out_ref[i] = w->state[i].out.state->id; break;
      case AS_LSET:  outstyle[i] = JB200_AS_LSET;  out_ref[i] = cd_intern(cd, w->state[i].out.lset); break;
      case AS_RSET:
      case AS_LRSET: {
        HMM_Logical *h; int loc, style, j, found = -1, cat = -1;
        if (w->outstyle[i] == AS_RSET) { h = w->state[i].out.rset->hmm; loc = w->state[i].out.rset->state_loc; style = JB200_AS_RSET; }
        else {
          h = w->state[i].out.lrset->hmm; loc = w->state[i].out.lrset->state_loc; style = JB200_AS_LRSET;
          if (w->category_tree) cat = (int)w->state[i].out.lrset->category;     /* category-indexed cd sets, outprob_style.c:448-459 */
        }
        for (j = 0; j < nr; j++) if (rkeys[j].hmm == h && rkeys[j].loc == loc && rkeys[j].style == style && rkeys[j].cat == cat) { found = j; break; }
        if (found < 0) {
          if (nr == rcap) { rcap = rcap ? rcap * 2 : 256; rkeys = (RKey *)realloc(rkeys, sizeof(RKey) * rcap); }
          rkeys[nr].hmm = h; rkeys[nr].loc = loc; rkeys[nr].style = style; rkeys[nr].cat = cat; found = nr++;
        }
        outstyle[i] = (unsigned char)style; out_ref[i] = found;
      } break;
      default: jlog("ERROR: jb200: unknown outstyle\n"); return -1;
    }
  }

  /* ---- context table: replay outprob_style()'s resolution for every (class, context) */
  {
    int *tab = (int *)malloc(sizeof(int) * (size_t)(nr ? nr : 1) * (nctx + 1));
    int c;
    for (i = 0; i < nr; i++) {
      for (c = 0; c <= nctx; c++) {
        HMM_Logical *base = rkeys[i].hmm, *rhmm, *ohmm;
        int loc = rkeys[i].loc, ref;
        if (rkeys[i].style == JB200_AS_RSET) {
          /* outprob_style.c:385-436 */
          if (c < nctx && (ohmm = get_left_context_HMM(base, ctxnames[c], hi)) != NULL) rhmm = ohmm;
          else rhmm = base;
          if (rhmm->is_pseudo) ref = -cd_intern(cd, &(rhmm->body.pseudo->stateset[loc])) - 1;
          else ref = rhmm->body.defined->s[loc]->id;
        } else {
          /* outprob_style.c:437-486 */
          CD_Set *lcd;
          rhmm = base;
          strcpy(rbuf, rhmm->name);
          if (c < nctx) add_left_context(rbuf, ctxnames[c]);
          if (w->category_tree) {
            /* category-indexed cd sets (outprob_style.c:448-459) */
            if (c < nctx && (ohmm = get_left_context_HMM(rhmm, ctxnames[c], hi)) != NULL)
              lcd = lcdset_lookup_with_category(w, ohmm, (WORD_ID)rkeys[i].cat);
            else
              lcd = lcdset_lookup_with_category(w, rhmm, (WORD_ID)rkeys[i].cat);
          } else lcd = lcdset_lookup_by_hmmname(hi, rbuf);
          if (lcd != NULL) ref = -cd_intern(cd, &(lcd->stateset[loc])) - 1;
          else if (rhmm->is_pseudo) ref = -cd_intern(cd, &(rhmm->body.pseudo->stateset[loc])) - 1;
          else ref = rhmm->body.defined->s[loc]->id;
        }
        tab[(size_t)i * (nctx + 1) + c] = ref;
      }
    }
    jb200_blob_add(b, "tree.rset_ctx", JB200_I32, (int64_t)nr * (nctx + 1), tab);
    free(tab);
  }

  /* ---- roots in visiting order stid = startnum-1 .. 0 (beam.c:2334, :2565) */
  {
    IVec iso_node = {0}, iso_word = {0}, iso_id = {0}, shared = {0};
    int stid;
    for (stid = w->startnum - 1; stid >= 0; stid--) {
      int node = w->startnode[stid];
      int iso;
      if (is_dfa) {
        /* grammar mode: every root takes cross-word arrivals, gated by the category pair (beam.c:2404-2411) */
        iv_push(&iso_node, node); iv_push(&iso_id, stid); iv_push(&iso_word, (int)w->start2wid[stid]);
        continue;
      }
      iso = w->start2isolate[stid];
      if (iso == -1) { iv_push(&shared, node); continue; }
      if (w->state[node].scid <= 0) { jlog("ERROR: jb200: isolated root without successor word\n"); return -1; }
      iv_push(&iso_node, node); iv_push(&iso_id, iso); iv_push(&iso_word, (int)w->scword[w->state[node].scid]);
    }
    if (!is_dfa && iso_node.n != w->isolatenum) { jlog("ERROR: jb200: isolatenum mismatch\n"); return -1; }
    jb200_blob_add_i(b, "tree.n_iso", iso_node.n);
    jb200_blob_add_i(b, "tree.n_shared", shared.n);
    jb200_blob_add(b, "tree.iso_node", JB200_I32, iso_node.n, iso_node.d ? iso_node.d : (int *)&stid);
    jb200_blob_add(b, "tree.iso_word", JB200_I32, iso_word.n, iso_word.d ? iso_word.d : (int *)&stid);
    jb200_blob_add(b, "tree.iso_id", JB200_I32, iso_id.n, iso_id.d ? iso_id.d : (int *)&stid);
    jb200_blob_add(b, "tree.shared_node", JB200_I32, shared.n, shared.d ? shared.d : (int *)&stid);
    free(iso_node.d); free(iso_word.d); free(iso_id.d); free(shared.d);
  }

  /* ---- words */
  {
    float *wea = (float *)calloc((size_t)V, sizeof(float)), *cprob = (float *)calloc((size_t)V, sizeof(float));
    int *wend = (int *)malloc(sizeof(int) * V), *wbeg = (int *)malloc(sizeof(int) * V), *wton = (int *)malloc(sizeof(int) * V);
    unsigned char *tr = (unsigned char *)malloc((size_t)V);
    for (i = 0; i < V; i++) {
      wea[i] = hi->multipath ? 0.0f : w->wordend_a[i];
      wend[i] = w->wordend[i];
      wbeg[i] = hi->multipath ? w->wordbegin[i] : w->offset[i][0];
      wton[i] = (int)wi->wton[i];
      tr[i] = wi->is_transparent[i] ? 1 : 0;
#ifdef CLASS_NGRAM
      cprob[i] = wi->cprob[i];
#endif
      /* -userlm: the tabulated values below are indexed by dictionary word and already final (x + 0.0f == x) */
      if (!is_dfa && w->lmvar == LM_NGRAM_USER) { wton[i] = i; cprob[i] = 0.0f; }
    }
    jb200_blob_add(b, "tree.wordend_a", JB200_F32, V, wea);
    jb200_blob_add(b, "tree.wordend", JB200_I32, V, wend);
    jb200_blob_add(b, "tree.wordbegin", JB200_I32, V, wbeg);
    jb200_blob_add(b, "tree.wton", JB200_I32, V, wton);
    jb200_blob_add(b, "tree.is_transparent", JB200_U8, V, tr);
    jb200_blob_add(b, "tree.cprob", JB200_F32, V, cprob);
    free(wea); free(cprob); free(wend); free(wbeg); free(wton); free(tr);
  }

  if (is_dfa) {
    /* ---- grammar mode: category-pair table, sentence-initial words, penalty (beam.c:1669-1760, :2444-2450) */
    DFA_INFO *dfa = w->dfa;
    const int ns = w->startnum;
    unsigned char *cp = (unsigned char *)calloc((size_t)V * (ns ? ns : 1), 1);
    IVec iw_ = {0}, in_ = {0};
    float *il;
    MULTIGRAM *m;
    float zero = 0.0f; int izero = 0;
    for (i = 0; i < V; i++)
      for (k = 0; k < ns; k++)
        cp[(size_t)i * ns + k] = dfa_cp(dfa, (int)wi->wton[i], (int)wi->wton[w->start2wid[k]]) ? 1 : 0;
    for (m = r->lm->grammars; m; m = m->next) {
      int t, tb, te;
      if (!m->active) continue;
      tb = m->cate_begin; te = tb + m->dfa->term_num;
      for (t = tb; t < te; t++) {
        int x;
        if (!dfa_cp_begin(dfa, t)) continue;
        for (x = 0; x < dfa->term.wnum[t]; x++) {
          int wd = (int)dfa->term.tw[t][x], node = hi->multipath ? w->wordbegin[wd] : w->offset[wd][0], dup = 0, y;
          for (y = 0; y < in_.n; y++) if (in_.d[y] == node) { dup = 1; break; }     /* node_exist_token, beam.c:1719 */
          if (dup) continue;
          iv_push(&iw_, wd); iv_push(&in_, node);
        }
      }
    }
    il = (float *)calloc((size_t)(iw_.n ? iw_.n : 1), sizeof(float));
    for (i = 0; i < iw_.n; i++) {
      float ls = r->config->lmp.penalty1;
#ifdef CLASS_NGRAM
      ls += wi->cprob[iw_.d[i]];
#endif
      il[i] = ls;
    }
    jb200_blob_add_i(b, "tree.lm_type", JB200_LM_DFA);
    jb200_blob_add_i(b, "tree.n_init", iw_.n);
    jb200_blob_add_f(b, "tree.penalty1", r->config->lmp.penalty1);
    jb200_blob_add(b, "tree.init_word", JB200_I32, iw_.n, iw_.d ? iw_.d : &izero);
    jb200_blob_add(b, "tree.init_node", JB200_I32, in_.n, in_.d ? in_.d : &izero);
    jb200_blob_add(b, "tree.init_lscore", JB200_F32, iw_.n, il);
    jb200_blob_add(b, "tree.cp_allowed", JB200_U8, (int64_t)V * ns, cp);
    /* the N-gram side of the descriptor stays empty */
    jb200_blob_add_i(b, "tree.n_fscore", 0); jb200_blob_add_i(b, "tree.n_scword", 0);
    jb200_blob_add(b, "tree.fscore", JB200_F32, 0, &zero); jb200_blob_add(b, "tree.scword", JB200_I32, 0, &izero);
    jb200_blob_add_i(b, "tree.lm_nvocab", 0); jb200_blob_add_i(b, "tree.lm_nbigram", 0);
    jb200_blob_add_i(b, "tree.lm_mode", 0); jb200_blob_add_i(b, "tree.lm_unk_id", -1);
    jb200_blob_add_f(b, "tree.lm_unk_num_log", 0.0f);
    jb200_blob_add(b, "tree.uni_prob", JB200_F32, 0, &zero); jb200_blob_add(b, "tree.uni_bow", JB200_F32, 0, &zero);
    jb200_blob_add(b, "tree.bi_bgn", JB200_I32, 0, &izero); jb200_blob_add(b, "tree.bi_num", JB200_I32, 0, &izero);
    jb200_blob_add(b, "tree.bi_wid", JB200_I32, 0, &izero); jb200_blob_add(b, "tree.bi_prob", JB200_F32, 0, &zero);
    free(cp); free(iw_.d); free(in_.d); free(il);
  } else {
  /* ---- factoring values */
  {
    int *scw = (int *)calloc((size_t)w->scnum + 1, sizeof(int));
    for (i = 1; i < w->scnum; i++) scw[i] = (int)w->scword[i];
    jb200_blob_add_i(b, "tree.n_fscore", w->fsnum);
    jb200_blob_add_i(b, "tree.n_scword", w->scnum);
    jb200_blob_add(b, "tree.fscore", JB200_F32, w->fsnum, w->fscore);
    jb200_blob_add(b, "tree.scword", JB200_I32, w->scnum, scw);
    free(scw);
  }

  /* ---- LM */
  if (w->lmvar == LM_NGRAM_USER) {
    /* User-defined LM.  What pass 1 asks of it (factoring_sub.c:963-981 for a node with one successor word, :1118-1128
     * for the isolated roots) is  g(lw, w) = bi_prob_user(winfo, lw, w, ngram 2-gram(lw, w) + cprob[w])  with LOG_ZERO in
     * place of the N-gram term when no N-gram is loaded; the 1-gram factoring values (wchmm->fscore, above) went through
     * uni_prob_user when the host built the tree (wchmm.c:1497,1626).  g is tabulated as a DENSE 2-gram over the dictionary
     * itself: every row holds all V words, so the device's binary search always hits and returns the entry unchanged. */
    const int64_t VV = (int64_t)V * V;
    float *g = (float *)malloc(sizeof(float) * (size_t)VV), *zf = (float *)calloc((size_t)V, sizeof(float));
    int *bw = (int *)malloc(sizeof(int) * (size_t)VV), *bgn = (int *)malloc(sizeof(int) * V), *num = (int *)malloc(sizeof(int) * V);
    int a, c;
    if (!g || !zf || !bw || !bgn || !num) { jlog("ERROR: jb200: out of memory tabulating the user LM\n"); return -1; }
    for (a = 0; a < V; a++) {
      bgn[a] = a * V; num[a] = V;
      for (c = 0; c < V; c++) {
        LOGPROB p;
        if (ng != NULL) {
          p = (*(ng->bigram_prob))(ng, wi->wton[a], wi->wton[c])
#ifdef CLASS_NGRAM
            + wi->cprob[c]
#endif
            ;
        } else p = LOG_ZERO;
        g[(size_t)a * V + c] = (*(w->bi_prob_user))(wi, (WORD_ID)a, (WORD_ID)c, p);
        bw[(size_t)a * V + c] = c;
      }
    }
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
    free(g); free(zf); free(bw); free(bgn); free(num);
  } else {
    /* the 1-/2-gram tables bi_prob_*() reads (ngram_access.c:249-466) */
    NGRAM_TUPLE_INFO *t1 = &ng->d[0], *t2 = &ng->d[1];
    int Vn = ng->max_word_num, mode;
    const float *bow, *biprob;
    int *bgn = (int *)malloc(sizeof(int) * Vn), *num = (int *)malloc(sizeof(int) * Vn);
    int *bwid = (int *)malloc(sizeof(int) * (t2->totalnum + 1));
    if (t2->is24bit) { jlog("ERROR: jb200: 24-bit 2-gram index is not supported\n"); return -1; }
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
    free(bgn); free(num); free(bwid);
  }
  }

  /* ---- scalars + per-node arrays */
  jb200_blob_add_i(b, "tree.n_nodes", n);
  jb200_blob_add_i(b, "tree.n_arcs", narc);
  jb200_blob_add_i(b, "tree.n_words", V);
  jb200_blob_add_i(b, "tree.n_start", w->startnum);
  jb200_blob_add_i(b, "tree.n_rset", nr);
  jb200_blob_add_i(b, "tree.n_ctx", nctx);
  jb200_blob_add_i(b, "tree.head_silwid", (is_dfa || wi->head_silwid == WORD_INVALID) ? -1 : (int)wi->head_silwid);
  jb200_blob_add_i(b, "tree.tail_silwid", (is_dfa || wi->tail_silwid == WORD_INVALID) ? -1 : (int)wi->tail_silwid);
  jb200_blob_add_i(b, "tree.multipath", hi->multipath ? 1 : 0);
  jb200_blob_add_i(b, "tree.beam_width", r->trellis_beam_width);
  jb200_blob_add_f(b, "tree.lm_weight", r->config->lmp.lm_weight);
  jb200_blob_add_f(b, "tree.lm_penalty", r->config->lmp.lm_penalty);
  jb200_blob_add_f(b, "tree.lm_penalty_trans", r->pass1.lm_penalty_trans);   /* FSBeam copy, what beam.c:2441 reads */
  jb200_blob_add_f(b, "tree.score_pruning_width", r->config->pass1.score_pruning_width);
  jb200_blob_add(b, "tree.self_a", JB200_F32, n, w->self_a);
  jb200_blob_add(b, "tree.next_a", JB200_F32, n, w->next_a);
  jb200_blob_add(b, "tree.arc_off", JB200_I32, n + 1, arc_off);
  jb200_blob_add(b, "tree.arc_to", JB200_I32, narc, arc_to);
  jb200_blob_add(b, "tree.arc_a", JB200_F32, narc, arc_a);
  jb200_blob_add(b, "tree.stend", JB200_I32, n, stend);
  jb200_blob_add(b, "tree.scid", JB200_I32, n, scid);
  jb200_blob_add(b, "tree.outstyle", JB200_U8, n, outstyle);
  jb200_blob_add(b, "tree.out_ref", JB200_I32, n, out_ref);
  jb200_blob_add(b, "tree.word_ctx", JB200_I32, V, word_ctx);
  for (i = 0; i < nctx; i++) free(ctxnames[i]);
  free(ctxnames); free(word_ctx); free(rkeys);
  free(arc_off); free(arc_to); free(arc_a); free(stend); free(scid); free(out_ref); free(outstyle);
  return 0;
}

/* ---------------------------------------------------------------- entry: build the blob */
int jb200_flatten(PROCESS_AM *am, RecogProcess *r, jb200_blob *b) {
  CdReg cd;
  int rc = 0;

  memset(&cd, 0, sizeof(cd));
  pm_init(&cd.map, 4096);
  iv_push(&cd.off, 0);
  if (am == NULL) { jlog("ERROR: jb200: no acoustic model\n"); return -1; }

  if (am->dnn != NULL) rc = flatten_dnn(am, b);
  else rc = flatten_gmm(am, b);
  if (rc == 0 && r != NULL && r->wchmm != NULL) rc = flatten_tree(r, &cd, b);
  if (rc == 0) {
    int meth = JB200_IWCD_NBEST;
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
    jb200_blob_add(b, "am.cd_states", JB200_I32, cd.states.n, cd.states.d ? cd.states.d : cd.off.d);
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
