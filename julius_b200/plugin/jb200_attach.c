/* jb200_attach.c -- in-process attach of the GPU acoustic scorer to a running Julius engine.
 *
 * Part of the .jpi plugin (built with jb200_export.c).  With JB200_ATTACH=1 the startup() hook
 *   1. flattens the live models (jb200_export.c),
 *   2. loads libjb200.so and creates the GPU scorer (GMM, exact arithmetic by default; or DNN),
 *   3. registers a CALLBACK_EVENT_PASS1_BEGIN handler (libjulius/include/julius/callback.h:119) that,
 *      for buffered input (all T frames present), scores [T x S] on the GPU in one call and stores the
 *      rows in HMMWork.outprob_cache (libsent/include/sent/hmm_calc.h:115).  Every later
 *      outprob_state() (libsent/src/phmm/outprob.c:183-249) is a cache hit: pass 1, pass 2 and
 *      -outprobout all consume the GPU's numbers.  This is the "HMMWork function pointers / cache"
 *      boundary of SURVEY.md 8b.
 * It also provides the calcmix hook set so that "-gprune jb200" is a valid jconf value
 * (libjulius/src/plugin.c:336-354, contract plugin/calcmix.c:226-323): per-Gaussian ln scores of the
 * current frame come from the GPU (jb200_gmm_gauss_host), one device call per frame, sliced per state.
 * JB200_ATTACH=calcmix attaches only this hook (no cache fill), JB200_ATTACH=1 the whole-utterance scoring.
 * JB200_GMM_MODE=fast selects the FMA/exact-LSE arithmetic (<=1e-4) instead of the bit-exact one.
 */
#include "jb200_host.h"

static jb200_api g_api;
static jb200_scorer g_sc;
static jb200_rows g_in, g_scores;
/* calcmix state */
static float *g_gauss = NULL; static int g_gauss_time = -2;

static void on_pass1_begin(Recog *recog, void *dummy) {
  PROCESS_AM *am = recog->amlist;
  HMMWork *wrk = &(am->hmmwrk);
  HTK_Param *param = am->mfcc->param;
  const int T = param->samplenum, S = wrk->statenum, D = g_sc.gd.dim;
  int t, rc;
  (void)dummy;
  if (T <= 0 || param->is_outprob) return;
  if (recog->jconf->decodeopt.realtime_flag) {
    jlog("WARNING: jb200: real-time (frame-by-frame) input: the per-utterance GPU scoring is skipped\n");
    return;
  }
  if (param->veclen < D) { jlog("ERROR: jb200: parameter vector shorter than the model's input\n"); return; }
  if (jb200_rows_reserve(&g_scores, (size_t)T * S) != 0 || jb200_gather(&g_in, param, 0, T, D) != 0) {
    jlog("ERROR: jb200: out of memory\n");
    return;
  }
  rc = g_sc.dnn ? g_api.dnn_score_host(g_sc.dnn, g_in.x, T, g_scores.x) : g_api.gmm_score_host(g_sc.gmm, g_in.x, T, g_scores.x);
  if (rc != 0) { jlog("ERROR: jb200: GPU scoring failed: %s\n", g_api.last_error()); return; }
  /* make the cache rows exist (outprob_cache_extend is static: outprob.c:116), then overwrite them */
  outprob_state(wrk, T - 1, am->hmminfo->ststart, param);
  for (t = 0; t < T; t++) memcpy(wrk->outprob_cache[t], g_scores.x + (size_t)t * S, sizeof(float) * S);
  wrk->OP_time = -1;          /* force outprob_state() to re-latch its per-frame pointers */
  wrk->OP_last_time = -1;
}

/* calcmix-only attach: a new utterance must not reuse the last utterance's frame of Gaussian scores */
static void on_pass1_begin_calcmix(Recog *recog, void *dummy) { (void)recog; (void)dummy; g_gauss_time = -2; }

int jb200_attach(Recog *recog, jb200_blob *b) {
  const char *how = getenv("JB200_ATTACH");
  int rc;
  if (jb200_api_load(&g_api, (void *)&jb200_attach) != 0) return -1;
  rc = jb200_scorer_open(&g_sc, &g_api, b, 0);
  if (rc > 0) { jlog("ERROR: jb200: no acoustic model in the flattened blob\n"); return -1; }
  if (rc != 0) { jlog("ERROR: jb200: cannot create the GPU scorer: %s\n", g_api.last_error()); return -1; }
  if (how && strcmp(how, "calcmix") == 0) {
    /* only the -gprune jb200 surface: the host keeps calling outprob_state -> calc_mix -> calcmix() */
    callback_add(recog, CALLBACK_EVENT_PASS1_BEGIN, on_pass1_begin_calcmix, NULL);
    jlog("STAT: jb200: GPU Gaussian scoring attached behind the calcmix hook (-gprune jb200)\n");
    return 0;
  }
  callback_add(recog, CALLBACK_EVENT_PASS1_BEGIN, on_pass1_begin, NULL);
  jlog("STAT: jb200: GPU acoustic scoring attached (%s)\n", g_sc.dnn ? "DNN, tensor cores" : "GMM");
  return 0;
}

/* ---------------------------------------------------------------- calcmix hook set (-gprune jb200) */
void calcmix_get_optname(char *buf, int buflen) { strncpy(buf, "jb200", buflen); }

boolean calcmix_init(HMMWork *wrk) {
  /* same work-area contract as gprune_none_init (libsent/src/phmm/gprune_none.c:92-103) */
  wrk->OP_calced_maxnum = wrk->OP_hmminfo->maxmixturenum * wrk->OP_nstream;
  wrk->OP_calced_score = (LOGPROB *)malloc(sizeof(LOGPROB) * wrk->OP_calced_maxnum);
  wrk->OP_calced_id = (int *)malloc(sizeof(int) * wrk->OP_calced_maxnum);
  wrk->OP_gprune_num = wrk->OP_calced_maxnum;
  if (wrk->OP_calced_score == NULL || wrk->OP_calced_id == NULL) { jlog("ERROR: jb200: out of memory\n"); return FALSE; }
  return TRUE;
}

void calcmix_free(HMMWork *wrk) { free(wrk->OP_calced_score); free(wrk->OP_calced_id); }

void calcmix(HMMWork *wrk, HTK_HMM_Dens **g, int num, int *last_id, int lnum) {
  int i, base;
  (void)g; (void)last_id; (void)lnum;
  if (g_sc.gmm == NULL) { j_internal_error("jb200 calcmix: the GPU scorer is not attached (set JB200_ATTACH=1)\n"); return; }
  if (g_gauss == NULL && (g_gauss = (float *)malloc(sizeof(float) * (g_sc.gd.n_gauss + 1))) == NULL) {
    j_internal_error("jb200 calcmix: out of memory\n");
    return;
  }
  if (wrk->OP_time != g_gauss_time) {
    if (g_api.gmm_gauss_host(g_sc.gmm, wrk->OP_vec, g_gauss) != 0) j_internal_error("jb200 calcmix: %s\n", g_api.last_error());
    g_gauss_time = wrk->OP_time;
  }
  base = g_sc.gd.state_off[wrk->OP_state_id];
  for (i = 0; i < num; i++) { wrk->OP_calced_score[i] = g_gauss[base + i]; wrk->OP_calced_id[i] = i; }
  wrk->OP_calced_num = num;
}
