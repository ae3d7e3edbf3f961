/* jb200_beam_shim.c -- link-time replacement of libjulius/src/beam.c's entry points.
 *
 * pass1.c calls the pass-1 beam by name (libjulius/src/pass1.c:234,242,503,409/567;
 * libjulius/include/julius/extern.h:56-61).  Linking libjulius with this object INSTEAD of beam.o
 * turns the stock Julius host into a front for the GPU path, jconf surface unchanged:
 *
 *   get_back_trellis_init(param, r)      beam.c:1825  bt_prepare and the per-utterance host state, as the original
 *   get_back_trellis_proceed(t, ...)     beam.c:2663  two modes.  Buffered (default for file input): nothing per frame.
 *                                                    Frame-synchronous (real-time input, -progout, or JB200_STREAM=1):
 *                                                    frame t has just arrived in param (realtime-1stpass.c:681 calls
 *                                                    _init with ONE frame and grows param as audio comes in); the
 *                                                    frames not yet decoded are fed to the device stream every
 *                                                    JB200_STREAM_FRAMES frames (default 10 = 100 ms), and always when
 *                                                    the host is due an interim result (beam.c:2983-2993: every
 *                                                    progout_interval_frame frames r->result.pass1 gets the best word
 *                                                    sequence so far and have_interim is raised); returns FALSE once
 *                                                    the beam ran empty (beam.c:3012-3015)
 *   get_back_trellis_end(param, r)       beam.c:3052  param now holds ALL frames of the input.  Buffered mode: this is
 *                                                    where the utterance is scored and decoded on the GPU
 *                                                    (jb200_decode_batch_host); frame-synchronous mode: the remaining
 *                                                    frames go to the stream together with the end-of-utterance mark.
 *                                                    Either way r->backtrellis is materialised from the GPU's atoms
 *                                                    through bt_new/bt_store (backtrellis.c:154,190)
 *   finalize_1st_pass(r, len)            beam.c:3133  bt_relocate_rw + bt_sort_rw, then publishes the
 *                                                    pass-1 best exactly where find_1pass_result does
 *                                                    (beam.c:497-512)
 *   fsbeam_free(d)                       beam.c:3180
 * Restrictions (checked, fail loudly): N-gram LM, no short-pause segmentation, feature-vector input at least as wide
 * as the model's.
 * (normal and multipath trees both run on the device).  The models are flattened on first use with the same code as the plugin.
 */
#include "jb200_host.h"
#include <time.h>

static double shim_now(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec + 1e-9 * ts.tv_nsec; }

extern int jb200_flatten(PROCESS_AM *am, RecogProcess *r, jb200_blob *b);   /* jb200_export.c */

/* one decoded utterance, copied out of the decoder (decode-ahead cache, and the current utterance) */
typedef struct {
  unsigned long long hash;   /* of the feature vectors it was decoded from */
  int n_frames;
  jb200_utt_result u;
  jb200_atom *atoms;         /* [u.n_atoms] */
  int32_t *words;            /* [u.n_words] */
} ShimResult;

typedef struct {
  RecogProcess *r;
  jb200_blob blob;
  jb200_tree_desc td;
  jb200_scorer sc;
  jb200_decoder *dec;
  int max_frames, max_utts;
  boolean ok;            /* last decode succeeded */
  /* options, read once when the instance is attached */
  boolean verbose;       /* JB200_SHIM_VERBOSE: a line per interim result, decode-ahead batch and cached utterance */
  int stream_opt;        /* JB200_STREAM: 1 / 0 forces frame-synchronous / buffered decoding, -1 lets the input decide */
  int stream_frames;     /* JB200_STREAM_FRAMES: feed granularity (default 10 frames) */
  const char *filelist;  /* JB200_FILELIST: the list given to -filelist, or NULL */
  int ahead_files;       /* JB200_AHEAD: files per decode-ahead batch (default 32) */
  /* frame-synchronous mode */
  boolean streaming;     /* this utterance runs on a device stream */
  int fed;               /* frames handed to the stream so far */
  jb200_rows in;         /* the frames of one feed, or of one buffered utterance */
  ShimResult cur;        /* result of the utterance being finished */
  /* decode-ahead over the file list */
  char **files; int n_files, next_file;   /* n_files: 0 = not read yet, -1 = none; next_file: the utterance the host finishes next */
  jb200_rows batch;      /* the frames of one decode-ahead batch */
  ShimResult *ahead; int n_ahead, ahead_first;
  long n_from_cache, n_single;
} Shim;

static jb200_api g_api;
static int g_api_loaded = 0;
static Shim g_shim[8];
static int g_nshim = 0;

static int shim_oom(void) { jlog("ERROR: jb200: out of memory\n"); return -1; }
static int shim_api_error(void) { jlog("ERROR: jb200: %s\n", g_api.last_error()); return -1; }

/* ---- results: copies that outlive the decoder's buffers -------------------------------------------------------- */
static void result_free(ShimResult *x) { free(x->atoms); free(x->words); memset(x, 0, sizeof(*x)); }

static int result_copy(ShimResult *x, const jb200_utt_result *u, const jb200_atom *atoms, const int32_t *words) {
  result_free(x);
  x->u = *u;
  x->atoms = (jb200_atom *)malloc(sizeof(jb200_atom) * (size_t)(u->n_atoms > 0 ? u->n_atoms : 1));
  x->words = (int32_t *)malloc(sizeof(int32_t) * (size_t)(u->n_words > 0 ? u->n_words : 1));
  if (!x->atoms || !x->words) { result_free(x); return shim_oom(); }
  if (u->n_atoms > 0) memcpy(x->atoms, atoms + u->atom_offset, sizeof(jb200_atom) * (size_t)u->n_atoms);
  if (u->n_words > 0) memcpy(x->words, words + u->word_offset, sizeof(int32_t) * (size_t)u->n_words);
  x->u.atom_offset = 0; x->u.word_offset = 0;
  return 0;
}

static void ahead_clear(Shim *s) {
  int i;
  for (i = 0; i < s->n_ahead; i++) result_free(&s->ahead[i]);
  free(s->ahead); s->ahead = NULL; s->n_ahead = 0;
}

static void files_free(Shim *s) {
  int i;
  for (i = 0; i < s->n_files; i++) free(s->files[i]);
  free(s->files); s->files = NULL; s->n_files = -1;
}

/* ---- the recognition instances ----------------------------------------------------------------------------------- */
/* releases everything an instance holds on the device and the host, and empties its slot */
static void shim_release(Shim *s) {
  if (s->dec) g_api.decoder_destroy(s->dec);
  jb200_scorer_close(&s->sc, &g_api);
  ahead_clear(s); result_free(&s->cur); files_free(s);
  free(s->in.x); free(s->batch.x);
  jb200_blob_free(&s->blob);
  memset(s, 0, sizeof(*s));
}

/* the instance of r, or NULL before its first utterance */
static Shim *shim_get(RecogProcess *r) {
  int i;
  for (i = 0; i < g_nshim; i++) if (g_shim[i].r == r) return &g_shim[i];
  return NULL;
}

/* First use of r: checks the restrictions, flattens the models, opens the scorer and reads the options.  NULL after an
 * error (logged); nothing is kept then, and the next utterance tries again. */
static Shim *shim_attach(RecogProcess *r) {
  Shim *s;
  const char *e;
  int rc;
  if (!g_api_loaded) { if (jb200_api_load(&g_api, (void *)&shim_attach) != 0) return NULL; g_api_loaded = 1; }
  if (g_nshim >= 8) { jlog("ERROR: jb200: too many recognition instances\n"); return NULL; }
  if (r->lmtype != LM_PROB || r->config->successive.enabled) {
    jlog("ERROR: jb200: the GPU beam supports N-gram, non-segmented decoding only\n");
    return NULL;
  }
  s = &g_shim[g_nshim];
  memset(s, 0, sizeof(*s));
  jb200_blob_init(&s->blob);
  rc = jb200_flatten(r->am, r, &s->blob);
  if (rc == 0 && (rc = jb200_tree_from_blob(&s->blob, &s->td)) != 0) jlog("ERROR: jb200: no lexicon tree in the flattened model\n");
  if (rc == 0 && (rc = jb200_scorer_open(&s->sc, &g_api, &s->blob, 1)) != 0) {
    if (rc > 0) jlog("ERROR: jb200: no acoustic model\n");
    else shim_api_error();
  }
  if (rc != 0) { shim_release(s); return NULL; }
  s->r = r;
  s->verbose = getenv("JB200_SHIM_VERBOSE") != NULL;
  s->stream_opt = (e = getenv("JB200_STREAM")) != NULL ? (atoi(e) != 0) : -1;
  s->stream_frames = ((e = getenv("JB200_STREAM_FRAMES")) != NULL && atoi(e) > 0) ? atoi(e) : 10;
  s->filelist = getenv("JB200_FILELIST");
  s->ahead_files = (e = getenv("JB200_AHEAD")) != NULL ? atoi(e) : 32;
  g_nshim++;
  jlog("STAT: jb200: GPU pass-1 beam attached to %02d %s\n", r->config->id, r->config->name);
  return s;
}

/* A decoder for at least `frames` frames in `utts` utterances.  A new one is sized for the longest input seen so far:
 * the old one (device work areas, pinned host buffers) is released first, and the capacity is recorded only once the
 * new one exists.  0, or -1 after an error (logged). */
static int shim_reserve(Shim *s, int frames, int utts) {
  int want = frames < 4096 ? 4096 : frames + frames / 2, rc;
  const int want_utts = utts > s->max_utts ? utts : (s->max_utts > 0 ? s->max_utts : 1);
  if (frames <= s->max_frames && utts <= s->max_utts) return 0;
  if (want < s->max_frames) want = s->max_frames;
  if (s->dec) { g_api.decoder_destroy(s->dec); s->dec = NULL; s->max_frames = 0; s->max_utts = 0; }
  rc = g_api.decoder_create(&s->td, s->sc.gmm, want_utts, want, &s->dec);
  if (rc == 0 && s->sc.dnn) rc = g_api.decoder_attach_dnn(s->dec, s->sc.dnn);
  if (rc != 0) {
    shim_api_error();
    if (s->dec) { g_api.decoder_destroy(s->dec); s->dec = NULL; }
    return -1;
  }
  s->max_frames = want; s->max_utts = want_utts;
  return 0;
}

boolean get_back_trellis_init(HTK_Param *param, RecogProcess *r) {
  Shim *s;
  bt_prepare(r->backtrellis);
  r->pass1.bos.wid = WORD_INVALID;
  r->pass1.bos.begintime = r->pass1.bos.endtime = -1;
  /* host-side state that init_nodescore resets per utterance and pass 2 relies on (beam.c:1595):
   * the per-node triphone caches of outprob_style (bt_discount_pescore and the stack decoder read them) */
  outprob_style_cache_init(r->wchmm);
  r->config->output.progout_interval_frame = (int)((float)r->config->output.progout_interval / ((float)param->header.wshift / 10000.0));
  if ((s = shim_get(r)) == NULL && (s = shim_attach(r)) == NULL) return FALSE;
  s->ok = FALSE;
  if (shim_reserve(s, 1, 1) != 0) return FALSE;
  if (param->is_outprob) { jlog("ERROR: jb200: outprob-vector input is not supported by the GPU beam shim\n"); return FALSE; }
  if (param->veclen < s->sc.gd.dim) {
    jlog("ERROR: jb200: input vectors have %d components, the acoustic model takes %d\n", (int)param->veclen, s->sc.gd.dim);
    return FALSE;
  }
  /* frame-synchronous decoding when the input is live, when the host wants interim results, or on request */
  {
    /* live input: realtime-1stpass.c:681-682 hands _init the first frame alone (a RecogProcess has no way to ask its
     * Recog for decodeopt.realtime_flag); a buffered one-frame input takes the same route, which is equally right */
    const boolean live = (param->samplenum <= 1);
    const int shift = (r->am != NULL && r->am->config != NULL) ? r->am->config->analysis.para.frameshift : 0;
    s->streaming = (s->stream_opt >= 0) ? s->stream_opt : (live || r->config->output.progout_flag);
    s->fed = 0;
    if (s->streaming) {
      /* live input has no length yet: room for the longest input the host accepts (MAXSPEECHLEN samples) */
      int cap = (shift > 0) ? MAXSPEECHLEN / shift + 16 : 4096;
      if (cap < (int)param->samplenum) cap = param->samplenum;
      if (shim_reserve(s, cap, 1) != 0) return FALSE;
      if (g_api.stream_open(s->dec, 1) != 0) { shim_api_error(); return FALSE; }
    }
  }
  return TRUE;
}

/* hand frames [s->fed, upto) of param to the device stream */
static boolean stream_push(Shim *s, HTK_Param *param, int upto, boolean last, boolean interim) {
  int32_t n_new = upto - s->fed; uint8_t fin = last ? 1 : 0;
  if (n_new < 0) return FALSE;
  if (jb200_gather(&s->in, param, s->fed, upto, s->sc.gd.dim) != 0) { shim_oom(); return FALSE; }
  if (g_api.stream_feed_host(s->dec, s->in.x, &n_new, &fin, interim ? 1 : 0) != 0) { shim_api_error(); return FALSE; }
  s->fed = upto;
  return TRUE;
}

boolean get_back_trellis_proceed(int t, HTK_Param *param, RecogProcess *r, boolean final_for_multipath) {
  Shim *s = shim_get(r);
  boolean want_interim;
  r->have_interim = FALSE;
  if (s == NULL || !s->streaming || final_for_multipath) return TRUE;
  /* beam.c:2983-2993: after frame t the best path ending at t-1 is published every progout_interval_frame frames */
  want_interim = (t > 0 && r->config->output.progout_flag && r->config->output.progout_interval_frame > 0 &&
                  ((t - 1) % r->config->output.progout_interval_frame) == 0);
  if (t + 1 - s->fed < s->stream_frames && !want_interim) return TRUE;
  if (!stream_push(s, param, t + 1, FALSE, want_interim)) return FALSE;
  {
    int32_t done = 0, alive = 1, ended = 0;
    g_api.stream_status(s->dec, 0, &done, &alive, &ended);
    if (!alive) {
      jlog("ERROR: get_back_trellis_proceed: %02d %s: frame %d: no nodes left in beam, now terminates search\n", r->config->id, r->config->name, t);
      return FALSE;
    }
  }
  if (want_interim) {
    int32_t words[MAXSEQNUM], nw = 0, frame = -1; float score = LOG_ZERO; int i;
    if (g_api.stream_partial(s->dec, 0, words, MAXSEQNUM, &nw, &score, &frame) == 0) {
      /* what bt_current_max leaves in r->result (beam.c:898-920) */
      r->have_interim = TRUE;
      r->result.status = J_RESULT_STATUS_SUCCESS;
      r->result.num_frame = t - 1;
      r->result.pass1.word_num = nw;
      for (i = 0; i < nw; i++) r->result.pass1.word[i] = (WORD_ID)words[i];
      if (nw > 0) { r->result.pass1.score = score; r->result.pass1.score_am = score; r->result.pass1.score_lm = 0.0; }
      if (s->verbose) { printf("JB200_SHIM interim t=%d words=%d score=%f\n", t, (int)nw, score); fflush(stdout); }
    }
  }
  return TRUE;
}

static unsigned long long feat_hash(const float *x, size_t n) {      /* FNV-1a over the bit patterns */
  const unsigned char *b = (const unsigned char *)x;
  unsigned long long h = 1469598103934665603ULL;
  size_t i;
  for (i = 0; i < n * sizeof(float); i++) { h ^= b[i]; h *= 1099511628211ULL; }
  return h;
}

/* ---- decode-ahead: the host hands over one utterance at a time (pass1.c:220-254), one utterance occupies one of several
 * hundred resident thread blocks.  With JB200_FILELIST = the list the host reads its HTK parameter files from, the shim
 * reads the next JB200_AHEAD files itself, decodes them in ONE batch, and answers the host's following utterances from
 * the cache -- but only when the vectors the host presents hash to what was decoded (any host-side processing of the
 * input, or a list that does not match, silently falls back to the one-utterance path). */

/* Appends the vectors of an HTK parameter file to m at frame `at`.  Returns the number of frames; 0 when the file cannot
 * be read or does not hold D-component vectors; -1 when out of memory. */
static int read_htk_param(const char *fn, int D, jb200_rows *m, int at) {
  FILE *fp = fopen(fn, "rb");
  unsigned char h[12];
  unsigned int ns, ssize;
  float *x; size_t i, n;
  if (!fp) return 0;
  if (fread(h, 1, 12, fp) != 12) { fclose(fp); return 0; }
  ns = ((unsigned)h[0] << 24) | ((unsigned)h[1] << 16) | ((unsigned)h[2] << 8) | h[3];
  ssize = ((unsigned)h[8] << 8) | h[9];
  if (ns < 1 || ns > 32767 || ssize != (unsigned)D * 4u) { fclose(fp); return 0; }
  n = (size_t)ns * D;
  if (jb200_rows_reserve(m, (size_t)at * D + n) != 0) { fclose(fp); return -1; }
  x = m->x + (size_t)at * D;
  if (fread(x, 4, n, fp) != n) { fclose(fp); return 0; }
  fclose(fp);
  for (i = 0; i < n; i++) {                                           /* big-endian floats (rdparam.c:83-187) */
    unsigned char *b = (unsigned char *)(x + i), t;
    t = b[0]; b[0] = b[3]; b[3] = t; t = b[1]; b[1] = b[2]; b[2] = t;
  }
  return (int)ns;
}

/* s->files <- the names in s->filelist; n_files = -1 when it gives none.  0, or -1 when out of memory. */
static int load_filelist(Shim *s) {
  char line[4096]; FILE *fp = fopen(s->filelist, "r");
  if (!fp) { s->n_files = -1; return 0; }
  while (fgets(line, sizeof(line), fp)) {
    size_t L = strlen(line);
    char **f;
    while (L > 0 && (line[L - 1] == '\n' || line[L - 1] == '\r' || line[L - 1] == ' ')) line[--L] = '\0';
    if (L == 0 || line[0] == '#') continue;
    f = (char **)realloc(s->files, sizeof(char *) * (size_t)(s->n_files + 1));
    if (f != NULL) s->files = f;
    if (f == NULL || (s->files[s->n_files] = strdup(line)) == NULL) { fclose(fp); files_free(s); return shim_oom(); }
    s->n_files++;
  }
  fclose(fp);
  jlog("STAT: jb200: decode-ahead over %d files of %s\n", s->n_files, s->filelist);
  if (s->n_files == 0) s->n_files = -1;
  return 0;
}

static boolean ahead_has(const Shim *s, int utt) { return s->n_ahead > 0 && utt >= s->ahead_first && utt < s->ahead_first + s->n_ahead; }

/* Decodes files [first, first + ahead_files) of the list in one batch into the cache.  The batch ends before the first
 * file that cannot be read; with fewer than two files there is none.  0, or -1 after an error (logged). */
static int ahead_fill(Shim *s, int first) {
  const int D = s->sc.gd.dim, k = s->n_files - first < s->ahead_files ? s->n_files - first : s->ahead_files;
  const jb200_utt_result *u; const jb200_atom *a; const int32_t *w;
  const double t0 = shim_now();
  double t1, t2;
  int32_t *off;
  int i, n = 0, T = 0, rc = 0;
  ahead_clear(s);
  if (k < 2) return 0;
  if ((off = (int32_t *)malloc(sizeof(int32_t) * (size_t)(k + 1))) == NULL) return shim_oom();
  off[0] = 0;
  while (n < k && (T = read_htk_param(s->files[first + n], D, &s->batch, off[n])) > 0) { off[n + 1] = off[n] + T; n++; }
  t1 = shim_now();
  if (T < 0) rc = shim_oom();
  else if (n >= 2 && (rc = shim_reserve(s, off[n], n)) == 0) {
    t2 = shim_now();
    if (g_api.decode_batch_host(s->dec, s->batch.x, off, n) != 0 || g_api.decoder_results(s->dec, &u, &a, &w) != 0)
      jlog("WARNING: jb200: decode-ahead batch failed (%s); continuing one utterance at a time\n", g_api.last_error());
    else if ((s->ahead = (ShimResult *)calloc((size_t)n, sizeof(ShimResult))) == NULL) rc = shim_oom();
    else {
      s->n_ahead = n; s->ahead_first = first;
      if (s->verbose) { printf("JB200_SHIM batch first=%d n=%d frames=%d read=%.3fs decoder=%.3fs decode=%.3fs\n", first, n, off[n], t1 - t0, t2 - t1, shim_now() - t2); fflush(stdout); }
      for (i = 0; i < n && rc == 0; i++) {
        rc = result_copy(&s->ahead[i], &u[i], a, w);
        s->ahead[i].hash = feat_hash(s->batch.x + (size_t)off[i] * D, (size_t)(off[i + 1] - off[i]) * D);
        s->ahead[i].n_frames = off[i + 1] - off[i];
      }
    }
  }
  free(off);
  return rc;
}

/* s->cur <- the result of the utterance in param: from the device stream, from the decode-ahead cache, or decoded on
 * its own.  0, or -1 after an error (logged). */
static int shim_result(Shim *s, HTK_Param *param) {
  const int T = param->samplenum, D = s->sc.gd.dim;
  const jb200_utt_result *u; const jb200_atom *a; const int32_t *w;
  int32_t off[2];
  int utt;
  if (s->streaming) {
    /* frame-synchronous mode: the rest of the input and the end-of-utterance mark */
    if (!stream_push(s, param, T, TRUE, FALSE)) return -1;
    if (g_api.stream_result(s->dec, 0, &u, &a, &w) != 0) return shim_api_error();
    if (result_copy(&s->cur, u, a, w) != 0) return -1;
    s->next_file++;
    return 0;
  }
  if (shim_reserve(s, T, 1) != 0) return -1;
  if (jb200_gather(&s->in, param, 0, T, D) != 0) return shim_oom();
  utt = s->next_file++;
  if (s->filelist != NULL && s->n_files == 0 && load_filelist(s) != 0) return -1;
  if (utt < s->n_files) {
    if (!ahead_has(s, utt) && ahead_fill(s, utt) != 0) return -1;
    if (ahead_has(s, utt)) {
      const ShimResult *c = &s->ahead[utt - s->ahead_first];
      if (c->atoms != NULL && c->n_frames == T && c->hash == feat_hash(s->in.x, (size_t)T * D)) {
        if (result_copy(&s->cur, &c->u, c->atoms, c->words) != 0) return -1;
        s->n_from_cache++;
        if (s->verbose) { printf("JB200_SHIM utt=%d from_cache\n", utt); fflush(stdout); }
        return 0;
      }
    }
  }
  off[0] = 0; off[1] = T;
  if (g_api.decode_batch_host(s->dec, s->in.x, off, 1) != 0 || g_api.decoder_results(s->dec, &u, &a, &w) != 0) return shim_api_error();
  if (result_copy(&s->cur, u, a, w) != 0) return -1;
  s->n_single++;
  return 0;
}

/* r->backtrellis <- the atoms of x, through bt_new / bt_store (backtrellis.c:154,190); FALSE when out of memory */
static boolean store_trellis(RecogProcess *r, const ShimResult *x) {
  const jb200_atom *a = x->atoms;
  TRELLIS_ATOM **idx = (TRELLIS_ATOM **)malloc(sizeof(void *) * (size_t)(x->u.n_atoms + 1));
  int i;
  if (idx == NULL) { shim_oom(); return FALSE; }
  for (i = 0; i < x->u.n_atoms; i++) {
    TRELLIS_ATOM *tre = bt_new(r->backtrellis);
    tre->wid = (WORD_ID)a[i].wid;
    tre->begintime = (short)a[i].begintime; tre->endtime = (short)a[i].endtime;
    tre->backscore = a[i].backscore; tre->lscore = a[i].lscore;
    tre->dfa_state = -1;
    tre->last_tre = (a[i].last < 0) ? &(r->pass1.bos) : idx[a[i].last];
    bt_store(r->backtrellis, tre);
    idx[i] = tre;
  }
  free(idx);
  return TRUE;
}

void get_back_trellis_end(HTK_Param *param, RecogProcess *r) {
  Shim *s = shim_get(r);
  if (s == NULL) return;
  s->ok = FALSE;
  if (param->samplenum < 1 || param->is_outprob || param->veclen < s->sc.gd.dim) return;       /* refused at _init already */
  if (shim_result(s, param) != 0) return;
  if (s->cur.u.overflow) { jlog("ERROR: jb200: device work area overflow (code %d); pass 1 result dropped\n", s->cur.u.overflow); return; }
  s->ok = store_trellis(r, &s->cur);
}

void finalize_1st_pass(RecogProcess *r, int len) {
  const jb200_utt_result *u; const jb200_atom *a; const int32_t *w;
  BACKTRELLIS *bt = r->backtrellis;
  Shim *s = shim_get(r);
  int i;
  bt->framelen = len;
  bt_relocate_rw(bt);
  bt_sort_rw(bt);
  if (bt->num == NULL || s == NULL || !s->ok) {
    if (bt->framelen > 0) jlog("WARNING: %02d %s: input processed, but no survived word found\n", r->config->id, r->config->name);
    r->result.status = J_RESULT_STATUS_FAIL;
    return;
  }
  u = &s->cur.u; a = s->cur.atoms; w = s->cur.words;
  if (u->status != 0) {
    jlog("WARNING: %02d %s: no tail silence word survived on the last frame, search failed\n", r->config->id, r->config->name);
    r->result.status = J_RESULT_STATUS_FAIL;
    return;
  }
  /* what find_1pass_result publishes (beam.c:497-517) */
  r->result.status = J_RESULT_STATUS_SUCCESS;
  r->result.num_frame = len;
  for (i = 0; i < u->n_words; i++) r->result.pass1.word[i] = (WORD_ID)w[i];
  r->result.pass1.word_num = u->n_words;
  r->result.pass1.score = u->score;
  {
    /* total LM score along the best path = sum of lscore of its atoms (trace_backptr, beam.c:253-301) */
    LOGPROB lsum = 0.0; int k, best = -1;
    for (k = u->n_atoms - 1; k >= 0 && best < 0; k--)
      if (a[k].wid == (int)r->lm->winfo->tail_silwid && a[k].backscore == u->score) best = k;
    for (k = best; k >= 0; k = a[k].last) { lsum += a[k].lscore; if (a[k].begintime <= 0) break; }
    r->result.pass1.score_lm = lsum;
    r->result.pass1.score_am = u->score - lsum;
  }
  for (i = 0; i < u->n_words; i++) r->pass1_wseq[i] = (WORD_ID)w[i];
  r->pass1_wnum = u->n_words;
  r->pass1_score = u->score;
}

void fsbeam_free(FSBeam *d) {
  int i;
  if (d->pausemodelnames != NULL) { free(d->pausemodelnames); free(d->pausemodel); }
  if (d->boslist != NULL) free(d->boslist);
  /* release the device side of the recognition instance this work area belongs to */
  for (i = 0; i < g_nshim; i++) {
    Shim *s = &g_shim[i];
    if (s->r == NULL || &(s->r->pass1) != d) continue;
    if (s->n_files > 0) jlog("STAT: jb200: %ld utterances answered from decode-ahead batches, %ld decoded singly\n", s->n_from_cache, s->n_single);
    shim_release(s);
  }
}
