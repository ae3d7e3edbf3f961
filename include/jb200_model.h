/* jb200_model.h -- flattened (pointer-free) model descriptors and their blob container.
 *
 * The reference keeps its models as pointer graphs (HTK_HMM_INFO, WCHMM_INFO,
 * NGRAM_INFO ...).  Everything the hot path reads is flattened once, on the
 * host, into the plain arrays below; the arrays are what goes to HBM.  The
 * same descriptors are filled
 *   - by the .jpi plugin's startup(Recog*) hook straight from the live Julius
 *     structures (julius_b200/plugin/jb200_export.c), and
 *   - from a "JB2M" blob file written by that plugin (offline harness, tests,
 *     bench), via jb200_blob_load().
 *
 * Reference structures flattened here (file:line in /root/reference):
 *   GMM    HTK_HMM_INFO / HTK_HMM_State / HTK_HMM_PDF / HTK_HMM_Dens
 *          libsent/include/sent/htk_hmm.h:104-253; inverted variances
 *          libsent/src/phmm/outprob_init.c:75-79
 *   CDSET  CD_State_Set            libsent/include/sent/htk_hmm.h:249-253
 *   TREE   WCHMM_INFO              libjulius/include/julius/wchmm.h:211-278
 *          A_CELL2 arc cells       wchmm.h:162-172  (kept in list order)
 *          RC_INFO / LRC_INFO      wchmm.h:55-83    (tabulated per left-context phone)
 *   LM     NGRAM_INFO 1-/2-gram    libsent/include/sent/ngram2.h:137-188
 *   WORDS  WORD_INFO wton/cprob/is_transparent  libsent/include/sent/vocabulary.h
 *   DNN    DNNData / DNNLayer      libsent/include/sent/dnn.h:25-74
 *
 * Plain C, no torch / CUDA types: this header is part of the C-ABI boundary.
 */
#ifndef JB200_MODEL_H
#define JB200_MODEL_H

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#ifdef __cplusplus
extern "C" {
#endif

/* reference constants (libsent/include/sent/stddefs.h:107-111,171-176) */
#define JB200_LOG_ZERO      (-1000000.0f)
#define JB200_LOG_ADDMIN    (-13.815510558)
#define JB200_LOG_TEN       2.30258509
#define JB200_INV_LOG_TEN   .434294482
#define JB200_WORD_INVALID  (-1)      /* reference: 65535 (unsigned short WORD_ID) */
#define JB200_LOG_UNDEF     (JB200_LOG_ZERO - 1.0f)

/* -gprune methods (libjulius/include/julius/jconf.h GPRUNE_SEL_*) */
enum { JB200_GPRUNE_NONE = 0, JB200_GPRUNE_SAFE = 1, JB200_GPRUNE_HEU = 2, JB200_GPRUNE_BEAM = 3 };
/* -iwcd1 methods (libsent/include/sent/htk_hmm.h IWCD_*) */
enum { JB200_IWCD_AVG = 0, JB200_IWCD_MAX = 1, JB200_IWCD_NBEST = 2 };
/* outstyle (wchmm.h:100-106) */
enum { JB200_AS_STATE = 0, JB200_AS_LSET = 1, JB200_AS_RSET = 2, JB200_AS_LRSET = 3 };
/* bigram access mode (libsent/src/ngram/ngram_access.c:288-466) */
enum { JB200_BI_NORMAL = 0, JB200_BI_ADDITIONAL_OLDBIN = 1, JB200_BI_ADDITIONAL = 2, JB200_BI_COMPUTE = 3 };

/* ---- GMM acoustic model ------------------------------------------------------------ */
typedef struct {
  int32_t n_states;          /* S: HTK_HMM_INFO.totalstatenum, index = HTK_HMM_State.id */
  int32_t dim;               /* D: veclen (single stream only) */
  int32_t n_gauss;           /* G: total mixture slots */
  int32_t max_mix;           /* maxmixturenum */
  int32_t gprune_method;     /* JB200_GPRUNE_* */
  int32_t gprune_num;        /* -tmix */
  int32_t iwcd_method;       /* JB200_IWCD_* */
  int32_t iwcd_nbest;        /* cdmax_num */
  int32_t n_cdsets;          /* C */
  int32_t n_cdset_states;    /* total length of cd_states */
  const int32_t *state_off;  /* [S+1] first mixture slot of each state */
  const float *mean;         /* [G][D] */
  const float *ivar;         /* [G][D] inverse variances (as the reference stores them) */
  const float *gconst;       /* [G] */
  const float *lnweight;     /* [G] ln mixture weight (bweight) */
  const uint8_t *valid;      /* [G] 0 where the reference has a NULL density */
  const int32_t *cd_off;     /* [C+1] */
  const int32_t *cd_states;  /* [n_cdset_states] state ids, list order of CD_State_Set.s[] */
} jb200_gmm_desc;

/* ---- DNN acoustic model -------------------------------------------------------------- */
#define JB200_DNN_MAX_LAYERS 16
typedef struct {
  int32_t n_layers;          /* hidden layers + output layer */
  int32_t in_dim;            /* inputnodenum (already spliced) */
  int32_t out_dim;           /* outputnodenum == n_states */
  int32_t layer_in[JB200_DNN_MAX_LAYERS];
  int32_t layer_out[JB200_DNN_MAX_LAYERS];
  const float *w[JB200_DNN_MAX_LAYERS];   /* [out][in] row-major (calc_dnn.c:225-336) */
  const float *b[JB200_DNN_MAX_LAYERS];   /* [out] */
  const float *state_prior;               /* [out_dim], already log10(prior*factor) if log10nize */
} jb200_dnn_desc;

/* ---- lexicon tree + LM + search parameters ---------------------------------------- */
typedef struct {
  int32_t n_nodes;           /* wchmm->n */
  int32_t n_arcs;            /* total A_CELL2 arcs (excluding self/next) */
  int32_t n_words;           /* winfo->num */
  int32_t n_start;           /* startnum */
  int32_t n_iso;             /* isolatenum */
  int32_t n_shared;          /* startnum - isolatenum */
  int32_t n_fscore;          /* fsnum */
  int32_t n_scword;          /* scnum */
  int32_t n_rset;            /* distinct (hmm,state_loc,style) context classes */
  int32_t n_ctx;             /* distinct left-context centre phones (+1 column for "no word") */
  int32_t head_silwid, tail_silwid;
  int32_t multipath;         /* hmminfo->multipath */
  int32_t beam_width;        /* r->trellis_beam_width */
  int32_t lm_nvocab;         /* ngram->max_word_num */
  int32_t lm_nbigram;        /* d[1].totalnum */
  int32_t lm_mode;           /* JB200_BI_* */
  int32_t lm_unk_id;
  float lm_unk_num_log;
  float lm_weight, lm_penalty, lm_penalty_trans;
  float score_pruning_width; /* <0: disabled (default) */
  /* per node */
  const float *self_a;       /* [n] */
  const float *next_a;       /* [n] */
  const int32_t *arc_off;    /* [n+1] */
  const int32_t *arc_to;     /* [n_arcs] */
  const float *arc_a;        /* [n_arcs] */
  const int32_t *stend;      /* [n] word id or -1 */
  const int32_t *scid;       /* [n] */
  const uint8_t *outstyle;   /* [n] JB200_AS_* ; 255 = non-emitting (multipath) */
  const int32_t *out_ref;    /* [n] AS_STATE: state id; AS_LSET: cdset id; AS_RSET/LRSET: rset class */
  /* context classes: ref >= 0 state id, ref < 0 -> cdset id = -ref-1 */
  const int32_t *rset_ctx;   /* [n_rset][n_ctx+1]; column n_ctx = last word invalid */
  const int32_t *word_ctx;   /* [n_words] context column of each word's last phone */
  /* roots, in the order the reference visits them (stid = startnum-1 .. 0) */
  const int32_t *iso_node;   /* [n_iso] */
  const int32_t *iso_word;   /* [n_iso] scword[scid[node]] */
  const int32_t *iso_id;     /* [n_iso] start2isolate value (index into iw cache row) */
  const int32_t *shared_node;/* [n_shared] */
  /* words */
  const float *wordend_a;    /* [n_words] */
  const int32_t *wordend;    /* [n_words] node id */
  const int32_t *wordbegin;  /* [n_words] (multipath) or offset[w][0] */
  const uint8_t *is_transparent; /* [n_words] */
  const int32_t *wton;       /* [n_words] word -> n-gram entry */
  const float *cprob;        /* [n_words] class n-gram in-class prob (0 for word n-gram) */
  /* factoring */
  const float *fscore;       /* [n_fscore] (index 0 unused) */
  const int32_t *scword;     /* [n_scword] (index 0 unused) */
  /* LM */
  const float *uni_prob;     /* [lm_nvocab] d[0].prob */
  const float *uni_bow;      /* [lm_nvocab] d[0].bo_wt (or bo_wt_1) */
  const int32_t *bi_bgn;     /* [lm_nvocab] -1 = no bigram */
  const int32_t *bi_num;     /* [lm_nvocab] */
  const int32_t *bi_wid;     /* [lm_nbigram] nnid2wid */
  const float *bi_prob;      /* [lm_nbigram] d[1].prob (or p_2) */
  /* ---- grammar (DFA) mode, category tree (beam.c:1669-1760, :2404-2455, :435-458).  lm_type = JB200_LM_DFA:
   * every root is listed in iso_* (n_shared = 0, no factoring: scid is all zero), the bigram arrays are empty, and
   * a cross-word transition from word w into root i is allowed iff cp_allowed[w * n_iso + iso_id[i]] (the category
   * pair constraint dfa_cp(category(w), category(start2wid))); its language score is penalty1 + cprob[w]. */
  int32_t lm_type;           /* JB200_LM_NGRAM / JB200_LM_DFA */
  int32_t n_init;            /* sentence-initial words (dfa_cp_begin), in the order init_nodescore creates their tokens */
  float penalty1;            /* -penalty1: word insertion penalty of pass 1 */
  int32_t reserved_;
  const int32_t *init_word;  /* [n_init] */
  const int32_t *init_node;  /* [n_init] offset[w][0], or wordbegin[w] on a multipath tree */
  const float *init_lscore;  /* [n_init] penalty1 + cprob[w] */
  const uint8_t *cp_allowed; /* [n_words][n_iso] */
} jb200_tree_desc;
enum { JB200_LM_NGRAM = 0, JB200_LM_DFA = 1 };

/* ======================================================================================
 * "JB2M" blob container: a flat list of named little-endian arrays.
 *   header : char magic[4]="JB2M"; int32 version=1; int32 n_entries; int32 pad
 *   entry  : char name[48]; int32 dtype (0=f32,1=i32,2=u8); int32 pad; int64 count; data padded to 16 B
 * Scalars are stored as 1-element arrays.  Header-only so the plugin, the
 * product library and the oracle share one implementation.
 * ==================================================================================== */
enum { JB200_F32 = 0, JB200_I32 = 1, JB200_U8 = 2 };

typedef struct {
  char name[48];
  int32_t dtype;
  int64_t count;
  void *data;
} jb200_blob_entry;

typedef struct {
  int32_t n;
  int32_t cap;
  int32_t failed;            /* 1 once an add ran out of memory: entries are missing */
  jb200_blob_entry *e;
} jb200_blob;

static inline size_t jb200_dtype_size(int dtype) { return dtype == JB200_U8 ? 1 : 4; }

static inline void jb200_blob_init(jb200_blob *b) { b->n = 0; b->cap = 0; b->failed = 0; b->e = NULL; }

static inline void jb200_blob_free(jb200_blob *b) {
  int i;
  for (i = 0; i < b->n; i++) free(b->e[i].data);
  free(b->e);
  jb200_blob_init(b);
}

/* Copies the data; with count 0 nothing is read, so data may be NULL.  When an allocation fails the entry is not added
 * and b->failed is set, so that a writer of many entries checks once, after the last. */
static inline void jb200_blob_add(jb200_blob *b, const char *name, int dtype, int64_t count, const void *data) {
  jb200_blob_entry *x;
  size_t nbytes = (size_t)count * jb200_dtype_size(dtype), len = strlen(name);
  void *copy;
  if (b->n == b->cap) {
    int32_t cap = b->cap ? b->cap * 2 : 64;
    jb200_blob_entry *e = (jb200_blob_entry *)realloc(b->e, sizeof(jb200_blob_entry) * cap);
    if (e == NULL) { b->failed = 1; return; }
    b->e = e; b->cap = cap;
  }
  if ((copy = malloc(nbytes ? nbytes : 1)) == NULL) { b->failed = 1; return; }
  if (nbytes) memcpy(copy, data, nbytes);
  x = &b->e[b->n++];
  /* at most 47 characters, zero-padded: the name field always ends in '\0' */
  if (len > sizeof(x->name) - 1) len = sizeof(x->name) - 1;
  memset(x->name, 0, sizeof(x->name));
  memcpy(x->name, name, len);
  x->dtype = dtype; x->count = count;
  x->data = copy;
}
static inline void jb200_blob_add_i(jb200_blob *b, const char *name, int32_t v) { jb200_blob_add(b, name, JB200_I32, 1, &v); }
static inline void jb200_blob_add_f(jb200_blob *b, const char *name, float v) { jb200_blob_add(b, name, JB200_F32, 1, &v); }

static inline const jb200_blob_entry *jb200_blob_find(const jb200_blob *b, const char *name) {
  int i;
  for (i = 0; i < b->n; i++) if (strcmp(b->e[i].name, name) == 0) return &b->e[i];
  return NULL;
}

/* 0, or -1 when the file cannot be opened, a write comes up short (a full disk) or closing it fails */
static inline int jb200_blob_save(const jb200_blob *b, const char *path) {
  FILE *fp = fopen(path, "wb");
  int32_t hdr[3]; int i, ok;
  static const char zero[16] = {0};
  if (!fp) return -1;
  hdr[0] = 1; hdr[1] = b->n; hdr[2] = 0;
  ok = fwrite("JB2M", 1, 4, fp) == 4 && fwrite(hdr, 4, 3, fp) == 3;
  for (i = 0; i < b->n && ok; i++) {
    const jb200_blob_entry *x = &b->e[i];
    size_t nbytes = (size_t)x->count * jb200_dtype_size(x->dtype), pad = (16 - nbytes % 16) % 16;
    int32_t dt[2]; dt[0] = x->dtype; dt[1] = 0;
    ok = fwrite(x->name, 1, 48, fp) == 48 && fwrite(dt, 4, 2, fp) == 2 && fwrite(&x->count, 8, 1, fp) == 1 &&
         fwrite(x->data, 1, nbytes, fp) == nbytes && fwrite(zero, 1, pad, fp) == pad;
  }
  if (fclose(fp) != 0) ok = 0;
  return ok ? 0 : -1;
}

/* Reads a blob file.  The file is not trusted: dtype must be one of the three known types, every count must fit in
 * what is left of the file, allocations are checked.  On any error the blob is left empty and a negative code is
 * returned (-1 cannot open, -2 not a JB2M v1 file, -3 truncated or inconsistent, -4 out of memory). */
static inline int jb200_blob_load(jb200_blob *b, const char *path) {
  FILE *fp = fopen(path, "rb");
  char magic[4]; int32_t hdr[3]; int i, rc = 0;
  long fsize, pos;
  jb200_blob_init(b);
  if (!fp) return -1;
  if (fseek(fp, 0, SEEK_END) != 0 || (fsize = ftell(fp)) < 0 || fseek(fp, 0, SEEK_SET) != 0) { fclose(fp); return -3; }
  if (fread(magic, 1, 4, fp) != 4 || memcmp(magic, "JB2M", 4) != 0) { fclose(fp); return -2; }
  if (fread(hdr, 4, 3, fp) != 3 || hdr[0] != 1) { fclose(fp); return -2; }
  if (hdr[1] < 0 || (long)hdr[1] > (fsize - 16) / 64) { fclose(fp); return -3; }       /* an entry header is 64 bytes */
  b->e = (jb200_blob_entry *)calloc((size_t)(hdr[1] > 0 ? hdr[1] : 1), sizeof(jb200_blob_entry));
  if (!b->e) { fclose(fp); return -4; }
  b->cap = hdr[1];
  for (i = 0; i < hdr[1] && rc == 0; i++) {
    jb200_blob_entry *x = &b->e[i];
    int32_t dt[2]; size_t nbytes;
    if (fread(x->name, 1, 48, fp) != 48 || fread(dt, 4, 2, fp) != 2 || fread(&x->count, 8, 1, fp) != 1) { rc = -3; break; }
    x->name[47] = '\0';
    x->dtype = dt[0];
    pos = ftell(fp);
    if (x->dtype != JB200_F32 && x->dtype != JB200_I32 && x->dtype != JB200_U8) { rc = -3; break; }
    if (pos < 0 || x->count < 0 || x->count > (int64_t)(fsize - pos) / (int64_t)jb200_dtype_size(x->dtype)) { rc = -3; break; }
    nbytes = (size_t)x->count * jb200_dtype_size(x->dtype);
    x->data = malloc(nbytes ? nbytes : 1);
    if (!x->data) { rc = -4; break; }
    b->n = i + 1;                                   /* x->data is owned by the blob from here on */
    if (nbytes && fread(x->data, 1, nbytes, fp) != nbytes) { rc = -3; break; }
    if (nbytes % 16) fseek(fp, (long)(16 - nbytes % 16), SEEK_CUR);
  }
  fclose(fp);
  if (rc != 0) jb200_blob_free(b);
  return rc;
}

/* 1 when the entry exists with the given type and at least `need` elements */
static inline int jb200_blob_has(const jb200_blob *b, const char *name, int dtype, int64_t need) {
  const jb200_blob_entry *x = jb200_blob_find(b, name);
  return x != NULL && x->dtype == dtype && need >= 0 && x->count >= need;
}

/* typed getters: return NULL / default when missing */
static inline const void *jb200_blob_ptr(const jb200_blob *b, const char *name, int64_t *count) {
  const jb200_blob_entry *x = jb200_blob_find(b, name);
  if (count) *count = x ? x->count : 0;
  return x ? x->data : NULL;
}
static inline int32_t jb200_blob_get_i(const jb200_blob *b, const char *name, int32_t dflt) {
  const jb200_blob_entry *x = jb200_blob_find(b, name);
  return (x && x->dtype == JB200_I32 && x->count >= 1) ? ((int32_t *)x->data)[0] : dflt;
}
static inline float jb200_blob_get_f(const jb200_blob *b, const char *name, float dflt) {
  const jb200_blob_entry *x = jb200_blob_find(b, name);
  return (x && x->dtype == JB200_F32 && x->count >= 1) ? ((float *)x->data)[0] : dflt;
}

/* Fill descriptors from a loaded blob (pointers alias the blob's storage).
 * Return 0 on success, -1 if the section is absent or an array is shorter than its declared dimensions. */

/* Only the state / cd-set layout, for a model without Gaussians (DNN-HMM): dim, the mixture counts and every Gaussian
 * array stay 0 / NULL.  This is what the beam decoder reads of its scorer. */
static inline int jb200_cd_gmm_from_blob(const jb200_blob *b, jb200_gmm_desc *g) {
  memset(g, 0, sizeof(*g));
  g->n_states = jb200_blob_get_i(b, "gmm.n_states", 0);
  g->iwcd_method = jb200_blob_get_i(b, "am.iwcd_method", JB200_IWCD_NBEST);
  g->iwcd_nbest = jb200_blob_get_i(b, "am.iwcd_nbest", 3);
  g->n_cdsets = jb200_blob_get_i(b, "am.n_cdsets", 0);
  g->n_cdset_states = jb200_blob_get_i(b, "am.n_cdset_states", 0);
  g->cd_off = (const int32_t *)jb200_blob_ptr(b, "am.cd_off", NULL);
  g->cd_states = (const int32_t *)jb200_blob_ptr(b, "am.cd_states", NULL);
  if (g->n_states < 0 || g->n_cdsets < 0 || g->n_cdset_states < 0) return -1;
  if (g->n_cdsets > 0 && (!jb200_blob_has(b, "am.cd_off", JB200_I32, (int64_t)g->n_cdsets + 1) ||
                          !jb200_blob_has(b, "am.cd_states", JB200_I32, g->n_cdset_states))) return -1;
  return 0;
}

static inline int jb200_gmm_from_blob(const jb200_blob *b, jb200_gmm_desc *g) {
  if (jb200_cd_gmm_from_blob(b, g) != 0 || !jb200_blob_find(b, "gmm.mean")) return -1;
  g->dim = jb200_blob_get_i(b, "gmm.dim", 0);
  g->n_gauss = jb200_blob_get_i(b, "gmm.n_gauss", 0);
  g->max_mix = jb200_blob_get_i(b, "gmm.max_mix", 0);
  g->gprune_method = jb200_blob_get_i(b, "gmm.gprune_method", 0);
  g->gprune_num = jb200_blob_get_i(b, "gmm.gprune_num", 0);
  g->state_off = (const int32_t *)jb200_blob_ptr(b, "gmm.state_off", NULL);
  g->mean = (const float *)jb200_blob_ptr(b, "gmm.mean", NULL);
  g->ivar = (const float *)jb200_blob_ptr(b, "gmm.ivar", NULL);
  g->gconst = (const float *)jb200_blob_ptr(b, "gmm.gconst", NULL);
  g->lnweight = (const float *)jb200_blob_ptr(b, "gmm.lnweight", NULL);
  g->valid = (const uint8_t *)jb200_blob_ptr(b, "gmm.valid", NULL);
  if (g->dim < 1 || g->n_gauss < 0) return -1;
  if (!jb200_blob_has(b, "gmm.state_off", JB200_I32, (int64_t)g->n_states + 1) ||
      !jb200_blob_has(b, "gmm.mean", JB200_F32, (int64_t)g->n_gauss * g->dim) ||
      !jb200_blob_has(b, "gmm.ivar", JB200_F32, (int64_t)g->n_gauss * g->dim) ||
      !jb200_blob_has(b, "gmm.gconst", JB200_F32, g->n_gauss) || !jb200_blob_has(b, "gmm.lnweight", JB200_F32, g->n_gauss) ||
      !jb200_blob_has(b, "gmm.valid", JB200_U8, g->n_gauss)) return -1;
  return 0;
}

static inline int jb200_dnn_from_blob(const jb200_blob *b, jb200_dnn_desc *d) {
  int i; char nm[48];
  memset(d, 0, sizeof(*d));
  if (!jb200_blob_find(b, "dnn.n_layers")) return -1;
  d->n_layers = jb200_blob_get_i(b, "dnn.n_layers", 0);
  d->in_dim = jb200_blob_get_i(b, "dnn.in_dim", 0);
  d->out_dim = jb200_blob_get_i(b, "dnn.out_dim", 0);
  if (d->n_layers < 1 || d->n_layers > JB200_DNN_MAX_LAYERS || d->in_dim < 1 || d->out_dim < 1) return -1;   /* no silent truncation */
  for (i = 0; i < d->n_layers; i++) {
    snprintf(nm, sizeof(nm), "dnn.l%d.in", i);  d->layer_in[i] = jb200_blob_get_i(b, nm, 0);
    snprintf(nm, sizeof(nm), "dnn.l%d.out", i); d->layer_out[i] = jb200_blob_get_i(b, nm, 0);
    snprintf(nm, sizeof(nm), "dnn.l%d.w", i);   d->w[i] = (const float *)jb200_blob_ptr(b, nm, NULL);
    snprintf(nm, sizeof(nm), "dnn.l%d.b", i);   d->b[i] = (const float *)jb200_blob_ptr(b, nm, NULL);
    if (d->layer_in[i] < 1 || d->layer_out[i] < 1 || !jb200_blob_has(b, nm, JB200_F32, d->layer_out[i])) return -1;
    snprintf(nm, sizeof(nm), "dnn.l%d.w", i);
    if (!jb200_blob_has(b, nm, JB200_F32, (int64_t)d->layer_in[i] * d->layer_out[i])) return -1;
  }
  d->state_prior = (const float *)jb200_blob_ptr(b, "dnn.state_prior", NULL);
  if (!jb200_blob_has(b, "dnn.state_prior", JB200_F32, d->out_dim)) return -1;
  return 0;
}

static inline int jb200_tree_from_blob(const jb200_blob *b, jb200_tree_desc *t) {
  memset(t, 0, sizeof(*t));
  if (!jb200_blob_find(b, "tree.self_a")) return -1;
#define JB200_GI(f) t->f = jb200_blob_get_i(b, "tree." #f, 0)
#define JB200_GF(f) t->f = jb200_blob_get_f(b, "tree." #f, 0.0f)
#define JB200_GP(f, T) t->f = (const T *)jb200_blob_ptr(b, "tree." #f, NULL)
  JB200_GI(n_nodes); JB200_GI(n_arcs); JB200_GI(n_words); JB200_GI(n_start); JB200_GI(n_iso);
  JB200_GI(n_shared); JB200_GI(n_fscore); JB200_GI(n_scword); JB200_GI(n_rset); JB200_GI(n_ctx);
  JB200_GI(head_silwid); JB200_GI(tail_silwid); JB200_GI(multipath); JB200_GI(beam_width);
  JB200_GI(lm_nvocab); JB200_GI(lm_nbigram); JB200_GI(lm_mode); JB200_GI(lm_unk_id);
  JB200_GF(lm_unk_num_log); JB200_GF(lm_weight); JB200_GF(lm_penalty); JB200_GF(lm_penalty_trans);
  t->score_pruning_width = jb200_blob_get_f(b, "tree.score_pruning_width", -1.0f);
  JB200_GP(self_a, float); JB200_GP(next_a, float); JB200_GP(arc_off, int32_t); JB200_GP(arc_to, int32_t);
  JB200_GP(arc_a, float); JB200_GP(stend, int32_t); JB200_GP(scid, int32_t); JB200_GP(outstyle, uint8_t);
  JB200_GP(out_ref, int32_t); JB200_GP(rset_ctx, int32_t); JB200_GP(word_ctx, int32_t);
  JB200_GP(iso_node, int32_t); JB200_GP(iso_word, int32_t); JB200_GP(iso_id, int32_t); JB200_GP(shared_node, int32_t);
  JB200_GP(wordend_a, float); JB200_GP(wordend, int32_t); JB200_GP(wordbegin, int32_t);
  JB200_GP(is_transparent, uint8_t); JB200_GP(wton, int32_t); JB200_GP(cprob, float);
  JB200_GP(fscore, float); JB200_GP(scword, int32_t);
  JB200_GP(uni_prob, float); JB200_GP(uni_bow, float); JB200_GP(bi_bgn, int32_t); JB200_GP(bi_num, int32_t);
  JB200_GP(bi_wid, int32_t); JB200_GP(bi_prob, float);
  JB200_GI(lm_type); JB200_GI(n_init); JB200_GF(penalty1);
  JB200_GP(init_word, int32_t); JB200_GP(init_node, int32_t); JB200_GP(init_lscore, float); JB200_GP(cp_allowed, uint8_t);
#undef JB200_GI
#undef JB200_GF
#undef JB200_GP
  /* every array must be as long as the declared dimensions say (the decoder indexes them without further checks) */
  if (t->n_nodes < 1 || t->n_arcs < 0 || t->n_words < 1 || t->n_iso < 0 || t->n_shared < 0 || t->n_fscore < 0 ||
      t->n_scword < 0 || t->n_rset < 0 || t->n_ctx < 0 || t->lm_nvocab < 0 || t->lm_nbigram < 0 || t->n_init < 0) return -1;
#define JB200_NEED(f, dt, cnt) if (!jb200_blob_has(b, "tree." #f, dt, (int64_t)(cnt))) return -1
  JB200_NEED(self_a, JB200_F32, t->n_nodes); JB200_NEED(next_a, JB200_F32, t->n_nodes);
  JB200_NEED(arc_off, JB200_I32, (int64_t)t->n_nodes + 1); JB200_NEED(arc_to, JB200_I32, t->n_arcs); JB200_NEED(arc_a, JB200_F32, t->n_arcs);
  JB200_NEED(stend, JB200_I32, t->n_nodes); JB200_NEED(scid, JB200_I32, t->n_nodes);
  JB200_NEED(outstyle, JB200_U8, t->n_nodes); JB200_NEED(out_ref, JB200_I32, t->n_nodes);
  JB200_NEED(rset_ctx, JB200_I32, (int64_t)t->n_rset * (t->n_ctx + 1)); JB200_NEED(word_ctx, JB200_I32, t->n_words);
  JB200_NEED(iso_node, JB200_I32, t->n_iso); JB200_NEED(iso_word, JB200_I32, t->n_iso); JB200_NEED(iso_id, JB200_I32, t->n_iso);
  JB200_NEED(shared_node, JB200_I32, t->n_shared);
  JB200_NEED(wordend_a, JB200_F32, t->n_words); JB200_NEED(wordend, JB200_I32, t->n_words); JB200_NEED(wordbegin, JB200_I32, t->n_words);
  JB200_NEED(is_transparent, JB200_U8, t->n_words); JB200_NEED(wton, JB200_I32, t->n_words); JB200_NEED(cprob, JB200_F32, t->n_words);
  JB200_NEED(fscore, JB200_F32, t->n_fscore); JB200_NEED(scword, JB200_I32, t->n_scword);
  if (t->lm_type == JB200_LM_NGRAM) {
    JB200_NEED(uni_prob, JB200_F32, t->lm_nvocab); JB200_NEED(uni_bow, JB200_F32, t->lm_nvocab);
    JB200_NEED(bi_bgn, JB200_I32, t->lm_nvocab); JB200_NEED(bi_num, JB200_I32, t->lm_nvocab);
    JB200_NEED(bi_wid, JB200_I32, t->lm_nbigram); JB200_NEED(bi_prob, JB200_F32, t->lm_nbigram);
  } else {
    JB200_NEED(init_word, JB200_I32, t->n_init); JB200_NEED(init_node, JB200_I32, t->n_init); JB200_NEED(init_lscore, JB200_F32, t->n_init);
    JB200_NEED(cp_allowed, JB200_U8, (int64_t)t->n_words * t->n_iso);
  }
#undef JB200_NEED
  if (t->lm_type == JB200_LM_NGRAM &&
      (t->head_silwid < 0 || t->head_silwid >= t->n_words || t->tail_silwid < 0 || t->tail_silwid >= t->n_words)) return -1;
  return 0;
}

#ifdef __cplusplus
}
#endif
#endif /* JB200_MODEL_H */
