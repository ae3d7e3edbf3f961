/* jb200_host.h -- what the attach plugin (jb200_attach.c) and the beam shim (jb200_beam_shim.c) share: opening the
 * GPU scorer of a flattened model, and gathering the host's feature rows into one matrix. */
#ifndef JB200_HOST_H
#define JB200_HOST_H
#include <julius/juliuslib.h>
#include "jb200_model.h"
#include "jb200_dl.h"

typedef struct {
  jb200_gmm_desc gd;     /* a DNN model's has only the state / cd-set layout, and dim = the net's input width */
  jb200_dnn_desc dd;
  jb200_gmm *gmm;        /* a DNN model's is the Gaussian-free layout scorer, or NULL when it was not asked for */
  jb200_dnn *dnn;        /* NULL for a GMM model */
} jb200_scorer;

static void jb200_scorer_close(jb200_scorer *sc, const jb200_api *api) {
  if (sc->dnn) { api->dnn_destroy(sc->dnn); sc->dnn = NULL; }
  if (sc->gmm) { api->gmm_destroy(sc->gmm); sc->gmm = NULL; }
}

/* Opens the scorer of the model in b: a GMM scorer for a GMM model; a DNN scorer for a DNN model, plus the layout
 * scorer when dnn_layout is set (the beam decoder takes one).  JB200_GMM_MODE=fast selects the fast GMM arithmetic.
 * Returns 0; 1 when b holds no acoustic model; else the failed create's error code (api->last_error() says why).
 * After a failure nothing is left open. */
static int jb200_scorer_open(jb200_scorer *sc, const jb200_api *api, const jb200_blob *b, int dnn_layout) {
  const char *mode = getenv("JB200_GMM_MODE");
  int rc;
  memset(sc, 0, sizeof(*sc));
  if (jb200_dnn_from_blob(b, &sc->dd) == 0) {
    if (jb200_cd_gmm_from_blob(b, &sc->gd) != 0) return 1;
    sc->gd.dim = sc->dd.in_dim;
    rc = api->dnn_create(&sc->dd, 0, &sc->dnn);
    if (rc != 0 || !dnn_layout) return rc;
  } else if (jb200_gmm_from_blob(b, &sc->gd) != 0) return 1;
  rc = api->gmm_create(&sc->gd, 0, (mode && strcmp(mode, "fast") == 0) ? JB200_GMM_FAST : JB200_GMM_EXACT, &sc->gmm);
  if (rc != 0) jb200_scorer_close(sc, api);
  return rc;
}

/* a growable float array owned by the caller */
typedef struct { float *x; size_t cap; } jb200_rows;

/* room for n floats, keeping what m holds; 0, or -1 when out of memory (m is left as it was) */
static int jb200_rows_reserve(jb200_rows *m, size_t n) {
  float *x;
  if (n <= m->cap) return 0;
  if (n < 2 * m->cap) n = 2 * m->cap;
  x = (float *)realloc(m->x, sizeof(float) * n);
  if (x == NULL) return -1;
  m->x = x; m->cap = n;
  return 0;
}

/* frames [t0, t1) of param, D components each, into m as one row-major matrix (the host allocates each row on its
 * own); 0, or -1 when out of memory */
static int jb200_gather(jb200_rows *m, const HTK_Param *param, int t0, int t1, int D) {
  int t;
  if (jb200_rows_reserve(m, (size_t)(t1 - t0) * D) != 0) return -1;
  for (t = t0; t < t1; t++) memcpy(m->x + (size_t)(t - t0) * D, param->parvec[t], sizeof(float) * D);
  return 0;
}
#endif
