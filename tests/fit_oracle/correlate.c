/*
 * correlate.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of one K12 pair (astroz_b200/csrc/az_correlate.cuh) on the CPU oracle's SGP4 / SDP4.
 * It includes fit_oracle_obs.c for the variable map, the sets (build, state) and the measurement kinds (measure,
 * weights) and covariance.c for vars_of, so the sets and rows are those of the fit restatement.  Written from the
 * definition, on the stacked form rather than the push-through identity:
 *   rows      per observation z[c] = (observed - h(f0)) w[c] (azimuth / RA wrapped) and G[c][j] = (h(f_j) - h(f0)) w[c]
 *             / (x'_j - x_j); no stepped set when P is all zero, no B* set when P's B* row is zero;
 *   distance  d2 = z^T (I + G P G^T)^-1 z over the k stacked used residuals, by a Cholesky factorisation of the k x k
 *             matrix I + G P G^T.
 */
#include <stdlib.h>

#include "covariance.c"

/* One catalogue row: its P, its nominal and stepped sets (ok = 0 when they cannot be built) */
typedef struct {
    int ok, nv;
    double el[8], P[NV][NV], inv[NV + 1];
    model_t sets[NV + 1];
} ref_row_t;

static void ref_row(ref_row_t *R, const double *elements, uint32_t n, int grav, const double *covariance,
                    const uint8_t *model, uint32_t s) {
    const int deep = model ? model[s] : 0;
    double x[NV];
    memset(R->inv, 0, sizeof R->inv);
    for (int c = 0; c < 8; ++c) R->el[c] = elements[(size_t)c * n + s];
    int zero = 1;
    for (int j = 0, w = 0; j < NV; ++j)
        for (int k = j; k < NV; ++k, ++w) {
            R->P[j][k] = R->P[k][j] = covariance ? covariance[28 * (size_t)s + w] : 0.0;
            if (R->P[j][k] != 0.0) zero = 0;
        }
    R->nv = NV - 1;
    for (int j = 0; j < NV; ++j)
        if (R->P[j][NV - 1] != 0.0) R->nv = NV;
    if (zero) R->nv = 0;
    vars_of(R->el, deep, x);
    R->ok = 0;
    if (build(x, R->el[0], grav, deep, &R->sets[0]) != 0) return;
    for (int j = 0; j < R->nv; ++j) {
        double xs[NV];
        int built = 0;
        memcpy(xs, x, sizeof xs);
        for (int dir = 0; dir < 2 && !built; ++dir) {
            xs[j] = dir == 0 ? x[j] + 1e-8 : x[j] - 1e-8;
            if (build(xs, R->el[0], grav, deep, &R->sets[1 + j]) == 0) {
                R->inv[1 + j] = 1.0 / (xs[j] - x[j]);
                built = 1;
            }
        }
        if (!built) return;
    }
    R->ok = 1;
}

/* Pair (row R, observations [b, e)): z[L][6], G[L][6][7] (row-major per observation), *d2.  Returns 0, or 2 when a
 * cell fails. */
static int ref_pair(const ref_row_t *R, uint32_t b, uint32_t e, const double *jd, const double *fr,
                    const uint8_t *kind, const double *value, const double *sigma, const uint32_t *station,
                    const double *stations, double *z, double *G, double *d2) {
    const double *el = R->el;
    const int nv = R->nv;
    const model_t *sets = R->sets;
    const double(*P)[NV] = R->P;
    const double *inv = R->inv;
    const uint32_t L = e - b;
    job_t J;
    memset(&J, 0, sizeof J);
    J.value = value;
    J.sigma = sigma;
    J.kind = kind;
    /* the stacked used rows */
    double *zs = malloc(sizeof(double) * 6 * L), *gs = malloc(sizeof(double) * 6 * L * NV);
    int k = 0;
    for (uint32_t i = b; i < e; ++i) {
        const int kd = kind[i], wr = wrapped_of(kd);
        const double *v = value + 6 * (size_t)i;
        const double *llh = kd >= 2 ? stations + 3 * (size_t)station[i] : NULL;
        const double jdFull = jd[i] + fr[i];
        double w[6], f0[6], h0[6], sc[6];
        weights(&J, i, w);
        if (state(&sets[0], jd[i], fr[i], el[0], f0) != 0) goto cell;
        measure(kd, f0, jdFull, llh, h0, sc);
        double *zo = z + 6 * (size_t)(i - b), *go = G + 42 * (size_t)(i - b);
        for (int c = 0; c < 6; ++c) {
            zo[c] = w[c] != 0.0 ? (c == wr ? wrap_pi(v[c] - h0[c]) : v[c] - h0[c]) * w[c] : 0.0;
            for (int j = 0; j < NV; ++j) go[c * NV + j] = 0.0;
        }
        for (int j = 0; j < nv; ++j) {
            double f[6], hj[6], scj[6];
            if (state(&sets[1 + j], jd[i], fr[i], el[0], f) != 0) goto cell;
            measure(kd, f, jdFull, llh, hj, scj);
            for (int c = 0; c < 6; ++c)
                go[c * NV + j] = w[c] != 0.0 ? (c == wr ? wrap_pi(hj[c] - h0[c]) : hj[c] - h0[c]) * w[c] * inv[1 + j]
                                             : 0.0;
        }
        for (int c = 0; c < 6; ++c) {
            if (w[c] == 0.0) continue;
            zs[k] = zo[c];
            for (int j = 0; j < NV; ++j) gs[k * NV + j] = go[c * NV + j];
            ++k;
        }
    }
    {
        /* A = I + G P G^T (k x k), A = C C^T, v = C^-1 z, d2 = |v|^2 */
        double *A = malloc(sizeof(double) * k * k), gp[NV];
        for (int a = 0; a < k; ++a) {
            for (int j = 0; j < NV; ++j) {
                gp[j] = 0.0;
                for (int q = 0; q < NV; ++q) gp[j] += gs[a * NV + q] * P[q][j];
            }
            for (int c = 0; c <= a; ++c) {
                double acc = a == c ? 1.0 : 0.0;
                for (int j = 0; j < NV; ++j) acc += gp[j] * gs[c * NV + j];
                A[a * k + c] = acc;
            }
        }
        for (int j = 0; j < k; ++j) {
            double dj = A[j * k + j];
            for (int q = 0; q < j; ++q) dj -= A[j * k + q] * A[j * k + q];
            dj = sqrt(dj);
            A[j * k + j] = dj;
            for (int i = j + 1; i < k; ++i) {
                double a = A[i * k + j];
                for (int q = 0; q < j; ++q) a -= A[i * k + q] * A[j * k + q];
                A[i * k + j] = a / dj;
            }
        }
        double vv = 0.0;
        for (int i = 0; i < k; ++i) {
            double a = zs[i];
            for (int q = 0; q < i; ++q) a -= A[i * k + q] * zs[q];   /* zs overwritten by v */
            zs[i] = a / A[i * k + i];
            vv += zs[i] * zs[i];
        }
        *d2 = vv;
        free(A);
    }
    free(zs);
    free(gs);
    return 0;
cell:
    free(zs);
    free(gs);
    return 2;
}

/* Pair (row s, observations [b, e)): as ref_pair; returns 1 when the row's sets cannot be built. */
int corrref_pair(const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
                 uint32_t s, uint32_t b, uint32_t e, const double *jd, const double *fr, const uint8_t *kind,
                 const double *value, const double *sigma, const uint32_t *station, const double *stations, double *z,
                 double *G, double *d2) {
    ref_row_t *R = malloc(sizeof *R);
    ref_row(R, elements, n, grav, covariance, model, s);
    const int rc = R->ok ? ref_pair(R, b, e, jd, fr, kind, value, sigma, station, stations, z, G, d2) : 1;
    free(R);
    return rc;
}

/* Every (track, row) pair: rows dealt to pthreads, each row's sets built once; d2[t][n], NaN for a row that cannot be
 * built or a pair whose cell fails. */
typedef struct {
    const double *el, *cov;
    const uint8_t *model;
    uint32_t n, t;
    int grav;
    const uint32_t *off;
    const double *jd, *fr, *value, *sigma, *stations;
    const uint8_t *kind;
    const uint32_t *station;
    double *d2;
    uint32_t next;
    pthread_mutex_t m;
} sweep_t;

static void *sweep_worker(void *arg) {
    sweep_t *S = (sweep_t *)arg;
    uint32_t most = 0;
    for (uint32_t j = 0; j < S->t; ++j)
        if (S->off[j + 1] - S->off[j] > most) most = S->off[j + 1] - S->off[j];
    ref_row_t *R = malloc(sizeof *R);
    double *z = malloc(sizeof(double) * 6 * (most + 1)), *G = malloc(sizeof(double) * 42 * (most + 1));
    for (;;) {
        pthread_mutex_lock(&S->m);
        const uint32_t s = S->next++;
        pthread_mutex_unlock(&S->m);
        if (s >= S->n) break;
        ref_row(R, S->el, S->n, S->grav, S->cov, S->model, s);
        for (uint32_t j = 0; j < S->t; ++j) {
            double d = NAN;
            if (R->ok && ref_pair(R, S->off[j], S->off[j + 1], S->jd, S->fr, S->kind, S->value, S->sigma, S->station,
                                  S->stations, z, G, &d) != 0)
                d = NAN;
            S->d2[(size_t)j * S->n + s] = d;
        }
    }
    free(R);
    free(z);
    free(G);
    return NULL;
}

int corrref_sweep(const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
                  const uint32_t *offsets, uint32_t t, const double *jd, const double *fr, const uint8_t *kind,
                  const double *value, const double *sigma, const uint32_t *station, const double *stations,
                  int threads, double *d2) {
    sweep_t S = {elements, covariance, model, n, t, grav, offsets, jd, fr, value, sigma, stations, kind, station, d2,
                 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256];
    for (int k = 1; k < threads; ++k) pthread_create(&th[k], NULL, sweep_worker, &S);
    sweep_worker(&S);
    for (int k = 1; k < threads; ++k) pthread_join(th[k], NULL);
    return 0;
}
