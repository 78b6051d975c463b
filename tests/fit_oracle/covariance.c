/*
 * covariance.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of K10, the state covariance of astroz_cuda_propagate_covariance
 * (astroz_b200/csrc/az_covariance.cuh), on the CPU oracle's SGP4 / SDP4.  It includes fit_oracle_obs.c for the fit
 * restatement's variable map and model (to_tle, build, state: azo_sgp4_* for model 0, azo_sdp4_* for model 1), so the
 * variables and the sets are exactly the ones that restatement fits.  Written from the definition:
 *   nominal    the state of the set x = the variables of the element columns at ((jd + fr) - epoch) * 1440;
 *   Jacobian   J[c][j] = (f_j - f) / (x'_j - x_j), x'_j = x_j + 1e-8, or x_j - 1e-8 when the forward set cannot be built;
 *              the B* column is zero (and not built) when P's B* row is all zero;
 *   frame      0 TEME; 1 RTN of the nominal state, the same 3 x 3 rotation on the position and velocity rows;
 *   Sigma      J P J^T with P the symmetric matrix of the 28 words, its upper triangle row by row;
 *   status     1 when a set cannot be built, 2 when the nominal or a stepped deep-space state fails; all zeros then.
 * Satellites are dealt to pthreads.
 */
#include "fit_oracle_obs.c"

typedef struct {
    const double *el, *cov;
    const uint8_t *model;
    uint32_t n;
    int grav, frame;
    const uint32_t *off;
    const double *jd, *fr;
    double *state, *sig, *jac;
    uint8_t *status;
    uint32_t next;
    pthread_mutex_t m;
} cov_job_t;

static void vars_of(const double *el, int deep, double *x) {
    const double d2r = kPi / 180.0;
    if (!deep) {
        const double w = el[5] * d2r;
        x[0] = el[1]; x[1] = el[2] * cos(w); x[2] = el[2] * sin(w);
        x[3] = el[3] * d2r; x[4] = el[4] * d2r; x[5] = el[6] * d2r + w;
    } else {
        const double node = el[4] * d2r, P = el[5] * d2r + node, ti = tan(0.5 * el[3] * d2r);
        x[0] = el[1]; x[1] = el[2] * cos(P); x[2] = el[2] * sin(P);
        x[3] = ti * cos(node); x[4] = ti * sin(node); x[5] = el[6] * d2r + P;
    }
    x[6] = el[7];
}

static void fail(cov_job_t *J, uint32_t i, uint8_t st) {
    if (J->state) memset(J->state + 6 * (size_t)i, 0, 6 * sizeof(double));
    memset(J->sig + 21 * (size_t)i, 0, 21 * sizeof(double));
    if (J->jac) memset(J->jac + 42 * (size_t)i, 0, 42 * sizeof(double));
    J->status[i] = st;
}

static void one_sat(cov_job_t *J, uint32_t s) {
    const uint32_t n = J->n, b = J->off[s], e = J->off[s + 1];
    const int deep = J->model ? J->model[s] : 0;
    double el[8], P[NV][NV], x[NV], inv[NV + 1] = {0};
    for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * n + s];
    for (int j = 0, w = 0; j < NV; ++j)
        for (int k = j; k < NV; ++k, ++w) P[j][k] = P[k][j] = J->cov[28 * (size_t)s + w];
    int nv = NV - 1;
    for (int j = 0; j < NV; ++j)
        if (P[j][NV - 1] != 0.0) nv = NV;
    vars_of(el, deep, x);
    model_t sets[NV + 1];
    int ok = build(x, el[0], J->grav, deep, &sets[0]) == 0;
    for (int j = 0; j < nv && ok; ++j) {
        double xs[NV];
        int built = 0;
        memcpy(xs, x, sizeof xs);
        for (int dir = 0; dir < 2 && !built; ++dir) {
            xs[j] = dir == 0 ? x[j] + 1e-8 : x[j] - 1e-8;
            if (build(xs, el[0], J->grav, deep, &sets[1 + j]) == 0) {
                inv[1 + j] = 1.0 / (xs[j] - x[j]);
                built = 1;
            }
        }
        ok = built;
    }
    for (uint32_t i = b; i < e; ++i) {
        if (!ok) {
            fail(J, i, 1);
            continue;
        }
        double f0[6], jac[6][NV], rot[3][3];
        memset(jac, 0, sizeof jac);
        int cell = state(&sets[0], J->jd[i], J->fr[i], el[0], f0) == 0;
        for (int j = 0; j < nv; ++j) {
            double f[6];
            if (state(&sets[1 + j], J->jd[i], J->fr[i], el[0], f) != 0) {
                cell = 0;
                continue;
            }
            for (int c = 0; c < 6; ++c) jac[c][j] = (f[c] - f0[c]) * inv[1 + j];
        }
        if (!cell) {
            fail(J, i, 2);
            continue;
        }
        if (J->frame == 1) {   /* rows R, T, N */
            const double r = sqrt(dot3(f0, f0));
            double h[3] = {f0[1] * f0[5] - f0[2] * f0[4], f0[2] * f0[3] - f0[0] * f0[5], f0[0] * f0[4] - f0[1] * f0[3]};
            const double hn = sqrt(dot3(h, h));
            for (int c = 0; c < 3; ++c) rot[0][c] = f0[c] / r, rot[2][c] = h[c] / hn;
            rot[1][0] = rot[2][1] * rot[0][2] - rot[2][2] * rot[0][1];
            rot[1][1] = rot[2][2] * rot[0][0] - rot[2][0] * rot[0][2];
            rot[1][2] = rot[2][0] * rot[0][1] - rot[2][1] * rot[0][0];
            double t[6][NV];
            for (int blk = 0; blk < 6; blk += 3)
                for (int a = 0; a < 3; ++a)
                    for (int j = 0; j < NV; ++j)
                        t[blk + a][j] = rot[a][0] * jac[blk][j] + rot[a][1] * jac[blk + 1][j] + rot[a][2] * jac[blk + 2][j];
            memcpy(jac, t, sizeof jac);
        }
        double S[6][6];
        for (int a = 0; a < 6; ++a)
            for (int c = 0; c < 6; ++c) {
                double acc = 0.0;
                for (int j = 0; j < NV; ++j)
                    for (int k = 0; k < NV; ++k) acc += jac[a][j] * P[j][k] * jac[c][k];
                S[a][c] = acc;
            }
        if (J->state) memcpy(J->state + 6 * (size_t)i, f0, sizeof f0);
        for (int a = 0, w = 0; a < 6; ++a)
            for (int c = a; c < 6; ++c, ++w) J->sig[21 * (size_t)i + w] = S[a][c];
        if (J->jac) memcpy(J->jac + 42 * (size_t)i, jac, sizeof jac);
        J->status[i] = 0;
    }
}

static void *cov_worker(void *arg) {
    cov_job_t *J = (cov_job_t *)arg;
    for (;;) {
        pthread_mutex_lock(&J->m);
        const uint32_t s = J->next++;
        pthread_mutex_unlock(&J->m);
        if (s >= J->n) return NULL;
        one_sat(J, s);
    }
}

/* astroz_cuda_propagate_covariance restated; the argument layout of the C ABI (plus threads) */
int covref_propagate(const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
                     const uint32_t *offsets, const double *jd, const double *fr, int frame, int threads,
                     double *state, double *state_covariance, double *jacobian, uint8_t *status) {
    cov_job_t J = {elements, covariance, model, n, grav, frame, offsets, jd, fr, state, state_covariance, jacobian,
                   status, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256];
    for (int k = 1; k < threads; ++k) pthread_create(&th[k], NULL, cov_worker, &J);
    cov_worker(&J);
    for (int k = 1; k < threads; ++k) pthread_join(th[k], NULL);
    return 0;
}
