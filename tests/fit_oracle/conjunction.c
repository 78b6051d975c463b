/*
 * conjunction.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of the TCA and the per-object covariances of K11, astroz_cuda_conjunction
 * (astroz_b200/csrc/az_conjunction.cuh), on the CPU oracle's SGP4 / SDP4.  It includes covariance.c (and through it
 * fit_oracle_obs.c's variable map and model), so the sets are the ones the fit restatement builds.  From the
 * definition:
 *   states     each row's nominal state at tsince = ((jd + fr) - epoch) * 1440 + dt;
 *   TCA        g = dr . dv sampled at 241 points of [-w, w]; every - to + change is bisected to 1e-10 min and the root of
 *              least |dr| kept (status 0); no change: the window end of smaller |dr| (status 3);
 *   Sigma      covref_propagate (covariance.c) of each row at jd, fr + dt / 1440;
 *   status     1 when a set cannot be built, 2 when a deep-space cell fails; zeros then.
 * The plane and Pc are formed from these outputs by the caller.  Candidates are dealt to pthreads.
 */
#include "covariance.c"

typedef struct {
    const double *el, *cov;
    const uint8_t *model;
    uint32_t n;
    int grav, frame;
    const uint32_t *pr, *se;
    const double *jd, *fr, *win;
    uint32_t m;
    double *dt, *states, *sig;
    uint8_t *status;
    uint32_t next;
    pthread_mutex_t mu;
} conj_job_t;

static int at(const model_t *M, double ts, double f[6]) {
    if (!M->deep) {
        azo_sgp4_propagate(&M->ne, ts, f, f + 3);
        return 0;
    }
    return azo_sdp4_propagate(&M->ds, ts, f, f + 3) == 0 ? 0 : -1;
}

typedef struct { const model_t *p, *s; double tp, ts; int fail; } pair_t;

static void rel(pair_t *P, double t, double *g, double *d2) {
    double fp[6], fs[6];
    if (at(P->p, P->tp + t, fp) != 0 || at(P->s, P->ts + t, fs) != 0) P->fail = 1;
    *g = *d2 = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double dr = fs[c] - fp[c], dv = fs[3 + c] - fp[3 + c];
        *g += dr * dv;
        *d2 += dr * dr;
    }
}

static void one_candidate(conj_job_t *J, uint32_t i) {
    const uint32_t row[2] = {J->pr[i], J->se[i]};
    model_t M[2];
    double tsz[2];
    const double jdFull = J->jd[i] + J->fr[i], w = J->win[i];
    for (int o = 0; o < 2; ++o) {
        const int deep = J->model ? J->model[row[o]] : 0;
        double el[8], x[NV];
        for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * J->n + row[o]];
        vars_of(el, deep, x);
        if (build(x, el[0], J->grav, deep, &M[o]) != 0) {
            J->status[i] = 1;
            return;
        }
        tsz[o] = (jdFull - el[0]) * 1440.0;
    }
    pair_t P = {&M[0], &M[1], tsz[0], tsz[1], 0};
    enum { N = 241 };
    double g[N], d2[N], t[N];
    for (int k = 0; k < N; ++k) {
        t[k] = -w + 2.0 * w * k / (N - 1);
        rel(&P, t[k], &g[k], &d2[k]);
    }
    double tca = 0.0, best = -1.0;
    uint8_t st = 0;
    for (int k = 0; k + 1 < N; ++k) {
        if (!(g[k] < 0.0 && g[k + 1] >= 0.0)) continue;
        double a = t[k], b = t[k + 1];
        while (b - a > 1e-10) {
            const double c = 0.5 * (a + b);
            double gc, dc;
            rel(&P, c, &gc, &dc);
            if (gc < 0.0) a = c;
            else b = c;
        }
        double gm, dm;
        const double r = 0.5 * (a + b);
        rel(&P, r, &gm, &dm);
        if (best < 0.0 || dm < best) {
            best = dm;
            tca = r;
        }
    }
    if (best < 0.0) {
        tca = d2[N - 1] < d2[0] ? w : -w;
        st = 3;
    }
    if (P.fail) {
        J->status[i] = 2;
        return;
    }
    for (int o = 0; o < 2; ++o) {
        double f[6];
        if (at(&M[o], tsz[o] + tca, f) != 0) {
            J->status[i] = 2;
            return;
        }
        memcpy(J->states + 12 * (size_t)i + 6 * o, f, sizeof f);
        /* Sigma at the TCA through covariance.c, one single-query satellite */
        double el[8];
        for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * J->n + row[o]];
        const uint8_t md = J->model ? J->model[row[o]] : 0;
        const uint32_t off[2] = {0, 1};
        const double qjd = J->jd[i], qfr = J->fr[i] + tca / 1440.0;
        uint8_t cst = 0;
        cov_job_t C = {el, J->cov + 28 * (size_t)row[o], &md, 1, J->grav, J->frame, off, &qjd, &qfr, NULL,
                       J->sig + 42 * (size_t)i + 21 * o, NULL, &cst, 0, PTHREAD_MUTEX_INITIALIZER};
        one_sat(&C, 0);
        if (cst != 0) {
            J->status[i] = cst;
            return;
        }
    }
    J->dt[i] = tca;
    J->status[i] = st;
}

static void *conj_worker(void *arg) {
    conj_job_t *J = (conj_job_t *)arg;
    for (;;) {
        pthread_mutex_lock(&J->mu);
        const uint32_t i = J->next++;
        pthread_mutex_unlock(&J->mu);
        if (i >= J->m) return NULL;
        one_candidate(J, i);
    }
}

int conjref_assess(const double *elements, uint32_t n, int grav, const double *covariance, const uint8_t *model,
                   const uint32_t *primary, const uint32_t *secondary, const double *jd, const double *fr,
                   const double *window, uint32_t m, int frame, int threads, double *dt, double *states,
                   double *state_covariance, uint8_t *status) {
    conj_job_t J = {elements, covariance, model, n, grav, frame, primary, secondary, jd, fr, window, m, dt, states,
                    state_covariance, status, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256];
    for (int k = 1; k < threads; ++k) pthread_create(&th[k], NULL, conj_worker, &J);
    conj_worker(&J);
    for (int k = 1; k < threads; ++k) pthread_join(th[k], NULL);
    return 0;
}
