/*
 * fit_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of the element fit of K8 (astroz_b200/csrc/az_fit.cuh) on the CPU oracle's SGP4
 * (oracle/astroz_oracle.c): element sets go through azo_sgp4_init and azo_sgp4_propagate, never through the library.
 * The definition it restates:
 *   variables  x = [n rev/day, e cos w, e sin w, i rad, node rad, M + w rad, B*] (B* held when fit_bstar = 0);
 *   elements   e = |(x1, x2)|, w = atan2(x2, x1), M = x5 - w, node / w / M reduced to [0, 360) deg;
 *   time       tsince = ((jd + fr) - epoch) * 1440;
 *   residuals  (pos - model) / pos_sigma, (vel - model) / vel_sigma; cost F = sum of squares;
 *   Jacobian   forward differences, step 1e-8 on every variable, the backward step when the forward set fails init,
 *              divided by the step actually taken;
 *   damping    Marquardt, lambda diag(J^T J), solved by Cholesky on the unit-diagonal scaling; lambda starts at 1e-3,
 *              x 10 on a rejected step (cost not lower, or a trial set that fails init, or a failed factorisation),
 *              / 10 on an accepted one;
 *   stop       converged when a step changes F by at most 1e-10 F, or when F is at the rounding floor
 *              1e-24 sum (|r_obs|^2 / pos_sigma^2 + |v_obs|^2 / vel_sigma^2); else after max_iter steps tried.
 * Sums run over the observations in order (the library sums 32 lane partials in a butterfly: same value to rounding).
 * Built by the tests with oracle/astroz_oracle.c into one shared object; satellites are dealt to pthreads.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include "../../oracle/astroz_oracle.h"

#define NV 7
static const double kPi = 3.14159265358979323846264338327950288;

typedef struct {
    const double *el;
    uint32_t n;
    int grav;
    const uint32_t *off;
    const double *jd, *fr, *pos, *vel;
    double wp, wv;
    int fitBstar;
    uint32_t maxIter;
    double *fitted, *rms;
    uint32_t *iters;
    uint8_t *status;
    uint32_t next;
    pthread_mutex_t m;
} job_t;

static double wrap360(double x) {
    double r = fmod(x, 360.0);
    if (r != 0.0 && r < 0.0) r += 360.0;
    return r;
}

static void to_tle(const double *x, double epoch, azo_tle *t) {
    const double r2d = 180.0 / kPi;
    memset(t, 0, sizeof *t);
    t->epochJd = epoch;
    t->nRevDay = x[0];
    t->ecc = sqrt(x[1] * x[1] + x[2] * x[2]);
    const double w = atan2(x[2], x[1]);
    t->argpDeg = wrap360(w * r2d);
    t->inclDeg = x[3] * r2d;
    t->raanDeg = wrap360(x[4] * r2d);
    t->maDeg = wrap360((x[5] - w) * r2d);
    t->bstar = x[6];
}

static void propagate(const azo_sgp4 *s, double jd, double fr, double epoch, double out[6]) {
    const double ts = ((jd + fr) - epoch) * 1440.0;
    azo_sgp4_propagate(s, ts, out, out + 3);
}

typedef struct { double F, pos2, vel2, floor, N[NV][NV], g[NV]; } sums_t;

/* nominal set x and its perturbations over observations [b, e): 0, or -1 when a set fails init */
static int pass(const job_t *J, const double *x, double epoch, int nv, uint32_t b, uint32_t e, sums_t *S) {
    azo_sgp4 sets[NV + 1];
    double inv[NV + 1] = {0};
    azo_tle t;
    to_tle(x, epoch, &t);
    if (azo_sgp4_init(&t, J->grav, &sets[0]) != AZO_OK) return -1;
    for (int j = 0; j < nv; ++j) {
        double xs[NV];
        int ok = 0;
        memcpy(xs, x, sizeof xs);
        for (int dir = 0; dir < 2 && !ok; ++dir) {
            xs[j] = dir == 0 ? x[j] + 1e-8 : x[j] - 1e-8;
            to_tle(xs, epoch, &t);
            if (azo_sgp4_init(&t, J->grav, &sets[1 + j]) == AZO_OK) {
                inv[1 + j] = 1.0 / (xs[j] - x[j]);
                ok = 1;
            }
        }
        if (!ok) return -1;
    }
    memset(S, 0, sizeof *S);
    const int nc = J->vel ? 6 : 3;
    for (uint32_t i = b; i < e; ++i) {
        double f0[6], obs[6] = {0}, w[6], r[6], jac[NV][6];
        for (int c = 0; c < 3; ++c) {
            obs[c] = J->pos[3 * (size_t)i + c];
            if (J->vel) obs[3 + c] = J->vel[3 * (size_t)i + c];
            w[c] = J->wp;
            w[3 + c] = J->wv;
        }
        propagate(&sets[0], J->jd[i], J->fr[i], epoch, f0);
        for (int c = 0; c < nc; ++c) {
            r[c] = (obs[c] - f0[c]) * w[c];
            S->F += r[c] * r[c];
            const double fl = obs[c] * w[c] * 1e-12;
            S->floor += fl * fl;
            if (c < 3) S->pos2 += (obs[c] - f0[c]) * (obs[c] - f0[c]);
            else S->vel2 += (obs[c] - f0[c]) * (obs[c] - f0[c]);
        }
        for (int j = 0; j < nv; ++j) {
            double f[6];
            propagate(&sets[1 + j], J->jd[i], J->fr[i], epoch, f);
            for (int c = 0; c < nc; ++c) jac[j][c] = (f[c] - f0[c]) * w[c] * inv[1 + j];
        }
        for (int j = 0; j < nv; ++j) {
            for (int c = 0; c < nc; ++c) S->g[j] += jac[j][c] * r[c];
            for (int k = j; k < nv; ++k)
                for (int c = 0; c < nc; ++c) S->N[j][k] += jac[j][c] * jac[k][c];
        }
    }
    return 0;
}

static int solve(const sums_t *S, int nv, double lambda, double *d) {
    double sc[NV], L[NV][NV], y[NV];
    for (int j = 0; j < nv; ++j) sc[j] = S->N[j][j] > 0.0 ? 1.0 / sqrt(S->N[j][j]) : 0.0;
    for (int j = 0; j < NV; ++j) d[j] = 0.0;
    for (int j = 0; j < nv; ++j)
        for (int k = 0; k <= j; ++k) {
            double a = (k == j) ? (sc[j] > 0.0 ? 1.0 + lambda : 1.0) : S->N[k][j] * sc[j] * sc[k];
            for (int q = 0; q < k; ++q) a -= L[j][q] * L[k][q];
            if (k == j) {
                if (!(a > 0.0) || !isfinite(a)) return -1;
                L[j][j] = sqrt(a);
            } else {
                L[j][k] = a / L[k][k];
            }
        }
    for (int j = 0; j < nv; ++j) {
        double b = S->g[j] * sc[j];
        for (int q = 0; q < j; ++q) b -= L[j][q] * y[q];
        y[j] = b / L[j][j];
    }
    for (int j = nv - 1; j >= 0; --j) {
        double b = y[j];
        for (int q = j + 1; q < nv; ++q) b -= L[q][j] * d[q];
        d[j] = b / L[j][j];
    }
    for (int j = 0; j < nv; ++j) d[j] *= sc[j];
    return 0;
}

static void fit_one(const job_t *J, uint32_t s) {
    const uint32_t n = J->n;
    double el[8];
    for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * n + s];
    for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = el[c];
    J->rms[2 * s] = J->rms[2 * s + 1] = 0.0;
    J->iters[s] = 0;
    const int nv = J->fitBstar ? NV : NV - 1;
    azo_tle t;
    memset(&t, 0, sizeof t);
    t.epochJd = el[0]; t.nRevDay = el[1]; t.ecc = el[2]; t.inclDeg = el[3];
    t.raanDeg = el[4]; t.argpDeg = el[5]; t.maDeg = el[6]; t.bstar = el[7];
    azo_sgp4 probe;
    const int rc = azo_sgp4_init(&t, J->grav, &probe);
    if (rc != AZO_OK) {
        J->status[s] = rc == AZO_DEEP_SPACE ? 3 : 2;
        return;
    }
    const uint32_t b = J->off[s], e = J->off[s + 1], m = e > b ? e - b : 0;
    if ((uint64_t)m * (J->vel ? 6 : 3) < (uint64_t)nv) {
        J->status[s] = 4;
        return;
    }
    const double d2r = kPi / 180.0, w = el[5] * d2r;
    double x[NV] = {el[1], el[2] * cos(w), el[2] * sin(w), el[3] * d2r, el[4] * d2r, el[6] * d2r + w, el[7]};
    sums_t S, T;
    if (pass(J, x, el[0], nv, b, e, &S) != 0) {
        J->status[s] = 2;
        return;
    }
    int st = S.F <= S.floor ? 0 : 1;
    double lambda = 1e-3;
    uint32_t it = 0;
    while (st != 0 && it < J->maxIter) {
        ++it;
        double d[NV], xt[NV];
        int ok = solve(&S, nv, lambda, d) == 0;
        if (ok) {
            for (int j = 0; j < NV; ++j) xt[j] = x[j] + d[j];
            ok = pass(J, xt, el[0], nv, b, e, &T) == 0;
        }
        if (!ok || !(T.F < S.F)) {
            if (ok && T.F - S.F <= 1e-10 * S.F) st = 0;
            lambda *= 10.0;
            continue;
        }
        const int small = S.F - T.F <= 1e-10 * S.F;
        memcpy(x, xt, sizeof x);
        S = T;
        lambda *= 0.1;
        if (small || S.F <= S.floor) st = 0;
    }
    to_tle(x, el[0], &t);
    const double out[8] = {t.epochJd, t.nRevDay, t.ecc, t.inclDeg, t.raanDeg, t.argpDeg, t.maDeg, t.bstar};
    for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = out[c];
    J->rms[2 * s] = sqrt(S.pos2 / m);
    J->rms[2 * s + 1] = J->vel ? sqrt(S.vel2 / m) : 0.0;
    J->iters[s] = it;
    J->status[s] = (uint8_t)st;
}

static void *worker(void *arg) {
    job_t *J = (job_t *)arg;
    for (;;) {
        pthread_mutex_lock(&J->m);
        const uint32_t s = J->next++;
        pthread_mutex_unlock(&J->m);
        if (s >= J->n) return NULL;
        fit_one(J, s);
    }
}

int fitref_fit(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
               const double *fr, const double *pos, const double *vel, double pos_sigma, double vel_sigma,
               int fit_bstar, uint32_t max_iter, int threads, double *fitted, double *rms, uint32_t *iterations,
               uint8_t *status) {
    job_t J = {elements, n, grav, offsets, jd, fr, pos, vel, 1.0 / pos_sigma, 1.0 / vel_sigma, fit_bstar, max_iter,
               fitted, rms, iterations, status, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256];
    for (int k = 1; k < threads; ++k) pthread_create(&th[k], NULL, worker, &J);
    worker(&J);
    for (int k = 1; k < threads; ++k) pthread_join(th[k], NULL);
    return 0;
}

/* Observations of one numeric element set (el[8] as above) at m epochs: TEME pos / vel from the oracle, tsince as the
 * fit forms it.  Returns the oracle's init code. */
int fitref_observe(const double *el, int grav, const double *jd, const double *fr, uint32_t m, double *pos,
                   double *vel) {
    azo_tle t;
    memset(&t, 0, sizeof t);
    t.epochJd = el[0]; t.nRevDay = el[1]; t.ecc = el[2]; t.inclDeg = el[3];
    t.raanDeg = el[4]; t.argpDeg = el[5]; t.maDeg = el[6]; t.bstar = el[7];
    azo_sgp4 s;
    const int rc = azo_sgp4_init(&t, grav, &s);
    if (rc != AZO_OK) return rc;
    for (uint32_t i = 0; i < m; ++i) {
        double o[6];
        propagate(&s, jd[i], fr[i], el[0], o);
        memcpy(pos + 3 * (size_t)i, o, 24);
        memcpy(vel + 3 * (size_t)i, o + 3, 24);
    }
    return AZO_OK;
}
