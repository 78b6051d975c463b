/*
 * fit_oracle_deep.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of the deep-space element fit (astroz_b200/csrc/az_fit.cuh, FitDeepSpace, and the
 * _mixed calls) on the CPU oracle's SDP4 (oracle/astroz_oracle.c): element sets go through azo_sgp4_init,
 * azo_sdp4_init and azo_sdp4_propagate, never through the library.  Linked with fit_oracle.c, whose fitref_fit fits the
 * near-earth rows of a mixed batch.  The definition it restates, for a set whose initial elements are deep space
 * (azo_sgp4_init says AZO_DEEP_SPACE):
 *   variables  x = [n rev/day, k = e cos P, h = e sin P, q = tan(i/2) cos node, p = tan(i/2) sin node, L = M + P, B*],
 *              P = w + node (B* held when fit_bstar = 0);
 *   elements   e = |(k, h)|, P = atan2(h, k), i = 2 atan |(p, q)|, node = atan2(p, q), w = P - node, M = L - P,
 *              node / w / M reduced to [0, 360) deg;
 *   class      held: a set is built only when azo_sgp4_init says AZO_DEEP_SPACE (period > 225 min) and azo_sdp4_init
 *              succeeds; otherwise it cannot be built (the backward step, or a rejected step);
 *   model      azo_sdp4_propagate at tsince = ((jd + fr) - epoch) * 1440: the resonance integrator run fresh from
 *              atime = 0 for every observation; a non-zero status of any observation fails the pass (init failure of
 *              the initial set, a rejected step for a trial set);
 *   the rest   as fit_oracle.c: residuals, forward differences of 1e-8, Marquardt damping on the unit-diagonal scaling,
 *              lambda 1e-3 x 10 / 10, stop at a 1e-10 relative cost change or the rounding floor, max_iter steps.
 * Sums run over the observations in order.  Satellites are dealt to pthreads.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include "../../oracle/astroz_oracle.h"

#define NV 7
static const double kPi = 3.14159265358979323846264338327950288;

int fitref_fit(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
               const double *fr, const double *pos, const double *vel, double pos_sigma, double vel_sigma,
               int fit_bstar, uint32_t max_iter, int threads, double *fitted, double *rms, uint32_t *iterations,
               uint8_t *status);

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

static void tle_of(const double *el, azo_tle *t) {
    memset(t, 0, sizeof *t);
    t->epochJd = el[0]; t->nRevDay = el[1]; t->ecc = el[2]; t->inclDeg = el[3];
    t->raanDeg = el[4]; t->argpDeg = el[5]; t->maDeg = el[6]; t->bstar = el[7];
}

static void to_tle(const double *x, double epoch, azo_tle *t) {
    const double r2d = 180.0 / kPi;
    memset(t, 0, sizeof *t);
    t->epochJd = epoch;
    t->nRevDay = x[0];
    t->ecc = sqrt(x[1] * x[1] + x[2] * x[2]);
    const double P = atan2(x[2], x[1]), node = atan2(x[4], x[3]);
    t->inclDeg = 2.0 * atan(sqrt(x[3] * x[3] + x[4] * x[4])) * r2d;
    t->raanDeg = wrap360(node * r2d);
    t->argpDeg = wrap360((P - node) * r2d);
    t->maDeg = wrap360((x[5] - P) * r2d);
    t->bstar = x[6];
}

/* the deep-space set of t: 0, or -1 when it is not one */
static int build(const azo_tle *t, int grav, azo_sdp4 *d) {
    azo_sgp4 probe;
    if (azo_sgp4_init(t, grav, &probe) != AZO_DEEP_SPACE) return -1;
    return azo_sdp4_init(t, grav, d) == AZO_OK ? 0 : -1;
}

static int propagate(const azo_sdp4 *d, double jd, double fr, double epoch, double out[6]) {
    const double ts = ((jd + fr) - epoch) * 1440.0;
    return azo_sdp4_propagate(d, ts, out, out + 3);
}

typedef struct { double F, pos2, vel2, floor, N[NV][NV], g[NV]; } sums_t;

/* nominal set x and its perturbations over observations [b, e): 0, or -1 when a set cannot be built or an observation
 * cannot be propagated */
static int pass(const job_t *J, const double *x, double epoch, int nv, uint32_t b, uint32_t e, sums_t *S) {
    azo_sdp4 sets[NV + 1];
    double inv[NV + 1] = {0};
    azo_tle t;
    to_tle(x, epoch, &t);
    if (build(&t, J->grav, &sets[0]) != 0) return -1;
    for (int j = 0; j < nv; ++j) {
        double xs[NV];
        int ok = 0;
        memcpy(xs, x, sizeof xs);
        for (int dir = 0; dir < 2 && !ok; ++dir) {
            xs[j] = dir == 0 ? x[j] + 1e-8 : x[j] - 1e-8;
            to_tle(xs, epoch, &t);
            if (build(&t, J->grav, &sets[1 + j]) == 0) {
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
        if (propagate(&sets[0], J->jd[i], J->fr[i], epoch, f0) != 0) return -1;
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
            if (propagate(&sets[1 + j], J->jd[i], J->fr[i], epoch, f) != 0) return -1;
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

/* one deep-space row (the caller has checked its class); the near-earth rows keep what fitref_fit wrote */
static void fit_one(const job_t *J, uint32_t s) {
    const uint32_t n = J->n;
    double el[8];
    for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * n + s];
    for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = el[c];
    J->rms[2 * s] = J->rms[2 * s + 1] = 0.0;
    J->iters[s] = 0;
    const int nv = J->fitBstar ? NV : NV - 1;
    const uint32_t b = J->off[s], e = J->off[s + 1], m = e > b ? e - b : 0;
    if ((uint64_t)m * (J->vel ? 6 : 3) < (uint64_t)nv) {
        J->status[s] = 4;
        return;
    }
    const double d2r = kPi / 180.0, node = el[4] * d2r, P = el[5] * d2r + node, ti = tan(0.5 * el[3] * d2r);
    double x[NV] = {el[1], el[2] * cos(P), el[2] * sin(P), ti * cos(node), ti * sin(node), el[6] * d2r + P, el[7]};
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
    azo_tle t;
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
        if (J->status[s] == 3) fit_one(J, s);   /* fitref_fit's DEEP_SPACE rows */
    }
}

/* fitref_fit, and the deep-space rows fitted under the definition above */
int fitref_fit_mixed(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                     const double *fr, const double *pos, const double *vel, double pos_sigma, double vel_sigma,
                     int fit_bstar, uint32_t max_iter, int threads, double *fitted, double *rms, uint32_t *iterations,
                     uint8_t *status) {
    fitref_fit(elements, n, grav, offsets, jd, fr, pos, vel, pos_sigma, vel_sigma, fit_bstar, max_iter, threads, fitted,
               rms, iterations, status);
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

/* Observations of one deep-space element set (el[8], fit_oracle.c's columns) at m epochs: TEME pos / vel from the
 * oracle's SDP4, tsince as the fit forms it.  Returns 0, -1 when the set is not a deep-space set, or 100 + the
 * propagator's status at the first epoch it fails. */
int fitref_observe_deep(const double *el, int grav, const double *jd, const double *fr, uint32_t m, double *pos,
                        double *vel) {
    azo_tle t;
    azo_sdp4 d;
    tle_of(el, &t);
    if (build(&t, grav, &d) != 0) return -1;
    for (uint32_t i = 0; i < m; ++i) {
        double o[6];
        const int st = propagate(&d, jd[i], fr[i], el[0], o);
        if (st != 0) return 100 + st;
        memcpy(pos + 3 * (size_t)i, o, 24);
        memcpy(vel + 3 * (size_t)i, o + 3, 24);
    }
    return 0;
}
