/*
 * fit_oracle_obs.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Independent scalar restatement of the element fit from sensor observations (astroz_b200/csrc/az_obs.cuh and
 * az_fit_obs.cu) on the CPU oracle's SGP4 / SDP4 (oracle/astroz_oracle.c): element sets go through azo_sgp4_init,
 * azo_sgp4_propagate, azo_sdp4_init and azo_sdp4_propagate, never through the library.  Written from the definition:
 *   kinds      0 TEME state; 1 ECEF state, r_e = Rz(g) r, v_e = Rz(g) v - w x r_e with g the GMST polynomial of
 *              jd + fr and w its rate (360.98564736629 deg/day); 2 radar, range / azimuth (north through east) /
 *              elevation / range-rate rho . v_e / |rho| in the WGS84 geodetic horizon frame, rho = r_e - r_station;
 *              3 optical, topocentric right ascension / declination in TEME, rho = r - Rz(g)^T r_station;
 *   residuals  (observed - model) / sigma per component; azimuth / RA differences wrapped to (-pi, pi] and multiplied
 *              by cos of the observed elevation / declination, in the residual and in the forward differences;
 *              sigma = +inf: the component is not used (no cost, no sums, not counted, no floor);
 *   floor      1e-24 sum (s / sigma)^2 over used components, s = |observed value| for states and range, |rho dot| of
 *              the nominal model for range-rate, |r| / |rho| of the nominal model for the angles;
 *   too few    fewer used scalar residuals than fitted variables;
 *   the fit    fit_oracle.c's (near-earth rows) and fit_oracle_deep.c's (deep-space rows of a mixed call): variables,
 *              steps, damping, stopping rule;
 *   covariance at the final iterate, the inverse of J^T W J over the fitted variables, computed column by column
 *              from a Cholesky factorisation of N itself; 28 words of its upper triangle, zero when N is not positive
 *              definite or the row was not fitted;
 *   wrms       sqrt(F / used residuals) at the final iterate.
 * Sums run over the observations in order (the library sums 32 lane partials in a butterfly: same value to rounding).
 * Satellites are dealt to pthreads.
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
    const double *jd, *fr, *value, *sigma;
    const uint32_t *station;
    const uint8_t *kind;
    const double *stations;
    int fitBstar, mixed;
    uint32_t maxIter;
    double *fitted, *wrms, *cov;
    uint32_t *nres, *iters;
    uint8_t *status;
    uint32_t next;
    pthread_mutex_t m;
} job_t;

static double wrap360(double x) {
    double r = fmod(x, 360.0);
    if (r != 0.0 && r < 0.0) r += 360.0;
    return r;
}

static double wrap_pi(double d) {
    d = fmod(d, 2.0 * kPi);
    if (d > kPi) d -= 2.0 * kPi;
    if (d <= -kPi) d += 2.0 * kPi;
    return d;
}

static int count_of(int kind) { return kind <= 1 ? 6 : kind == 2 ? 4 : 2; }
static int wrapped_of(int kind) { return kind == 2 ? 1 : kind == 3 ? 0 : -1; }

/* ---- the model: one element set, near-earth or deep space ---------------------------------------------------------- */
typedef struct {
    int deep;
    azo_sgp4 ne;
    azo_sdp4 ds;
} model_t;

static void to_tle(const double *x, double epoch, int deep, azo_tle *t) {
    const double r2d = 180.0 / kPi;
    memset(t, 0, sizeof *t);
    t->epochJd = epoch;
    t->nRevDay = x[0];
    t->ecc = sqrt(x[1] * x[1] + x[2] * x[2]);
    const double P = atan2(x[2], x[1]);
    if (!deep) {
        t->argpDeg = wrap360(P * r2d);
        t->inclDeg = x[3] * r2d;
        t->raanDeg = wrap360(x[4] * r2d);
        t->maDeg = wrap360((x[5] - P) * r2d);
    } else {
        const double node = atan2(x[4], x[3]);
        t->inclDeg = 2.0 * atan(sqrt(x[3] * x[3] + x[4] * x[4])) * r2d;
        t->raanDeg = wrap360(node * r2d);
        t->argpDeg = wrap360((P - node) * r2d);
        t->maDeg = wrap360((x[5] - P) * r2d);
    }
    t->bstar = x[6];
}

static int build(const double *x, double epoch, int grav, int deep, model_t *M) {
    azo_tle t;
    to_tle(x, epoch, deep, &t);
    M->deep = deep;
    if (!deep) return azo_sgp4_init(&t, grav, &M->ne) == AZO_OK ? 0 : -1;
    azo_sgp4 probe;
    if (azo_sgp4_init(&t, grav, &probe) != AZO_DEEP_SPACE) return -1;
    return azo_sdp4_init(&t, grav, &M->ds) == AZO_OK ? 0 : -1;
}

/* TEME state at jd + fr: 0, or -1 when the deep-space propagator fails */
static int state(const model_t *M, double jd, double fr, double epoch, double f[6]) {
    const double ts = ((jd + fr) - epoch) * 1440.0;
    if (!M->deep) {
        azo_sgp4_propagate(&M->ne, ts, f, f + 3);
        return 0;
    }
    return azo_sdp4_propagate(&M->ds, ts, f, f + 3) == 0 ? 0 : -1;
}

/* ---- the measurement kinds ------------------------------------------------------------------------------------------ */
static double gmst(double jdFull) {
    const double d = jdFull - 2451545.0, t = d / 36525.0;
    double g = 280.46061837 + 360.98564736629 * d + 0.000387933 * t * t - t * t * t / 38710000.0;
    g = fmod(g, 360.0);
    if (g < 0.0) g += 360.0;
    return g * kPi / 180.0;
}

static void station_geometry(const double *llh, double r[3], double e[3], double n[3], double u[3]) {
    const double a = 6378.137, f = 1.0 / 298.257223563, e2 = f * (2.0 - f);
    const double lat = llh[0] * kPi / 180.0, lon = llh[1] * kPi / 180.0, h = llh[2];
    const double N = a / sqrt(1.0 - e2 * sin(lat) * sin(lat));
    r[0] = (N + h) * cos(lat) * cos(lon);
    r[1] = (N + h) * cos(lat) * sin(lon);
    r[2] = (N * (1.0 - e2) + h) * sin(lat);
    e[0] = -sin(lon); e[1] = cos(lon); e[2] = 0.0;
    n[0] = -sin(lat) * cos(lon); n[1] = -sin(lat) * sin(lon); n[2] = cos(lat);
    u[0] = cos(lat) * cos(lon); u[1] = cos(lat) * sin(lon); u[2] = sin(lat);
}

static double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* h[6] of one kind and the floor scales sc[6] (0: |observed value|) */
static void measure(int kind, const double f[6], double jdFull, const double *llh, double h[6], double sc[6]) {
    memset(h, 0, 6 * sizeof(double));
    memset(sc, 0, 6 * sizeof(double));
    if (kind == 0) {
        memcpy(h, f, 6 * sizeof(double));
        return;
    }
    const double g = gmst(jdFull), cg = cos(g), sg = sin(g);
    const double omega = 360.98564736629 * kPi / 180.0 / 86400.0;
    const double re[3] = {cg * f[0] + sg * f[1], -sg * f[0] + cg * f[1], f[2]};
    const double vr[3] = {cg * f[3] + sg * f[4], -sg * f[3] + cg * f[4], f[5]};
    const double ve[3] = {vr[0] + omega * re[1], vr[1] - omega * re[0], vr[2]};   /* v - w x r_e */
    if (kind == 1) {
        memcpy(h, re, sizeof re);
        memcpy(h + 3, ve, sizeof ve);
        return;
    }
    double rs[3], e[3], n[3], u[3];
    station_geometry(llh, rs, e, n, u);
    const double rabs = sqrt(dot3(f, f));
    if (kind == 2) {
        const double rho[3] = {re[0] - rs[0], re[1] - rs[1], re[2] - rs[2]};
        const double E = dot3(rho, e), N = dot3(rho, n), U = dot3(rho, u), range = sqrt(dot3(rho, rho));
        h[0] = range;
        h[1] = atan2(E, N);
        if (h[1] < 0.0) h[1] += 2.0 * kPi;
        h[2] = atan2(U, sqrt(E * E + N * N));
        h[3] = dot3(rho, ve) / range;
        sc[1] = sc[2] = rabs / range;
        sc[3] = sqrt(dot3(ve, ve));
        return;
    }
    const double st[3] = {cg * rs[0] - sg * rs[1], sg * rs[0] + cg * rs[1], rs[2]};   /* Rz(g)^T r_station */
    const double rho[3] = {f[0] - st[0], f[1] - st[1], f[2] - st[2]};
    h[0] = atan2(rho[1], rho[0]);
    if (h[0] < 0.0) h[0] += 2.0 * kPi;
    h[1] = atan2(rho[2], sqrt(rho[0] * rho[0] + rho[1] * rho[1]));
    sc[0] = sc[1] = rabs / sqrt(dot3(rho, rho));
}

/* observation i's weights (0: not used); returns the used count */
static int weights(const job_t *J, uint32_t i, double w[6]) {
    const int kind = J->kind[i], count = count_of(kind), wr = wrapped_of(kind);
    const double *v = J->value + 6 * (size_t)i, *s = J->sigma + 6 * (size_t)i;
    int used = 0;
    for (int c = 0; c < 6; ++c) {
        w[c] = 0.0;
        if (c < count && isfinite(s[c])) {
            w[c] = 1.0 / s[c];
            if (c == wr) w[c] *= cos(v[wr + 1]);
            ++used;
        }
    }
    return used;
}

/* ---- the fit ------------------------------------------------------------------------------------------------------- */
typedef struct { double F, floor, N[NV][NV], g[NV]; } sums_t;

static int pass(const job_t *J, const double *x, double epoch, int nv, int deep, uint32_t b, uint32_t e, sums_t *S) {
    model_t sets[NV + 1];
    double inv[NV + 1] = {0};
    if (build(x, epoch, J->grav, deep, &sets[0]) != 0) return -1;
    for (int j = 0; j < nv; ++j) {
        double xs[NV];
        int ok = 0;
        memcpy(xs, x, sizeof xs);
        for (int dir = 0; dir < 2 && !ok; ++dir) {
            xs[j] = dir == 0 ? x[j] + 1e-8 : x[j] - 1e-8;
            if (build(xs, epoch, J->grav, deep, &sets[1 + j]) == 0) {
                inv[1 + j] = 1.0 / (xs[j] - x[j]);
                ok = 1;
            }
        }
        if (!ok) return -1;
    }
    memset(S, 0, sizeof *S);
    for (uint32_t i = b; i < e; ++i) {
        const int kind = J->kind[i], wr = wrapped_of(kind);
        const double *v = J->value + 6 * (size_t)i;
        const double *llh = (kind >= 2) ? J->stations + 3 * (size_t)J->station[i] : NULL;
        const double jdFull = J->jd[i] + J->fr[i];
        double w[6], f0[6], h0[6], sc[6], r[6] = {0}, jac[NV][6];
        weights(J, i, w);
        if (state(&sets[0], J->jd[i], J->fr[i], epoch, f0) != 0) return -1;
        measure(kind, f0, jdFull, llh, h0, sc);
        for (int c = 0; c < 6; ++c) {
            if (w[c] == 0.0) continue;
            const double d = c == wr ? wrap_pi(v[c] - h0[c]) : v[c] - h0[c];
            r[c] = d * w[c];
            S->F += r[c] * r[c];
            const double fl = (sc[c] != 0.0 ? sc[c] : v[c]) * w[c] * 1e-12;
            S->floor += fl * fl;
        }
        for (int j = 0; j < nv; ++j) {
            double f[6], hj[6], scj[6];
            if (state(&sets[1 + j], J->jd[i], J->fr[i], epoch, f) != 0) return -1;
            measure(kind, f, jdFull, llh, hj, scj);
            for (int c = 0; c < 6; ++c) {
                const double d = c == wr ? wrap_pi(hj[c] - h0[c]) : hj[c] - h0[c];
                jac[j][c] = w[c] != 0.0 ? d * w[c] * inv[1 + j] : 0.0;
            }
        }
        for (int j = 0; j < nv; ++j) {
            for (int c = 0; c < 6; ++c) S->g[j] += jac[j][c] * r[c];
            for (int k = j; k < nv; ++k)
                for (int c = 0; c < 6; ++c) S->N[j][k] += jac[j][c] * jac[k][c];
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

/* N^-1 column by column: N = L L^T, solve L L^T c_k = e_k.  cov[28] upper triangle row by row; -1 if not SPD */
static int covariance(const sums_t *S, int nv, double *cov) {
    double L[NV][NV], P[NV][NV];
    memset(cov, 0, 28 * sizeof(double));
    for (int j = 0; j < nv; ++j)
        for (int k = 0; k <= j; ++k) {
            double a = S->N[k][j];
            for (int q = 0; q < k; ++q) a -= L[j][q] * L[k][q];
            if (k == j) {
                if (!(a > 0.0) || !isfinite(a)) return -1;
                L[j][j] = sqrt(a);
            } else {
                L[j][k] = a / L[k][k];
            }
        }
    for (int col = 0; col < nv; ++col) {
        double y[NV], c[NV];
        for (int j = 0; j < nv; ++j) {
            double b = j == col ? 1.0 : 0.0;
            for (int q = 0; q < j; ++q) b -= L[j][q] * y[q];
            y[j] = b / L[j][j];
        }
        for (int j = nv - 1; j >= 0; --j) {
            double b = y[j];
            for (int q = j + 1; q < nv; ++q) b -= L[q][j] * c[q];
            c[j] = b / L[j][j];
        }
        for (int j = 0; j < nv; ++j) P[j][col] = c[j];
    }
    int w = 0;
    for (int j = 0; j < NV; ++j)
        for (int k = j; k < NV; ++k, ++w) cov[w] = (j < nv && k < nv) ? 0.5 * (P[j][k] + P[k][j]) : 0.0;
    return 0;
}

static void fit_one(const job_t *J, uint32_t s, int deep) {
    const uint32_t n = J->n;
    double el[8];
    for (int c = 0; c < 8; ++c) el[c] = J->el[(size_t)c * n + s];
    for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = el[c];
    memset(J->cov + 28 * (size_t)s, 0, 28 * sizeof(double));
    J->wrms[s] = 0.0;
    J->iters[s] = 0;
    const int nv = J->fitBstar ? NV : NV - 1;
    const uint32_t b = J->off[s], e = J->off[s + 1];
    uint32_t used = 0;
    for (uint32_t i = b; i < e; ++i) {
        double w[6];
        used += (uint32_t)weights(J, i, w);
    }
    J->nres[s] = used;
    if (used < (uint32_t)nv) {
        J->status[s] = 4;
        return;
    }
    const double d2r = kPi / 180.0;
    double x[NV];
    if (!deep) {
        const double w = el[5] * d2r;
        const double x0[NV] = {el[1], el[2] * cos(w), el[2] * sin(w), el[3] * d2r, el[4] * d2r, el[6] * d2r + w, el[7]};
        memcpy(x, x0, sizeof x);
    } else {
        const double node = el[4] * d2r, P = el[5] * d2r + node, ti = tan(0.5 * el[3] * d2r);
        const double x0[NV] = {el[1], el[2] * cos(P), el[2] * sin(P), ti * cos(node), ti * sin(node), el[6] * d2r + P,
                               el[7]};
        memcpy(x, x0, sizeof x);
    }
    sums_t S, T;
    if (pass(J, x, el[0], nv, deep, b, e, &S) != 0) {
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
            ok = pass(J, xt, el[0], nv, deep, b, e, &T) == 0;
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
    to_tle(x, el[0], deep, &t);
    const double out[8] = {t.epochJd, t.nRevDay, t.ecc, t.inclDeg, t.raanDeg, t.argpDeg, t.maDeg, t.bstar};
    for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = out[c];
    covariance(&S, nv, J->cov + 28 * (size_t)s);
    J->wrms[s] = sqrt(S.F / used);
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
        azo_tle t;
        memset(&t, 0, sizeof t);
        const double *el = J->el;
        const uint32_t n = J->n;
        t.epochJd = el[s]; t.nRevDay = el[n + s]; t.ecc = el[2 * (size_t)n + s]; t.inclDeg = el[3 * (size_t)n + s];
        t.raanDeg = el[4 * (size_t)n + s]; t.argpDeg = el[5 * (size_t)n + s]; t.maDeg = el[6 * (size_t)n + s];
        t.bstar = el[7 * (size_t)n + s];
        azo_sgp4 probe;
        const int rc = azo_sgp4_init(&t, J->grav, &probe);
        if (rc == AZO_OK) {
            fit_one(J, s, 0);
        } else if (rc == AZO_DEEP_SPACE && J->mixed) {
            fit_one(J, s, 1);
        } else {   /* not fitted: the initial columns, DEEP_SPACE or INIT_FAILED */
            for (int c = 0; c < 8; ++c) J->fitted[(size_t)c * n + s] = el[(size_t)c * n + s];
            memset(J->cov + 28 * (size_t)s, 0, 28 * sizeof(double));
            uint32_t used = 0;
            for (uint32_t i = J->off[s]; i < J->off[s + 1]; ++i) {
                double w[6];
                used += (uint32_t)weights(J, i, w);
            }
            J->nres[s] = used;
            J->wrms[s] = 0.0;
            J->iters[s] = 0;
            J->status[s] = rc == AZO_DEEP_SPACE ? 3 : 2;
        }
    }
}

/* astroz_cuda_fit_observations (mixed = 0) and _mixed (mixed = 1), restated; the argument layout of the C ABI */
int fitref_fit_obs(const double *elements, uint32_t n, int grav, const uint32_t *offsets, const double *jd,
                   const double *fr, const double *value, const double *sigma, const uint32_t *station,
                   const uint8_t *kind, const double *stations, int fit_bstar, uint32_t max_iter, int mixed,
                   int threads, double *fitted, double *wrms, uint32_t *n_residuals, double *covariance_out,
                   uint32_t *iterations, uint8_t *status) {
    job_t J = {elements, n, grav, offsets, jd, fr, value, sigma, station, kind, stations, fit_bstar, mixed, max_iter,
               fitted, wrms, covariance_out, n_residuals, iterations, status, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t th[256];
    for (int k = 1; k < threads; ++k) pthread_create(&th[k], NULL, worker, &J);
    worker(&J);
    for (int k = 1; k < threads; ++k) pthread_join(th[k], NULL);
    return 0;
}
