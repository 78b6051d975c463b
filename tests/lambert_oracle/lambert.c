/* TEST INFRASTRUCTURE ONLY: a scalar C statement of Izzo's Lambert solver ("Revisiting Lambert's problem", Celest. Mech.
 * Dyn. Astron. 121, 2015) with the conventions of the library's K9: the unit normal n sets the direction (the long way
 * when (r1 x r2) . n < 0), S = 2 max_revs + 1 slots (0: M = 0; 2M - 1 left, 2M right), Householder steps until
 * |dx| < 1e-13 (at most 15), T_min by Halley steps for the largest candidate M, status bytes 0 ok, 1 no solution,
 * 2 degenerate, 3 not converged, non-OK slots zero-filled.  Compiled with gcc -ffp-contract=off.  lam_batch deals problems
 * to pthreads for the timing tool; a problem's arithmetic does not depend on the thread. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PI 3.141592653589793
#define MAX_ITER 15
#define TOL 1e-13

static double norm3(const double *a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }
static void cross3(const double *a, const double *b, double *o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

static double hyp2f1(double z) { /* 2F1(3, 1; 5/2; z) */
    double sum = 1.0, term = 1.0;
    for (int j = 0; j < 100; ++j) {
        term = term * (3.0 + j) / (2.5 + j) * z;
        sum = sum + term;
        if (fabs(term) < 1e-17) break;
    }
    return sum;
}

double lam_tof(double x, double lam, int M) {
    double dist = fabs(x - 1.0), l2 = lam * lam;
    if (dist < 0.2 && dist > 0.01) { /* Lagrange */
        double a = 1.0 / (1.0 - x * x);
        if (a > 0.0) {
            double alfa = 2.0 * acos(x), beta = 2.0 * asin(sqrt(l2 / a));
            if (lam < 0.0) beta = -beta;
            return a * sqrt(a) * ((alfa - sin(alfa)) - (beta - sin(beta)) + 2.0 * PI * M) / 2.0;
        } else {
            double alfa = 2.0 * acosh(x), beta = 2.0 * asinh(sqrt(-l2 / a));
            if (lam < 0.0) beta = -beta;
            return -a * sqrt(-a) * ((beta - sinh(beta)) - (alfa - sinh(alfa))) / 2.0;
        }
    }
    double E = x * x - 1.0, z = sqrt(1.0 + l2 * E);
    if (dist < 0.01) { /* Battin */
        double eta = z - lam * x, s1 = 0.5 * (1.0 - lam - x * eta);
        double q = 4.0 / 3.0 * hyp2f1(s1), rho = fabs(E);
        double rev = M ? M * PI / (rho * sqrt(rho)) : 0.0;
        return (eta * eta * eta * q + 4.0 * lam * eta) / 2.0 + rev;
    }
    double y = sqrt(fabs(E)), g = x * z - lam * E; /* Lancaster */
    double d = E < 0.0 ? M * PI + acos(g) : log(y * (z - lam * x) + g);
    return (x - lam * z - d / y) / E;
}

static void dtdx(double x, double T, double lam, double *d1, double *d2, double *d3) {
    double l2 = lam * lam, l3 = l2 * lam, umx2 = 1.0 - x * x;
    double y = sqrt(1.0 - l2 * umx2), y2 = y * y, y3 = y2 * y;
    *d1 = (3.0 * T * x - 2.0 + 2.0 * l3 * x / y) / umx2;
    *d2 = (3.0 * T + 5.0 * x * *d1 + 2.0 * (1.0 - l2) * l3 / y3) / umx2;
    *d3 = (7.0 * x * *d2 + 8.0 * *d1 - 6.0 * (1.0 - l2) * l2 * l3 * x / (y3 * y2)) / umx2;
}

double lam_tmin(double lam, int M) {
    double x = 0.0, t = acos(lam) + lam * sqrt(1.0 - lam * lam) + M * PI;
    for (int it = 0; it < MAX_ITER; ++it) {
        double d1, d2, d3;
        dtdx(x, t, lam, &d1, &d2, &d3);
        double xn = x - d1 * d2 / (d2 * d2 - d1 * d3 / 2.0), err = fabs(x - xn);
        x = xn;
        t = lam_tof(x, lam, M);
        if (err < TOL) break;
    }
    return t;
}

/* lam and T of a problem (0), or its whole-problem status */
int lam_geometry(const double *r1, const double *r2, double tof, double mu, const double *n, double *out) {
    if (!(tof > 0.0)) return 1;
    double r1n = norm3(r1), r2n = norm3(r2);
    if (r1n == 0.0 || r2n == 0.0) return 2;
    double h[3];
    cross3(r1, r2, h);
    double hn = norm3(h);
    if (hn < 1e-12 * (r1n * r2n)) return 2;
    double ih[3] = {h[0] / hn, h[1] / hn, h[2] / hn};
    double dn = ih[0] * n[0] + ih[1] * n[1] + ih[2] * n[2];
    if (dn == 0.0) return 2;
    double dd[3] = {r2[0] - r1[0], r2[1] - r1[1], r2[2] - r1[2]};
    double c = norm3(dd), s = (r1n + r2n + c) / 2.0;
    double ir1[3], ir2[3], it1[3], it2[3];
    for (int k = 0; k < 3; ++k) ir1[k] = r1[k] / r1n, ir2[k] = r2[k] / r2n;
    double lam = sqrt(1.0 - c / s);
    if (dn < 0.0) {
        lam = -lam;
        cross3(ir1, ih, it1);
        cross3(ir2, ih, it2);
    } else {
        cross3(ih, ir1, it1);
        cross3(ih, ir2, it2);
    }
    /* out: lam, T, s, c, r1n, r2n, ir1, ir2, it1, it2 */
    out[0] = lam;
    out[1] = sqrt(2.0 * mu / (s * s * s)) * tof;
    out[2] = s, out[3] = c, out[4] = r1n, out[5] = r2n;
    for (int k = 0; k < 3; ++k) out[6 + k] = ir1[k], out[9 + k] = ir2[k], out[12 + k] = it1[k], out[15 + k] = it2[k];
    return 0;
}

static int mmax(double T, double lam, uint32_t maxRevs) {
    double mt = floor(T / PI);
    int M = mt < (double)maxRevs ? (int)mt : (int)maxRevs;
    if (M > 0 && T < acos(lam) + lam * sqrt(1.0 - lam * lam) + M * PI && lam_tmin(lam, M) > T) --M;
    return M;
}

static double guess(double T, double lam, uint32_t slot) {
    int M = (int)((slot + 1) / 2);
    if (M == 0) {
        double l2 = lam * lam, l3 = l2 * lam;
        double t00 = acos(lam) + lam * sqrt(1.0 - l2), t1 = 2.0 / 3.0 * (1.0 - l3);
        if (T >= t00) return -(T - t00) / (T - t00 + 4.0);
        if (T <= t1) return t1 * (t1 - T) / (2.0 / 5.0 * (1.0 - l2 * l3) * T) + 1.0;
        return pow(T / t00, 0.69314718055994529 / log(t1 / t00)) - 1.0;
    }
    double v = (slot & 1) ? (M + 1) * PI / (8.0 * T) : 8.0 * T / (M * PI);
    double q = cbrt(v * v);
    return (q - 1.0) / (q + 1.0);
}

static int householder(double T, double lam, int M, double *x) {
    for (int it = 1; it <= MAX_ITER; ++it) {
        double t = lam_tof(*x, lam, M), d1, d2, d3;
        dtdx(*x, t, lam, &d1, &d2, &d3);
        double delta = t - T, d1s = d1 * d1;
        double xn = *x - delta * (d1s - delta * d2 / 2.0) / (d1 * (d1s - delta * d2) + d3 * delta * delta / 6.0);
        double err = fabs(*x - xn);
        *x = xn;
        if (err < TOL) return it;
    }
    return 0;
}

/* one problem: v1 / v2 [S][3], status / iters [S] */
void lam_solve(const double *r1, const double *r2, double tof, double mu, const double *n, uint32_t maxRevs, double *v1,
               double *v2, uint8_t *status, uint8_t *iters) {
    uint32_t S = 2 * maxRevs + 1;
    double g[18];
    memset(v1, 0, S * 24);
    memset(v2, 0, S * 24);
    memset(iters, 0, S);
    int st = lam_geometry(r1, r2, tof, mu, n, g);
    if (st) {
        memset(status, st, S);
        return;
    }
    double lam = g[0], T = g[1], s = g[2], c = g[3], r1n = g[4], r2n = g[5];
    int mMax = mmax(T, lam, maxRevs);
    for (uint32_t slot = 0; slot < S; ++slot) {
        int M = (int)((slot + 1) / 2);
        if (M > mMax) {
            status[slot] = 1;
            continue;
        }
        double x = guess(T, lam, slot);
        int it = householder(T, lam, M, &x);
        if (!it) {
            status[slot] = 3;
            iters[slot] = MAX_ITER;
            continue;
        }
        double gamma = sqrt(mu * s / 2.0), rho = (r1n - r2n) / c, sigma = sqrt(fmax(0.0, 1.0 - rho * rho));
        double y = sqrt(1.0 - lam * lam * (1.0 - x * x));
        double vr1 = gamma * ((lam * y - x) - rho * (lam * y + x)) / r1n;
        double vr2 = -gamma * ((lam * y - x) + rho * (lam * y + x)) / r2n;
        double vt = gamma * sigma * (y + lam * x), vt1 = vt / r1n, vt2 = vt / r2n;
        for (int k = 0; k < 3; ++k) {
            v1[3 * slot + k] = vr1 * g[6 + k] + vt1 * g[12 + k];
            v2[3 * slot + k] = vr2 * g[9 + k] + vt2 * g[15 + k];
        }
        status[slot] = 0;
        iters[slot] = (uint8_t)it;
    }
}

typedef struct {
    const double *r1, *r2, *tof, *normal;
    double mu;
    uint32_t maxRevs;
    double *v1, *v2;
    uint8_t *status, *iters;
    size_t begin, end;
} Job;

static void *run(void *p) {
    const Job *j = (const Job *)p;
    size_t S = 2 * (size_t)j->maxRevs + 1;
    const double z[3] = {0.0, 0.0, 1.0};
    for (size_t i = j->begin; i < j->end; ++i)
        lam_solve(j->r1 + 3 * i, j->r2 + 3 * i, j->tof[i], j->mu, j->normal ? j->normal + 3 * i : z, j->maxRevs,
                  j->v1 + 3 * S * i, j->v2 + 3 * S * i, j->status + S * i, j->iters + S * i);
    return NULL;
}

/* n problems (normal nullable: +z), dealt in contiguous ranges to `threads` pthreads */
void lam_batch(const double *r1, const double *r2, const double *tof, const double *normal, size_t n, double mu,
               uint32_t maxRevs, double *v1, double *v2, uint8_t *status, uint8_t *iters, int threads) {
    if (threads < 1) threads = 1;
    pthread_t *t = malloc(sizeof(pthread_t) * threads);
    Job *jobs = malloc(sizeof(Job) * threads);
    for (int k = 0; k < threads; ++k) {
        Job j = {r1, r2, tof, normal, mu, maxRevs, v1, v2, status, iters, n * k / threads, n * (k + 1) / threads};
        jobs[k] = j;
        pthread_create(&t[k], NULL, run, &jobs[k]);
    }
    for (int k = 0; k < threads; ++k) pthread_join(t[k], NULL);
    free(t);
    free(jobs);
}
