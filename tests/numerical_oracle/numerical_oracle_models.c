/* TEST INFRASTRUCTURE ONLY: scalar C restatement of the reference's force models (src/propagators/ForceModel.zig) and of
 * Propagator.propagate under an ordered list of them, the yardstick K7's model lists (astroz_b200/csrc/az_numerical.cuh)
 * are checked against.  Built with -ffp-contract=off.  It includes numerical_oracle.c for the DP87 tableau, the sampling
 * loop (azn_times) and the status values, and restates the integrators with the list's acceleration as the force.
 * Every function names the reference lines it restates. */
#include "numerical_oracle.c"

/* One force model of a list, laid out as astroz_force_model_t (include/astroz_b200.h), so a test can hand the same
 * descriptors to the product and to this restatement. */
typedef struct {
    int32_t kind;
    uint32_t flags;
    double mu, coef, rEq, rho0, H, maxAltitude, f107, c, area, mass, pos[3];
    const double *cArr, *areaArr, *massArr, *posTable;
} ListModel;
typedef struct {
    const ListModel *models;
    int count;
    size_t i;   /* batch item: its per-state coefficients */
    uint64_t k; /* output interval: its row of each position table */
    double rtol, atol;
    int k7Factor; /* 1: errNorm^(-1/8) as K7 forms it (three square roots) instead of the reference's pow */
} ListCtx;

/* ---- model lists: the force models of src/propagators/ForceModel.zig, one function per kind ---------------------- */
enum { M_TWO_BODY, M_J2, M_J3, M_J4, M_DRAG, M_IMPROVED_DRAG, M_SRP, M_THIRD_BODY };
enum { PS_C = 1, PS_AREA = 2, PS_MASS = 4, POS_TABLE = 8 };

static double coef(const ListModel *m, const ListCtx *l, unsigned flag, double scalar, const double *arr) {
    return (m->flags & flag) ? arr[l->i] : scalar;
}
static void position(const ListModel *m, const ListCtx *l, double q[3]) {
    const double *p = (m->flags & POS_TABLE) ? m->posTable + l->k * 3 : m->pos;
    q[0] = p[0], q[1] = p[1], q[2] = p[2];
}

/* TwoBody.acceleration, ForceModel.zig:49-55 */
static void two_body(const ListModel *m, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double r = sqrt(x * x + y * y + z * z);
    const double factor = -m->mu / (r * r * r);
    a[0] = factor * x, a[1] = factor * y, a[2] = factor * z;
}
/* J2.acceleration, ForceModel.zig:67-79 */
static void j2_accel(const ListModel *m, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double r2 = x * x + y * y + z * z;
    const double r = sqrt(r2);
    const double factor = -1.5 * m->coef * m->mu * m->rEq * m->rEq / (r2 * r2 * r);
    const double z2R2 = (z * z) / r2;
    a[0] = factor * x * (5.0 * z2R2 - 1.0), a[1] = factor * y * (5.0 * z2R2 - 1.0), a[2] = factor * z * (5.0 * z2R2 - 3.0);
}
/* J3.acceleration, ForceModel.zig:122-142 */
static void j3_accel(const ListModel *m, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double r2 = x * x + y * y + z * z;
    const double r = sqrt(r2);
    const double rEq3 = m->rEq * m->rEq * m->rEq;
    const double factor = 2.5 * m->coef * m->mu * rEq3 / (r2 * r2 * r2 * r);
    const double z2R2 = (z * z) / r2;
    const double xyCoeff = 3.0 * z / r - 7.0 * z * z2R2 / r;
    const double zCoeff = 6.0 * z * z - 7.0 * z * z * z2R2 - 0.6 * r2;
    a[0] = factor * x * xyCoeff, a[1] = factor * y * xyCoeff, a[2] = factor * zCoeff;
}
/* J4.acceleration, ForceModel.zig:154-175 */
static void j4_accel(const ListModel *m, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double r2 = x * x + y * y + z * z;
    const double r = sqrt(r2);
    const double r4 = r2 * r2, z2 = z * z;
    const double z4 = z2 * z2;
    const double z2R2 = z2 / r2, z4R4 = z4 / r4;
    const double rEq4 = m->rEq * m->rEq * m->rEq * m->rEq;
    const double factor = 1.875 * m->coef * m->mu * rEq4 / (r4 * r4 * r);
    const double xyTerm = 3.0 - 42.0 * z2R2 + 63.0 * z4R4;
    const double zTerm = 15.0 - 70.0 * z2R2 + 63.0 * z4R4;
    a[0] = factor * x * xyTerm, a[1] = factor * y * xyTerm, a[2] = factor * z * zTerm;
}
/* Drag.acceleration, ForceModel.zig:95-110 */
static void drag_accel(const ListModel *m, const ListCtx *l, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2], vx = s[3], vy = s[4], vz = s[5];
    a[0] = a[1] = a[2] = 0;
    const double r = sqrt(x * x + y * y + z * z);
    const double altitude = r - m->rEq;
    if (altitude > m->maxAltitude) return;
    const double v = sqrt(vx * vx + vy * vy + vz * vz);
    if (v < 1e-10) return;
    const double rho = m->rho0 * exp(-altitude / m->H);
    const double factor = -0.5 * coef(m, l, PS_C, m->c, m->cArr) * coef(m, l, PS_AREA, m->area, m->areaArr) * rho * v *
                          1e3 / coef(m, l, PS_MASS, m->mass, m->massArr);
    a[0] = factor * vx / v, a[1] = factor * vy / v, a[2] = factor * vz / v;
}
/* ImprovedDrag.getDensity, ForceModel.zig:283-320 */
static const double LAYERS[5][3] = {{100.0, 5.297e-7, 5.877}, {200.0, 2.789e-10, 37.105}, {400.0, 3.725e-12, 62.822},
                                    {600.0, 2.418e-13, 79.864}, {1000.0, 3.561e-15, 200.0}};
static double improved_density(double altitude, double f107) {
    int layerIdx = 0;
    for (int i = 0; i < 5; ++i)
        if (altitude >= LAYERS[i][0]) layerIdx = i;
    const double deltaH = altitude - LAYERS[layerIdx][0];
    double rho = LAYERS[layerIdx][1] * exp(-deltaH / LAYERS[layerIdx][2]);
    const double f107Scale = f107 / 150.0;
    rho *= f107Scale;
    return rho;
}
/* ImprovedDrag.acceleration, ForceModel.zig:322-348, omega 7.2921150e-5 (:292) */
static void improved_drag_accel(const ListModel *m, const ListCtx *l, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2], vx = s[3], vy = s[4], vz = s[5];
    a[0] = a[1] = a[2] = 0;
    const double r = sqrt(x * x + y * y + z * z);
    const double altitude = r - m->rEq;
    if (altitude > m->maxAltitude || altitude < 100.0) return;
    const double omega = 7.2921150e-5;
    const double vrelX = vx + omega * y, vrelY = vy - omega * x, vrelZ = vz;
    const double vrel = sqrt(vrelX * vrelX + vrelY * vrelY + vrelZ * vrelZ);
    if (vrel < 1e-10) return;
    const double rho = improved_density(altitude, m->f107);
    const double factor = -0.5 * coef(m, l, PS_C, m->c, m->cArr) * coef(m, l, PS_AREA, m->area, m->areaArr) * rho *
                          vrel * 1e3 / coef(m, l, PS_MASS, m->mass, m->massArr);
    a[0] = factor * vrelX / vrel, a[1] = factor * vrelY / vrel, a[2] = factor * vrelZ / vrel;
}
/* SolarRadiationPressure.acceleration, ForceModel.zig:197-227; pSr 4.56e-6, AU 1.495978707e8 (constants.zig:27-28) */
static void srp_accel(const ListModel *m, const ListCtx *l, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double pSr = 4.56e-6, au = 1.495978707e8;
    double sp[3];
    position(m, l, sp);
    a[0] = a[1] = a[2] = 0;
    const double dx = sp[0] - x, dy = sp[1] - y, dz = sp[2] - z;
    const double dist = sqrt(dx * dx + dy * dy + dz * dz);
    if (dist < 1e-10) return;
    const double sunDir[3] = {dx / dist, dy / dist, dz / dist};
    const double sunDist = sqrt(sp[0] * sp[0] + sp[1] * sp[1] + sp[2] * sp[2]);
    if (sunDist < 1e-10) return;
    const double sunHat[3] = {sp[0] / sunDist, sp[1] / sunDist, sp[2] / sunDist};
    const double proj = x * sunHat[0] + y * sunHat[1] + z * sunHat[2];
    if (proj < 0) {
        const double perpX = x - proj * sunHat[0], perpY = y - proj * sunHat[1], perpZ = z - proj * sunHat[2];
        const double rho = sqrt(perpX * perpX + perpY * perpY + perpZ * perpZ);
        if (rho < m->rEq) return;
    }
    const double scale = (au / dist) * (au / dist);
    const double factor = -coef(m, l, PS_C, m->c, m->cArr) * pSr * scale * coef(m, l, PS_AREA, m->area, m->areaArr) /
                          coef(m, l, PS_MASS, m->mass, m->massArr) * 1e-3;
    a[0] = factor * sunDir[0], a[1] = factor * sunDir[1], a[2] = factor * sunDir[2];
}
/* ThirdBody.acceleration, ForceModel.zig:244-265 */
static void third_body_accel(const ListModel *m, const ListCtx *l, const double s[6], double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    double q[3];
    position(m, l, q);
    a[0] = a[1] = a[2] = 0;
    const double qMag = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    if (qMag < 1e-10) return;
    const double qMag3 = qMag * qMag * qMag;
    const double dx = q[0] - x, dy = q[1] - y, dz = q[2] - z;
    const double dMag = sqrt(dx * dx + dy * dy + dz * dz);
    if (dMag < 1e-10) return;
    const double dMag3 = dMag * dMag * dMag;
    a[0] = m->mu * (dx / dMag3 - q[0] / qMag3);
    a[1] = m->mu * (dy / dMag3 - q[1] / qMag3);
    a[2] = m->mu * (dz / dMag3 - q[2] / qMag3);
}

static void one_model(const ListModel *m, const ListCtx *l, const double s[6], double a[3]) {
    switch (m->kind) {
        case M_TWO_BODY: two_body(m, s, a); break;
        case M_J2: j2_accel(m, s, a); break;
        case M_J3: j3_accel(m, s, a); break;
        case M_J4: j4_accel(m, s, a); break;
        case M_DRAG: drag_accel(m, l, s, a); break;
        case M_IMPROVED_DRAG: improved_drag_accel(m, l, s, a); break;
        case M_SRP: srp_accel(m, l, s, a); break;
        default: third_body_accel(m, l, s, a); break;
    }
}

/* one model as it is (bindings/python/src/propagator.zig:138-146); several through Composite (ForceModel.zig:365-374) */
static void list_acceleration(const ListCtx *l, const double s[6], double out[3]) {
    if (l->count == 1) {
        one_model(&l->models[0], l, s, out);
        return;
    }
    double total[3] = {0, 0, 0};
    for (int j = 0; j < l->count; ++j) {
        double a[3];
        one_model(&l->models[j], l, s, a);
        total[0] += a[0];
        total[1] += a[1];
        total[2] += a[2];
    }
    memcpy(out, total, sizeof total);
}

/* The list's acceleration at n states s[n][6] for batch items items[n] in interval k: out[n][3] */
void azn_models_accel(const ListModel *models, int count, const double *s, const uint64_t *items, uint64_t k, size_t n,
                      double *out) {
    for (size_t j = 0; j < n; ++j) {
        ListCtx l = {models, count, (size_t)items[j], k, 0, 0, 0};
        list_acceleration(&l, s + 6 * j, out + 3 * j);
    }
}


/* ---- the integrators and the sampling loop over a model list: numerical_oracle.c's restatement of Integrator.zig and
 * Propagator.zig, with the list's acceleration as the force ------------------------------------------------------ */

/* derivative (Integrator.zig:47-50, :261-264) */
static void list_derivative(const ListCtx *l, const double s[6], double k[6]) {
    double a[3];
    list_acceleration(l, s, a);
    k[0] = s[3], k[1] = s[4], k[2] = s[5], k[3] = a[0], k[4] = a[1], k[5] = a[2];
}

/* Rk4.step (Integrator.zig:28-45) */
static void list_rk4_step(const ListCtx *l, double y[6], double dt) {
    double k1[6], k2[6], k3[6], k4[6], s[6];
    list_derivative(l, y, k1);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k1[c] * (0.5 * dt);
    list_derivative(l, s, k2);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k2[c] * (0.5 * dt);
    list_derivative(l, s, k3);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k3[c] * dt;
    list_derivative(l, s, k4);
    const double factor = dt / 6.0;
    for (int c = 0; c < 6; ++c) y[c] = y[c] + factor * (k1[c] + 2.0 * k2[c] + 2.0 * k3[c] + k4[c]);
}

/* DormandPrince87.adaptiveStep (Integrator.zig:190-259): y8 and errNorm of one attempt, *hNew */
static double list_dp87_attempt(const ListCtx *l, const double y[6], double h, double y8[6], double *hNew) {
    double k[13][6], y7[6];
    list_derivative(l, y, k[0]);
    for (int i = 1; i < 13; ++i) {
        double ys[6];
        memcpy(ys, y, sizeof ys);
        for (int j = 0; j < i; ++j)
            if (A_[i][j] != 0)
                for (int c = 0; c < 6; ++c) ys[c] = ys[c] + (A_[i][j] * h) * k[j][c];
        list_derivative(l, ys, k[i]);
    }
    memcpy(y8, y, 6 * sizeof(double));
    for (int i = 0; i < 13; ++i)
        if (B8_[i] != 0)
            for (int c = 0; c < 6; ++c) y8[c] = y8[c] + (B8_[i] * h) * k[i][c];
    memcpy(y7, y, sizeof y7);
    for (int i = 0; i < 13; ++i)
        if (B7_[i] != 0)
            for (int c = 0; c < 6; ++c) y7[c] = y7[c] + (B7_[i] * h) * k[i][c];
    double errNorm = 0;
    for (int c = 0; c < 6; ++c) {
        const double scale = l->atol + l->rtol * fmax(fabs(y[c]), fabs(y8[c]));
        const double se = (y8[c] - y7[c]) / scale;
        errNorm += se * se;
    }
    errNorm = sqrt(errNorm / 6.0);
    double hn;
    if (errNorm < 1e-10) {
        hn = h * 5.0;
    } else {
        const double factor = l->k7Factor ? 0.9 * sqrt(sqrt(sqrt(1.0 / errNorm))) : 0.9 * pow(1.0 / errNorm, 1.0 / 8.0);
        hn = h * fmin(5.0, fmax(0.1, factor)); /* fmin / fmax ignore a NaN, as Zig's @min / @max */
    }
    hn = fmin(hn, 3600.0);
    *hNew = fmax(hn, 0.001);
    return errNorm;
}

/* DormandPrince87.step (Integrator.zig:154-182) over one output interval; hCur carries across intervals */
static int list_dp87_step(const ListCtx *l, double y[6], double dt, double *hCur, uint64_t counts[2]) {
    double remaining = dt, h = fmin(*hCur, remaining);
    uint32_t substeps = 0;
    while (remaining > 1e-14 && substeps < 10000) {
        h = fmin(h, remaining);
        h = fmax(h, 0.001);
        double y8[6], hNew;
        const double errNorm = list_dp87_attempt(l, y, h, y8, &hNew);
        if (errNorm <= 1.0) {
            memcpy(y, y8, sizeof y8);
            remaining -= h;
            ++substeps;
            ++counts[0];
        } else {
            ++counts[1];
            if (h == 0.001) { /* the reference retries this attempt unchanged, forever */
                *hCur = hNew;
                return ST_STOPPED;
            }
        }
        h = hNew;
    }
    *hCur = h;
    return remaining > 1e-14 ? ST_SUBSTEP_LIMIT : ST_OK;
}

/* Propagator.propagate (Propagator.zig:22-48) for one state; before each step, l->k is set to the step's interval, the
 * SPICE example's updateSunPos / updatePos between steps (examples/spice_propagation.zig:74-82).  out[(K + 1) * 6],
 * counts[2]; returns the status byte. */
static int list_propagate_one(ListCtx *l, int integrator, const double y0[6], double t0, double duration, double dt,
                              double *out, uint64_t counts[2]) {
    pthread_once(&tableau_once, tableau_init);
    double y[6], t = t0, hCur = 60.0;
    const double t_end = t0 + duration;
    memcpy(y, y0, sizeof y);
    memcpy(out, y, sizeof y);
    counts[0] = counts[1] = 0;
    int status = ST_OK;
    uint64_t k = 0;
    while (t < t_end) {
        const double step = fmin(dt, t_end - t);
        l->k = k;
        ++k;
        if (integrator == 0) {
            list_rk4_step(l, y, step);
            ++counts[0];
            int finite = 1;
            for (int c = 0; c < 6; ++c) finite &= isfinite(y[c]) ? 1 : 0;
            if (status == ST_OK && !finite) status = ST_NON_FINITE;
        } else {
            const int st = list_dp87_step(l, y, step, &hCur, counts);
            if (st == ST_STOPPED) {
                uint64_t K = 0;
                azn_times(t0, duration, dt, NULL, UINT64_MAX, &K);
                memset(out + k * 6, 0, (K - k) * 6 * sizeof(double));
                return ST_STOPPED;
            }
            if (st == ST_SUBSTEP_LIMIT) status = ST_SUBSTEP_LIMIT;
        }
        t += step;
        memcpy(out + k * 6, y, sizeof y);
    }
    return status;
}

typedef struct {
    const double *states;
    const ListModel *models;
    int count, integrator, k7Factor;
    double t0, duration, dt, rtol, atol;
    size_t n, samples;
    double *out;
    uint8_t *status;
    uint64_t *counts;
    size_t next;
    pthread_mutex_t lock;
} ListBatch;

static void *list_worker(void *arg) {
    ListBatch *b = arg;
    for (;;) {
        pthread_mutex_lock(&b->lock);
        const size_t i = b->next++;
        pthread_mutex_unlock(&b->lock);
        if (i >= b->n) return NULL;
        ListCtx l = {b->models, b->count, i, 0, b->rtol, b->atol, b->k7Factor};
        b->status[i] = (uint8_t)list_propagate_one(&l, b->integrator, b->states + i * 6, b->t0, b->duration, b->dt,
                                                   b->out + i * b->samples * 6, b->counts + i * 2);
    }
}

/* Propagator.propagate (Propagator.zig:22-48) of n states under a model list, per-state coefficients and position
 * tables as the descriptors name them: out[n][samples][6], status[n], counts[n][2].  Returns the sample count, 0 on a
 * bad loop. */
uint64_t azn_propagate_models(const double *states, size_t n, double t0, double duration, double dt,
                              const ListModel *models, int count, int integrator, double rtol, double atol,
                              int k7Factor, double *out, uint8_t *status, uint64_t *counts, int threads) {
    uint64_t samples = 0;
    if (azn_times(t0, duration, dt, NULL, UINT64_MAX, &samples) != 0) return 0;
    ListBatch b = {states, models, count, integrator, k7Factor, t0, duration, dt, rtol, atol, n, samples, out, status,
                   counts, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t tid[256];
    int started = 0;
    for (int k = 1; k < threads; ++k)
        if (pthread_create(&tid[started], NULL, list_worker, &b) == 0) ++started;
    list_worker(&b);
    for (int k = 0; k < started; ++k) pthread_join(tid[k], NULL);
    return samples;
}
