/* TEST INFRASTRUCTURE ONLY: scalar C restatement of the reference's impulsive-maneuver loop, Spacecraft.propagate
 * (src/Spacecraft.zig:172-323), over a model list -- the yardstick the K7 maneuver core (maneuver_with in
 * astroz_b200/csrc/az_numerical.cuh) is checked against.  Built with -ffp-contract=off.  It includes
 * numerical_oracle_models.c for the model lists and its RK4 / DP87 steps (list_rk4_step, list_dp87_step), and states
 * the loop and the burns from the reference lines each function names.
 *
 * k7Forms = 0: pow(r, 3), pow(x, 2/3) and errNorm^(-1/8) through the C library's pow.  k7Forms = 1: the forms of the
 * device cores -- r * (r * r) and exp((2/3 - 1) log x) * x, which is how Zig's std.math.pow evaluates those exponents,
 * and errNorm^(-1/8) as three square roots (k7_step_factor).  sin, cos, exp and log are the C library's in both. */
#include "numerical_oracle_models.c"

typedef struct {
    double time;
    int32_t kind;
    uint32_t reserved;
    double p[3];
} Impulse; /* astroz_impulse_t */
enum { IMP_ABSOLUTE, IMP_PROGRADE, IMP_PHASE, IMP_PLANE_CHANGE };
enum { ST_ABNORMAL = 4, ST_TRUNCATED = 5 };
#define MAX_SAMPLES 0xfffffffeull
static const double PI = 3.14159265358979323846;

static double pow3(int k7, double x) { return k7 ? x * (x * x) : pow(x, 3.0); }
static double pow_two_thirds(int k7, double x) { return k7 ? exp((2.0 / 3.0 - 1.0) * log(x)) * x : pow(x, 2.0 / 3.0); }

/* calculations.posMag / velMag (calculations.zig:329-336) */
static double pos_mag(const double y[6]) { return sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]); }
static double vel_mag(const double y[6]) { return sqrt(y[3] * y[3] + y[4] * y[4] + y[5] * y[5]); }
/* calculations.impulse (calculations.zig:480-485) */
static void impulse(double y[6], const double dv[3]) {
    y[3] = y[3] + dv[0], y[4] = y[4] + dv[1], y[5] = y[5] + dv[2];
}
/* progradeVec (Spacecraft.zig:260-263) */
static void prograde_vec(const double y[6], double dvMag, double dv[3]) {
    const double vMag = vel_mag(y);
    dv[0] = y[3] / vMag * dvMag, dv[1] = y[4] / vMag * dvMag, dv[2] = y[5] / vMag * dvMag;
}
/* calculatePhaseChange (Spacecraft.zig:310-323) */
static double phase_change(int k7, double mu, double radius, double phaseAngle, double transferOrbits) {
    const double vCircular = sqrt(mu / radius);
    const double period = 2.0 * PI * sqrt(pow3(k7, radius) / mu);
    const double deltaT = phaseAngle * period / (2.0 * PI * transferOrbits);
    const double transferPeriod = period + deltaT;
    const double aTransfer = pow_two_thirds(k7, transferPeriod * sqrt(mu) / (2.0 * PI));
    const double vTransfer = sqrt(mu * (2.0 / radius - 1.0 / aTransfer));
    return vTransfer - vCircular;
}
/* applyPlaneChange (Spacecraft.zig:272-307) */
static void plane_change(double y[6], double deltaInclination, double deltaRaan) {
    const double vMag = vel_mag(y);
    const double totalAngle = sqrt(deltaInclination * deltaInclination + deltaRaan * deltaRaan);
    if (totalAngle < 1e-10) return;
    const double dvMag = 2.0 * vMag * sin(totalAngle / 2.0);
    const double r[3] = {y[0], y[1], y[2]}, v[3] = {y[3], y[4], y[5]};
    const double h[3] = {r[1] * v[2] - r[2] * v[1], r[2] * v[0] - r[0] * v[2], r[0] * v[1] - r[1] * v[0]};
    const double hMag = sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    const double dv[3] = {h[0] / hMag * dvMag * sin(deltaInclination), h[1] / hMag * dvMag * sin(deltaInclination),
                          h[2] / hMag * dvMag * cos(deltaInclination)};
    impulse(y, dv);
}

typedef struct {
    ListCtx *l;
    int integrator;
    double hCur; /* DP87's step size, carried through every step */
    uint64_t *counts;
    int status; /* sticky ST_SUBSTEP_LIMIT / ST_NON_FINITE */
    double *times, *out;
    uint64_t cap, count;
} Run;

/* integrator.step(y, t, dt, force); 0 when the reference would never return */
static int step(Run *u, double y[6], double dt) {
    if (u->integrator == 0) {
        list_rk4_step(u->l, y, dt);
        ++u->counts[0];
        int finite = 1;
        for (int c = 0; c < 6; ++c) finite &= isfinite(y[c]) ? 1 : 0;
        if (u->status == ST_OK && !finite) u->status = ST_NON_FINITE;
        return 1;
    }
    const int st = list_dp87_step(u->l, y, dt, &u->hCur, u->counts);
    if (st == ST_SUBSTEP_LIMIT) u->status = ST_SUBSTEP_LIMIT;
    return st != ST_STOPPED;
}
/* orbitPredictions.append; 0 past MAX_SAMPLES */
static int append(Run *u, double t, const double y[6]) {
    if (u->count == MAX_SAMPLES) return 0;
    if (u->count < u->cap) {
        u->times[u->count] = t;
        memcpy(u->out + u->count * 6, y, 6 * sizeof(double));
    }
    ++u->count;
    return 1;
}

/* Spacecraft.propagate (Spacecraft.zig:172-270) from y0 at t0 to tf with step h and impulses imp[m]; applyImpulse
 * (:226-258) for each burn.  Returns the status byte; u->count samples, the first u->cap written, the rest of the row
 * zero. */
static int maneuver_one(Run *u, const double y0[6], double t0, double tf, double h, double mu, const Impulse *imp,
                        size_t m, int k7) {
    double y[6], t = t0;
    memcpy(y, y0, sizeof y);
    int stopped = 0, abnormal = 0;
    append(u, t, y);
    size_t impulseIndex = 0;
    while (t < tf && !stopped) {
        while (impulseIndex < m && imp[impulseIndex].time <= t + h) {
            const Impulse *b = &imp[impulseIndex];
            const double dt = b->time - t;
            if (dt > 0) {
                if (!step(u, y, dt)) { stopped = 1; break; }
                t += dt;
                if (!append(u, t, y)) { stopped = 1; break; }
            }
            if (b->kind == IMP_ABSOLUTE) {
                impulse(y, b->p);
            } else if (b->kind == IMP_PROGRADE) {
                double dv[3];
                prograde_vec(y, b->p[0], dv);
                impulse(y, dv);
            } else if (b->kind == IMP_PHASE) {
                const double r = pos_mag(y);
                const double dvMag = phase_change(k7, mu, r, b->p[0], b->p[1]);
                double dv[3];
                prograde_vec(y, dvMag, dv);
                impulse(y, dv);
                const double period = 2 * PI * sqrt(pow3(k7, r) / mu);
                const double tEnd = t + period * b->p[1];
                while (t < tEnd) {
                    if (!step(u, y, h) || !append(u, t + h, y)) { stopped = 1; break; }
                    t += h;
                }
                if (stopped) break;
                const double back[3] = {-dv[0], -dv[1], -dv[2]};
                impulse(y, back);
            } else {
                plane_change(y, b->p[0], b->p[1]);
            }
            if (!append(u, t, y)) { stopped = 1; break; }
            impulseIndex += 1;
        }
        if (stopped) break;
        const double stepSize = fmin(h, tf - t);
        if (!step(u, y, stepSize)) { stopped = 1; break; }
        t += stepSize;
        if (!append(u, t, y)) { stopped = 1; break; }
        const double r = pos_mag(y), v = vel_mag(y);
        const double energy = 0.5 * v * v - mu / r;
        if (energy > 0 || isnan(energy) || r > 100000) {
            abnormal = 1;
            break;
        }
    }
    for (uint64_t j = u->count; j < u->cap; ++j) {
        u->times[j] = 0.0;
        memset(u->out + j * 6, 0, 6 * sizeof(double));
    }
    if (u->count > u->cap) return ST_TRUNCATED;
    if (stopped) return ST_STOPPED;
    if (u->status != ST_OK) return u->status;
    return abnormal ? ST_ABNORMAL : ST_OK;
}

typedef struct {
    const double *states;
    const ListModel *models;
    int count, integrator, k7;
    double t0, tf, h, mu, rtol, atol;
    const uint32_t *offsets;
    const Impulse *imp;
    size_t n, cap;
    double *times, *out;
    uint64_t *nSamples, *counts;
    uint8_t *status;
    size_t next;
    pthread_mutex_t lock;
} ManeuverBatch;

static void *maneuver_worker(void *arg) {
    ManeuverBatch *b = arg;
    for (;;) {
        pthread_mutex_lock(&b->lock);
        const size_t i = b->next++;
        pthread_mutex_unlock(&b->lock);
        if (i >= b->n) return NULL;
        ListCtx l = {b->models, b->count, i, 0, b->rtol, b->atol, b->k7};
        uint64_t *counts = b->counts + 2 * i;
        counts[0] = counts[1] = 0;
        Run u = {&l, b->integrator, 60.0, counts, ST_OK, b->times + i * b->cap, b->out + i * b->cap * 6, b->cap, 0};
        b->status[i] = (uint8_t)maneuver_one(&u, b->states + 6 * i, b->t0, b->tf, b->h, b->mu, b->imp + b->offsets[i],
                                             b->offsets[i + 1] - b->offsets[i], b->k7);
        b->nSamples[i] = u.count;
    }
}

/* Spacecraft.propagate of n states, state i with impulses imp[offsets[i] .. offsets[i + 1]): times[n][cap],
 * out[n][cap][6], nSamples[n], status[n], counts[n][2]. */
void azn_propagate_maneuvers(const double *states, size_t n, double t0, double duration, double h, double mu,
                             const uint32_t *offsets, const Impulse *imp, const ListModel *models, int count,
                             int integrator, double rtol, double atol, int k7Forms, size_t cap, double *times,
                             double *out, uint64_t *nSamples, uint8_t *status, uint64_t *counts, int threads) {
    pthread_once(&tableau_once, tableau_init);
    ManeuverBatch b = {states, models, count, integrator, k7Forms, t0, t0 + duration, h, mu, rtol, atol, offsets, imp,
                       n, cap, times, out, nSamples, counts, status, 0, PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t tid[256];
    int started = 0;
    for (int k = 1; k < threads; ++k)
        if (pthread_create(&tid[started], NULL, maneuver_worker, &b) == 0) ++started;
    maneuver_worker(&b);
    for (int k = 0; k < started; ++k) pthread_join(tid[k], NULL);
}

/* One burn of `kind` with parameters p applied to each of the states y[n][6] (a phasing burn: only its first, prograde
 * half): the restatement's arithmetic for tests that state the burns independently.  out[n][6]. */
void azn_apply_burn(const double *y, size_t n, int32_t kind, const double p[3], double mu, int k7Forms, double *out) {
    for (size_t i = 0; i < n; ++i) {
        double s[6], dv[3];
        memcpy(s, y + 6 * i, sizeof s);
        if (kind == IMP_ABSOLUTE) {
            impulse(s, p);
        } else if (kind == IMP_PROGRADE) {
            prograde_vec(s, p[0], dv);
            impulse(s, dv);
        } else if (kind == IMP_PHASE) {
            prograde_vec(s, phase_change(k7Forms, mu, pos_mag(s), p[0], p[1]), dv);
            impulse(s, dv);
        } else {
            plane_change(s, p[0], p[1]);
        }
        memcpy(out + 6 * i, s, sizeof s);
    }
}
