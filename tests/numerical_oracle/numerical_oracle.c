/* TEST INFRASTRUCTURE ONLY: scalar C restatement of the reference's numerical propagation, the yardstick K7
 * (astroz_b200/csrc/az_numerical.cuh) is checked against.  Built with -ffp-contract=off, like Zig's strict float mode.
 * Every function names the reference lines it restates (src/propagators/..., bindings/python/src/propagator.zig).
 * Where the reference never returns (a DP87 step rejected at hMin is retried with the same state and step forever), this
 * stops the state under the same rule as K7, so that no test can hang. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

enum { FORCE_J2 = 1, FORCE_DRAG = 2 };
enum { ST_OK = 0, ST_STOPPED = 1, ST_SUBSTEP_LIMIT = 2, ST_NON_FINITE = 3 };

typedef struct {
    double mu, j2, rEq, cd, area, mass, rtol, atol;
    int forces;
    int k7Factor; /* 1: errNorm^(-1/8) as K7 forms it (three square roots) instead of the reference's pow */
} Model;

/* Integrator.zig:73-138, entered from the published rationals */
static const double C_[13] = {0.0, 1.0 / 18, 1.0 / 12, 1.0 / 8, 5.0 / 16, 3.0 / 8, 59.0 / 400, 93.0 / 200,
                              5490023248.0 / 9719169821.0, 13.0 / 20, 1201146811.0 / 1299019798.0, 1.0, 1.0};
static double A_[13][12];
static const double B8_[13] = {14005451.0 / 335480064.0, 0, 0, 0, 0, -59238493.0 / 1068277825.0,
                               181606767.0 / 758867731.0, 561292985.0 / 797845732.0, -1041891430.0 / 1371343529.0,
                               760417239.0 / 1151165299.0, 118820643.0 / 751138087.0, -528747749.0 / 2220607170.0,
                               1.0 / 4};
static const double B7_[13] = {13451932.0 / 455176623.0, 0, 0, 0, 0, -808719846.0 / 976000145.0,
                               1757004468.0 / 5645159321.0, 656045339.0 / 265891186.0, -3867574721.0 / 1518517206.0,
                               465885868.0 / 322736535.0, 53011238.0 / 667516719.0, 2.0 / 45, 0};
/* rows of a as (numerator, denominator) pairs over the stages j < i; zero entries have numerator 0 */
static const double AQ_[13][12][2] = {
    {{0, 1}},
    {{1, 18}},
    {{1, 48}, {1, 16}},
    {{1, 32}, {0, 1}, {3, 32}},
    {{5, 16}, {0, 1}, {-75, 64}, {75, 64}},
    {{3, 80}, {0, 1}, {0, 1}, {3, 16}, {3, 20}},
    {{29443841, 614563906}, {0, 1}, {0, 1}, {77736538, 692538347}, {-28693883, 1125000000}, {23124283, 1800000000}},
    {{16016141, 946692911}, {0, 1}, {0, 1}, {61564180, 158732637}, {22789713, 633445777}, {545815736, 2771057229},
     {-180193667, 1043307555}},
    {{39632708, 573591083}, {0, 1}, {0, 1}, {-433636366, 683701615}, {-421739975, 2616292301},
     {100302831, 723423059}, {790204164, 839813087}, {800635310, 3783071287}},
    {{246121993, 1340847787}, {0, 1}, {0, 1}, {-37695042795, 15268766246}, {-309121744, 1061227803},
     {-12992083, 490766935}, {6005943493, 2108947869}, {393006217, 1396673457}, {123872331, 1001029789}},
    {{-1028468189, 846180014}, {0, 1}, {0, 1}, {8478235783, 508512852}, {1311729495, 1432422823},
     {-10304129995, 1701304382}, {-48777925059, 3047939560}, {15336726248, 1032824649}, {-45442868181, 3398467696},
     {3065993473, 597172653}},
    {{185892177, 718116043}, {0, 1}, {0, 1}, {-3185094517, 667107341}, {-477755414, 1098053517},
     {-703635378, 230739211}, {5731566787, 1027545527}, {5232866602, 850066563}, {-4093664535, 808688257},
     {3962137247, 1805957418}, {65686358, 487910083}},
    {{403863854, 491063109}, {0, 1}, {0, 1}, {-5068492393, 434740067}, {-411421997, 543043805},
     {652783627, 914296604}, {11173962825, 925320556}, {-13158990841, 6184727034}, {3936647629, 1978049680},
     {-160528059, 685178525}, {248638103, 1413531060}, {0, 1}},
};
static pthread_once_t tableau_once = PTHREAD_ONCE_INIT;
static void tableau_init(void) {
    for (int i = 0; i < 13; ++i)
        for (int j = 0; j < 12; ++j) A_[i][j] = (j < i) ? AQ_[i][j][0] / AQ_[i][j][1] : 0.0;
}

/* c[13], a[13][12], b8[13], b7[13] */
void azn_tableau(double *c, double *a, double *b8, double *b7) {
    pthread_once(&tableau_once, tableau_init);
    memcpy(c, C_, sizeof C_);
    memcpy(a, A_, sizeof A_);
    memcpy(b8, B8_, sizeof B8_);
    memcpy(b7, B7_, sizeof B7_);
}

/* TwoBody (ForceModel.zig:49-55), J2 (:67-79), Drag (:95-110) with rho0 1.225, H 7.249 (constants.zig:163-164) and the
 * binding's 1500 km cutoff (propagator.zig:11), summed by Composite (:365-374) when more than one is on
 * (propagator.zig:119-146) */
static void acceleration(const Model *m, const double s[6], double out[3]) {
    const double x = s[0], y = s[1], z = s[2];
    double tb[3];
    {
        const double r = sqrt(x * x + y * y + z * z);
        const double factor = -m->mu / (r * r * r);
        tb[0] = factor * x, tb[1] = factor * y, tb[2] = factor * z;
    }
    if (!m->forces) {
        memcpy(out, tb, sizeof tb);
        return;
    }
    double total[3] = {0, 0, 0};
    for (int c = 0; c < 3; ++c) total[c] += tb[c];
    if (m->forces & FORCE_J2) {
        const double r2 = x * x + y * y + z * z;
        const double r = sqrt(r2);
        const double factor = -1.5 * m->j2 * m->mu * m->rEq * m->rEq / (r2 * r2 * r);
        const double z2R2 = (z * z) / r2;
        const double a[3] = {factor * x * (5.0 * z2R2 - 1.0), factor * y * (5.0 * z2R2 - 1.0),
                             factor * z * (5.0 * z2R2 - 3.0)};
        for (int c = 0; c < 3; ++c) total[c] += a[c];
    }
    if (m->forces & FORCE_DRAG) {
        double a[3] = {0, 0, 0};
        const double r = sqrt(x * x + y * y + z * z);
        const double altitude = r - m->rEq;
        if (!(altitude > 1500.0)) {
            const double vx = s[3], vy = s[4], vz = s[5];
            const double v = sqrt(vx * vx + vy * vy + vz * vz);
            if (!(v < 1e-10)) {
                const double rho = 1.225 * exp(-altitude / 7.249);
                const double factor = -0.5 * m->cd * m->area * rho * v * 1e3 / m->mass;
                a[0] = factor * vx / v, a[1] = factor * vy / v, a[2] = factor * vz / v;
            }
        }
        for (int c = 0; c < 3; ++c) total[c] += a[c];
    }
    memcpy(out, total, sizeof total);
}

/* derivative (Integrator.zig:47-50, :261-264) */
static void derivative(const Model *m, const double s[6], double k[6]) {
    double a[3];
    acceleration(m, s, a);
    k[0] = s[3], k[1] = s[4], k[2] = s[5], k[3] = a[0], k[4] = a[1], k[5] = a[2];
}

/* Rk4.step (Integrator.zig:28-45) */
static void rk4_step(const Model *m, double y[6], double dt) {
    double k1[6], k2[6], k3[6], k4[6], s[6];
    derivative(m, y, k1);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k1[c] * (0.5 * dt);
    derivative(m, s, k2);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k2[c] * (0.5 * dt);
    derivative(m, s, k3);
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k3[c] * dt;
    derivative(m, s, k4);
    const double factor = dt / 6.0;
    for (int c = 0; c < 6; ++c) y[c] = y[c] + factor * (k1[c] + 2.0 * k2[c] + 2.0 * k3[c] + k4[c]);
}

/* DormandPrince87.adaptiveStep (Integrator.zig:190-259): y8 and errNorm of one attempt, *hNew */
static double dp87_attempt(const Model *m, const double y[6], double h, double y8[6], double *hNew) {
    double k[13][6], y7[6];
    derivative(m, y, k[0]);
    for (int i = 1; i < 13; ++i) {
        double ys[6];
        memcpy(ys, y, sizeof ys);
        for (int j = 0; j < i; ++j)
            if (A_[i][j] != 0)
                for (int c = 0; c < 6; ++c) ys[c] = ys[c] + (A_[i][j] * h) * k[j][c];
        derivative(m, ys, k[i]);
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
        const double scale = m->atol + m->rtol * fmax(fabs(y[c]), fabs(y8[c]));
        const double se = (y8[c] - y7[c]) / scale;
        errNorm += se * se;
    }
    errNorm = sqrt(errNorm / 6.0);
    double hn;
    if (errNorm < 1e-10) {
        hn = h * 5.0;
    } else {
        const double factor = m->k7Factor ? 0.9 * sqrt(sqrt(sqrt(1.0 / errNorm))) : 0.9 * pow(1.0 / errNorm, 1.0 / 8.0);
        hn = h * fmin(5.0, fmax(0.1, factor)); /* fmin / fmax ignore a NaN, as Zig's @min / @max */
    }
    hn = fmin(hn, 3600.0);
    *hNew = fmax(hn, 0.001);
    return errNorm;
}

/* DormandPrince87.step (Integrator.zig:154-182) over one output interval; hCur carries across intervals */
static int dp87_step(const Model *m, double y[6], double dt, double *hCur, uint64_t counts[2]) {
    double remaining = dt, h = fmin(*hCur, remaining);
    uint32_t substeps = 0;
    while (remaining > 1e-14 && substeps < 10000) {
        h = fmin(h, remaining);
        h = fmax(h, 0.001);
        double y8[6], hNew;
        const double errNorm = dp87_attempt(m, y, h, y8, &hNew);
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

/* Propagator.propagate (Propagator.zig:22-48): *count = samples; times (nullable) receives them.  Returns -1 for a loop
 * that would not end (t + step == t) or more than max_samples samples. */
int azn_times(double t0, double duration, double dt, double *times, uint64_t max_samples, uint64_t *count) {
    double t = t0;
    const double t_end = t0 + duration;
    uint64_t k = 0;
    if (times) times[0] = t;
    while (t < t_end) {
        const double step = fmin(dt, t_end - t);
        if (t + step == t || k + 2 > max_samples) return -1;
        t += step;
        ++k;
        if (times) times[k] = t;
    }
    *count = k + 1;
    return 0;
}

/* One state: out[(K + 1) * 6], counts[2]; returns the status byte */
static int propagate_one(const Model *m, int integrator, const double y0[6], double t0, double duration, double dt,
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
        ++k;
        if (integrator == 0) {
            rk4_step(m, y, step);
            ++counts[0];
            int finite = 1;
            for (int c = 0; c < 6; ++c) finite &= isfinite(y[c]) ? 1 : 0;
            if (status == ST_OK && !finite) status = ST_NON_FINITE;
        } else {
            const int st = dp87_step(m, y, step, &hCur, counts);
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
    const double *states, *cd, *area, *mass, *par;
    double t0, duration, dt;
    int forces, integrator;
    size_t n, samples;
    double *out;
    uint8_t *status;
    uint64_t *counts;
    size_t next;
    pthread_mutex_t lock;
} Batch;

static void run_state(Batch *b, size_t i) {
    Model m = {b->par[0], b->par[1], b->par[2], 0, 0, 0, b->par[3], b->par[4], b->forces, b->par[5] != 0.0};
    if (b->forces & FORCE_DRAG) m.cd = b->cd[i], m.area = b->area[i], m.mass = b->mass[i];
    b->status[i] = (uint8_t)propagate_one(&m, b->integrator, b->states + i * 6, b->t0, b->duration, b->dt,
                                          b->out + i * b->samples * 6, b->counts + i * 2);
}

static void *worker(void *arg) {
    Batch *b = arg;
    for (;;) {
        pthread_mutex_lock(&b->lock);
        const size_t i = b->next++;
        pthread_mutex_unlock(&b->lock);
        if (i >= b->n) return NULL;
        run_state(b, i);
    }
}

/* n states (the same arithmetic per state on every thread count): par = {mu, j2, r_eq, rtol, atol, k7Factor}; cd / area / mass
 * per state when drag is on; out[n][samples][6], status[n], counts[n][2].  Returns the sample count, 0 on a bad loop. */
uint64_t azn_propagate_batch(const double *states, size_t n, double t0, double duration, double dt, const double *par,
                             int forces, const double *cd, const double *area, const double *mass, int integrator,
                             double *out, uint8_t *status, uint64_t *counts, int threads) {
    uint64_t samples = 0;
    if (azn_times(t0, duration, dt, NULL, UINT64_MAX, &samples) != 0) return 0;
    Batch b = {states, cd, area, mass, par, t0, duration, dt, forces, integrator, n, samples, out, status, counts, 0,
               PTHREAD_MUTEX_INITIALIZER};
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t tid[256];
    int started = 0;
    for (int k = 1; k < threads; ++k)
        if (pthread_create(&tid[started], NULL, worker, &b) == 0) ++started;
    worker(&b);
    for (int k = 0; k < started; ++k) pthread_join(tid[k], NULL);
    return samples;
}
