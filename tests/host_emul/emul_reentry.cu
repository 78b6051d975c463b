// TEST INFRASTRUCTURE ONLY: runs K19 (az_reentry.cuh, __host__ __device__) on the CPU with the warps of reentry_kernel /
// reentry_deep_kernel (az_reentry.cu) restated serially: each request's nominal, then its samples, one after the other.
// emul_reentry is astroz_cuda_reentry_device's definition on host buffers; emul_reentry_density, _height, _accel,
// _locate, _integrate and _draw expose the pieces, with the call's scalars (J2, the atmosphere's rotation) as
// parameters.  Not part of the shipped library; nothing in astroz_b200/ references it.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#include "az_reentry.cuh"

using namespace az;

namespace {
ReentryCall call_of(double hi, double horizon_s, double step, double scale, double sigma, double omega, double mu,
                    double rEq, double j2) {
    return ReentryCall{hi, horizon_s, step, scale, sigma, omega, mu, rEq, j2};
}

void store(const ReentryOut &o, double *w) {
    const double v[15] = {o.dt, o.lat, o.lon, o.speed, o.fpa, o.y[0], o.y[1], o.y[2], o.y[3], o.y[4], o.y[5],
                          (double)o.counts[0], (double)o.counts[1], (double)o.status, 0.0};
    std::memcpy(w, v, sizeof v);
}
}  // namespace

extern "C" void emul_reentry_density(const double *h, uint32_t n, double *rho) {
    for (uint32_t i = 0; i < n; ++i) rho[i] = reentry_density(h[i]);
}

extern "C" void emul_reentry_height(const double *r, uint32_t n, double *h) {
    for (uint32_t i = 0; i < n; ++i) h[i] = reentry_height(r[3 * i], r[3 * i + 1], r[3 * i + 2]);
}

// acc[n][3] of states s[n][6] under ReentryForces{mu, rEq, j2, omega, bf}
extern "C" void emul_reentry_accel(const double *s, uint32_t n, double mu, double rEq, double j2, double omega,
                                   double bf, double *acc) {
    const ReentryForces F{mu, rEq, j2, omega, bf};
    for (uint32_t i = 0; i < n; ++i) F(s + 6 * i, acc + 3 * i);
}

// the crossing between end states a and b over dt seconds: s, or -1 when there is none
extern "C" double emul_reentry_locate(const double *a, const double *b, double dt, double hi) {
    double A[6], Bv[6], s;
    std::memcpy(A, a, sizeof A);
    std::memcpy(Bv, b, sizeof Bv);
    return reentry_locate(A, Bv, dt, hi, s) ? s : -1.0;
}

// the Hermite position and velocity at s
extern "C" void emul_reentry_hermite(const double *a, const double *b, double dt, double s, double *q) {
    double A[6], Bv[6], Q[6];
    std::memcpy(A, a, sizeof A);
    std::memcpy(Bv, b, sizeof Bv);
    reentry_hermite(A, Bv, dt, s, Q);
    std::memcpy(q, Q, sizeof Q);
}

// One trajectory from y0 with every scalar given: out[15] = dt, lat, lon, speed, fpa, state[6], accepted, rejected,
// status, 0
extern "C" void emul_reentry_integrate(const double *y0, double epochJd, double B, double f, double hi,
                                       double horizon_s, double step, double scale, double omega, double mu,
                                       double rEq, double j2, double *out) {
    const ReentryCall c = call_of(hi, horizon_s, step, scale, 0.0, omega, mu, rEq, j2);
    double Y[6], y[6];
    std::memcpy(Y, y0, sizeof Y);
    ReentryOut o;
    reentry_integrate(Y, epochJd, B, f, c, y, o);
    store(o, out);
}

// The drawn variables, B, f and epoch state of samples k[0 .. n) of one row (the request's status returned):
// x[n][7], B[n], f[n], y[n][6], built[n]
extern "C" int emul_reentry_draw(const double *el, int model, const double *P, const double *ballistic, double sigma,
                                 uint64_t seed, const uint64_t *k, uint32_t n, int grav, double *x, double *B,
                                 double *f, double *y, uint8_t *built) {
    double e[8];
    std::memcpy(e, el, sizeof e);
    ReentryRow R;
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const uint8_t st = reentry_row(e, P, model, gr, ballistic != nullptr, ballistic ? *ballistic : 0.0, R);
    if (st != kReOk) return st;
    double cols[kSgp4Cols];
    Sdp4Sat set;
    for (uint32_t i = 0; i < n; ++i) {
        double xs[kFitVars], ys[6];
        reentry_params(R, true, seed, k[i], sigma, xs, B[i], f[i]);
        std::memcpy(x + (size_t)kFitVars * i, xs, sizeof xs);
        built[i] = model ? reentry_epoch_deep(xs, R.epoch, gr, g, set, ys) : reentry_epoch_near(xs, R.epoch, gr, g, cols, ys);
        std::memcpy(y + (size_t)6 * i, ys, sizeof ys);
    }
    return st;
}

extern "C" int emul_reentry(const double *elements, uint32_t n, int grav, const double *covariance,
                            const uint8_t *model, const uint32_t *rows, const double *ballistic,
                            const uint64_t *samples, const uint64_t *first, const uint64_t *seed, uint32_t m,
                            double hi, double horizon_days, double step, double scale, double sigma, uint32_t record,
                            double *out, double *states, uint8_t *nominalStatus, uint64_t *counts, double *sampleOut,
                            uint8_t *status, int threads) {
    const Gravity gr = gravity(grav);
    const GravConsts g = grav_consts(gr);
    const ReentryCall c = call_of(hi, horizon_days * 86400.0, step, scale, sigma, kReEarthOmega, gr.mu,
                                  gr.radiusEarthKm, gr.j2);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    auto one = [&](uint32_t i) {
        double cols[kSgp4Cols];
        Sdp4Sat set;
        uint64_t *cnt = counts + (size_t)i * kReCountWords;
        cnt[0] = cnt[1] = cnt[2] = 0;
        double *sw = sampleOut + (size_t)i * record * kReSampleWords;
        for (size_t q = 0; q < (size_t)record * kReSampleWords; ++q) sw[q] = nan;
        double *rec = out + (size_t)i * kReRecordWords;
        ReentryRow R;
        R.B = nan;
        R.model = 0;
        R.status = kReBadRow;
        if (rows[i] < n) {
            double el[8];
            for (int q = 0; q < 8; ++q) el[q] = elements[(size_t)q * n + rows[i]];
            const int md = model ? model[rows[i]] : 0;
            reentry_row(el, covariance + (size_t)rows[i] * kFitN, md, gr, ballistic != nullptr,
                        ballistic ? ballistic[i] : 0.0, R);
        }
        status[i] = (uint8_t)R.status;
        if (R.status != kReOk) {
            for (int q = 0; q < 5; ++q) rec[q] = nan;
            rec[5] = R.B;
            rec[6] = rec[7] = 0.0;
            if (states)
                for (int q = 0; q < 6; ++q) states[(size_t)i * 6 + q] = nan;
            nominalStatus[i] = kReTrajInitFailed;
            return;
        }
        const uint64_t f0 = first ? first[i] : 0, sd = seed ? seed[i] : 0;
        for (uint64_t j = 0; j <= samples[i]; ++j) {   // j = 0: the nominal; j >= 1: sample first + j - 1
            const bool sample = j > 0;
            double x[kFitVars], B, f, y0[6], y[6];
            reentry_params(R, sample, sd, f0 + j - 1, sigma, x, B, f);
            const bool built = R.model ? reentry_epoch_deep(x, R.epoch, gr, g, set, y0)
                                       : reentry_epoch_near(x, R.epoch, gr, g, cols, y0);
            ReentryOut o;
            o.counts[0] = o.counts[1] = 0;
            if (built) reentry_integrate(y0, R.epoch, B, f, c, y, o);
            else reentry_fail(o, kReTrajInitFailed);
            if (!sample) {
                const double w[8] = {o.dt, o.lat, o.lon, o.speed, o.fpa, B, (double)o.counts[0], (double)o.counts[1]};
                std::memcpy(rec, w, sizeof w);
                if (states) std::memcpy(states + (size_t)i * 6, o.y, sizeof o.y);
                nominalStatus[i] = o.status;
                continue;
            }
            cnt[o.status == kReReentered ? 0 : o.status == kReAbove ? 1 : 2] += 1;
            if (j - 1 < record) {
                double *d = sw + (j - 1) * kReSampleWords;
                d[0] = o.dt;
                d[1] = o.lat;
                d[2] = o.lon;
                d[3] = (double)(o.counts[0] + o.counts[1]);
            }
        }
    };
    // requests cyclically over the threads: every request's words are its own
    std::vector<std::thread> pool;
    const int T = threads > 1 ? threads : 1;
    for (int t = 0; t < T; ++t)
        pool.emplace_back([&, t] {
            for (uint32_t i = (uint32_t)t; i < m; i += (uint32_t)T) one(i);
        });
    for (auto &th : pool) th.join();
    return 0;
}
