// az_reentry.cuh -- K19: reentry prediction of catalogue rows and their covariance draws.  __host__ __device__, so the
// kernels (az_reentry.cu) and the host emulation (tests/host_emul/emul_reentry.cu) run this source.
//
// Request i names a catalogue row (element columns, covariance P, model byte, as K11 / K14).  A trajectory starts at
// the row's epoch (tsince 0) from the TEME state of a set -- the row's own set for the nominal, K14's drawn primary set
// of sample k for a sample -- built under the row's model with the call's grav, and is integrated by K7's DP87
// (dp87_interval, K7's tolerances and step control) over intervals of `step` seconds until the first crossing of the
// interface height h_i or the horizon.
//   force     ReentryForces: two-body + textbook J2 (the call's grav), and drag quadratic in the speed relative to a
//             co-rotating atmosphere, a = -1/2 B f rho(h) |v_rel| v_rel 1e3 km/s^2, v_rel = v - w x r (w = 7.292115e-5
//             rad/s about TEME z), rho(h) = density_scale x Vallado's piecewise-exponential table (Fundamentals of
//             Astrodynamics and Applications, Table 8-4) at the WGS-84 geodetic height h of the TEME position
//             (ecef_to_geodetic; the ellipsoid is symmetric about z, so no GMST is needed).  None of K7's models change.
//   B         B_row = ballistic[i] [m^2/kg], or 12.741621 B* (B* = B rho0 / 2, rho0 = 0.15696615 kg m^-2 ER^-1); a
//             sample's B_k = B_row + 12.741621 (B*_k - B*_row).  B <= 0 or non-finite is NONPHYSICAL.
//   draws     sample k: K14's normals 0..6 (mc_row_normals of the primary) through K14's factor and draw, and normal 7
//             (block 3's second normal) as the density factor f_k = exp(sigma_rho z_7); the nominal has f = 1.
//   crossing  after each interval, the cubic Hermite of position over it from its end states: a crossing when the end
//             height is <= h_i, or when the radial velocity goes from - to + inside the interval and the Hermite's
//             minimum height (golden-section search) is <= h_i (a perigee dip).  The crossing is the root of height - h_i by
//             bisection to 2^-30 of the interval, its state the Hermite and its derivative there.  A start at or below
//             h_i crosses at dt = 0.
// A trajectory's words depend on its row's inputs, the call's scalars, the seed and k alone.
#pragma once

#include "az_conjunction_mc.cuh"
#include "az_kernels.cuh"
#include "az_numerical.cuh"

namespace az {

// the record words (dt, lat, lon, speed, flight-path angle, B, accepted, rejected), the sample words (dt, lat, lon,
// attempts), the count words (reentered, above, failed) and the state words
constexpr int kReRecordWords = 8, kReSampleWords = 4, kReCountWords = 3, kReStateWords = 6;
// trajectory statuses (ASTROZ_REENTRY_TRAJ_*)
constexpr uint8_t kReReentered = 0, kReAbove = 1, kReTrajInitFailed = 2, kReNonphysical = 3, kReStopped = 4;
// request statuses (ASTROZ_REENTRY_*)
constexpr uint8_t kReOk = 0, kReInitFailed = 1, kReNotPsd = 2, kReBadRow = 3;
constexpr double kReBstarToB = 12.741621;     // B = 2 B* / rho0 [m^2/kg per 1/ER]
constexpr double kReEarthOmega = 7.292115e-5;  // rad/s
constexpr double kReRtol = 1e-9, kReAtol = 1e-12;   // K7's default DP87 tolerances
constexpr int kReHalvings = 30;                // 2^-30 < 1e-9 of the interval
constexpr int kReGolden = 46;                  // golden-section steps: 0.618^46 < 1e-9
constexpr int kReBands = 28;

// Vallado Table 8-4: base height h0 [km], density rho0 [kg/m^3] and scale height H [km] of each band
struct ReAtmosphere {
    double h0[kReBands], rho0[kReBands], H[kReBands];
};
// clang-format off
#define AZ_RE_ATMOSPHERE {                                                                                             \
    {0, 25, 30, 40, 50, 60, 70, 80, 90, 100, 110, 120, 130, 140,                                                       \
     150, 180, 200, 250, 300, 350, 400, 450, 500, 600, 700, 800, 900, 1000},                                           \
    {1.225, 3.899e-2, 1.774e-2, 3.972e-3, 1.057e-3, 3.206e-4, 8.770e-5, 1.905e-5, 3.396e-6, 5.297e-7, 9.661e-8,       \
     2.438e-8, 8.484e-9, 3.845e-9, 2.070e-9, 5.464e-10, 2.789e-10, 7.248e-11, 2.418e-11, 9.518e-12, 3.725e-12,         \
     1.585e-12, 6.967e-13, 1.454e-13, 3.614e-14, 1.170e-14, 5.245e-15, 3.019e-15},                                     \
    {7.249, 6.349, 6.682, 7.554, 8.382, 7.714, 6.549, 5.799, 5.382, 5.877, 7.263, 9.473, 12.636, 16.149,               \
     22.523, 29.740, 37.105, 45.546, 53.628, 53.298, 58.515, 60.828, 63.822, 71.835, 88.667, 124.64, 181.05, 268.00}}
// clang-format on
static __constant__ ReAtmosphere kReAtmDev = AZ_RE_ATMOSPHERE;
static const ReAtmosphere kReAtmHost = AZ_RE_ATMOSPHERE;
#ifdef __CUDA_ARCH__
#define AZ_RE_ATM(field) (::az::kReAtmDev.field)
#else
#define AZ_RE_ATM(field) (::az::kReAtmHost.field)
#endif

// rho(h) [kg/m^3]: the band with the largest h0 <= h (band 0 below 0 km, the last band above 1000 km).  The band's
// index comes from unrolled compares against constant-bank words; its three words are then read once by that index.
AZ_HD double reentry_density(double h) {
    int j = 0;
#pragma unroll
    for (int b = 1; b < kReBands; ++b) j += h >= AZ_RE_ATM(h0[b]) ? 1 : 0;
    return AZ_RE_ATM(rho0[j]) * exp(-(h - AZ_RE_ATM(h0[j])) / AZ_RE_ATM(H[j]));
}

// The WGS-84 geodetic height [km] of a TEME (or ECEF) position: ecef_to_geodetic's
AZ_HD double reentry_height(double x, double y, double z) {
    ecef_to_geodetic(x, y, z);
    return z;
}

// The K7 force policy of K19 (file comment).  bf = B f density_scale [m^2/kg].
struct ReentryForces {
    double mu, rEq, j2, omega, bf;
    AZ_HD void interval(uint32_t) {}
    AZ_HD void operator()(const double s[6], double acc[3]) const {
        const double x = s[0], y = s[1], z = s[2];
        const double r2 = x * x + y * y + z * z;
        const double r = sqrt(r2);
        const double f = -mu / (r2 * r);
        const double q = 1.5 * j2 * mu * rEq * rEq / (r2 * r2 * r);   // 3/2 J2 mu R^2 / r^5
        const double zz = 5.0 * (z * z) / r2;
        const double vx = s[3] + omega * y, vy = s[4] - omega * x, vz = s[5];
        const double vr = sqrt(vx * vx + vy * vy + vz * vz);
        const double d = -0.5 * bf * reentry_density(reentry_height(x, y, z)) * vr * 1e3;
        acc[0] = f * x - q * x * (1.0 - zz) + d * vx;
        acc[1] = f * y - q * y * (1.0 - zz) + d * vy;
        acc[2] = f * z - q * z * (3.0 - zz) + d * vz;
    }
};

// The cubic Hermite of position over an interval of dt seconds from end states a and b, at s in [0, 1]: position and
// its time derivative into q
AZ_HD void reentry_hermite(const double (&a)[6], const double (&b)[6], double dt, double s, double (&q)[6]) {
    const double s2 = s * s, s3 = s2 * s;
    const double h00 = 2.0 * s3 - 3.0 * s2 + 1.0, h10 = s3 - 2.0 * s2 + s, h01 = 3.0 * s2 - 2.0 * s3, h11 = s3 - s2;
    const double d00 = 6.0 * s2 - 6.0 * s, d10 = 3.0 * s2 - 4.0 * s + 1.0, d11 = 3.0 * s2 - 2.0 * s;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        q[c] = h00 * a[c] + h10 * dt * a[3 + c] + h01 * b[c] + h11 * dt * b[3 + c];
        q[3 + c] = d00 * (a[c] - b[c]) / dt + d10 * a[3 + c] + d11 * b[3 + c];
    }
}

AZ_HD double reentry_hermite_height(const double (&a)[6], const double (&b)[6], double dt, double s) {
    double q[6];
    reentry_hermite(a, b, dt, s, q);
    return reentry_height(q[0], q[1], q[2]);
}

AZ_HD double reentry_rdot(const double (&q)[6]) { return q[0] * q[3] + q[1] * q[4] + q[2] * q[5]; }

// The crossing inside the interval from a (above h_i) to b, as s in (0, 1]; false when there is none.  When the
// radial velocity goes from - to + the interval holds a perigee, and the Hermite's minimum height is found by golden-
// section search over [0, 1] (kReGolden steps: 0.618^46 < 1e-9 of the interval).  The locator assumes at most one
// perigee per interval and a cubic that follows the arc: intervals well below a quarter of the orbital period (the
// default 60 s; step_s is refused above 3600 s, a fifth of the shortest orbit that reaches 80 km).
AZ_HD bool reentry_locate(const double (&a)[6], const double (&b)[6], double dt, double hi, double &s) {
    double up = 1.0;
    bool cross = false;
    if (reentry_rdot(a) < 0.0 && reentry_rdot(b) > 0.0) {   // a perigee inside: the Hermite's minimum height
        constexpr double g = 0.38196601125010515;           // (3 - sqrt 5) / 2
        double lo = 0.0, top = 1.0;
        double x1 = lo + g * (top - lo), x2 = top - g * (top - lo);
        double f1 = reentry_hermite_height(a, b, dt, x1), f2 = reentry_hermite_height(a, b, dt, x2);
        for (int k = 0; k < kReGolden; ++k) {
            if (f1 <= f2) {
                top = x2, x2 = x1, f2 = f1;
                x1 = lo + g * (top - lo);
                f1 = reentry_hermite_height(a, b, dt, x1);
            } else {
                lo = x1, x1 = x2, f1 = f2;
                x2 = top - g * (top - lo);
                f2 = reentry_hermite_height(a, b, dt, x2);
            }
        }
        const double sm = f1 <= f2 ? x1 : x2;
        if ((f1 <= f2 ? f1 : f2) <= hi) {
            up = sm;
            cross = true;
        }
    }
    if (!cross && !(reentry_height(b[0], b[1], b[2]) <= hi)) return false;
    double lo = 0.0;
    for (int k = 0; k < kReHalvings; ++k) {
        const double mid = 0.5 * (lo + up);
        if (reentry_hermite_height(a, b, dt, mid) <= hi) up = mid;
        else lo = mid;
    }
    s = 0.5 * (lo + up);
    return true;
}

// One trajectory's result
struct ReentryOut {
    double dt;               // minutes from epoch to the crossing; +inf ABOVE, NaN failed
    double lat, lon;         // geodetic latitude, east longitude [deg] (NaN unless REENTERED)
    double speed, fpa;       // inertial speed [km/s], inertial flight-path angle [deg]
    double y[6];             // TEME state at the crossing
    uint64_t counts[2];      // accepted, rejected DP87 attempts
    uint8_t status;          // kRe*
};

AZ_HD void reentry_fail(ReentryOut &o, uint8_t status) {
    const double nan = std::numeric_limits<double>::quiet_NaN();
    o.dt = o.lat = o.lon = o.speed = o.fpa = nan;
    for (int c = 0; c < 6; ++c) o.y[c] = nan;
    o.status = status;
}

// The crossing's words from its TEME state y at t seconds after epochJd: the footprint by the ECEF mode's GMST rotation
AZ_HD void reentry_footprint(const double (&y)[6], double epochJd, double t, ReentryOut &o) {
    constexpr double r2d = 180.0 / detail::kHPi;
    double sg, cg;
    sincos_full(pairs_gmst(epochJd + t / 86400.0), sg, cg);
    double x = y[0], yy = y[1], z = y[2];
    eci_to_ecef(x, yy, sg, cg);
    ecef_to_geodetic(x, yy, z);
    o.dt = t / 60.0;
    o.lat = x * r2d;
    o.lon = yy * r2d;
    const double r = sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
    o.speed = sqrt(y[3] * y[3] + y[4] * y[4] + y[5] * y[5]);
    o.fpa = asin((y[0] * y[3] + y[1] * y[4] + y[2] * y[5]) / (r * o.speed)) * r2d;
    for (int c = 0; c < 6; ++c) o.y[c] = y[c];
    o.status = kReReentered;
}

// One trajectory from the epoch state y0 with ballistic coefficient B [m^2/kg] and density factor f.  y[6] holds each
// interval's start state: memory the caller gives (the warp's shared slot on the device), so that it does not hold
// registers while DP87's stages do.
AZ_HD void reentry_integrate(const double (&y0)[6], double epochJd, double B, double f, const ReentryCall &c,
                             double (&y)[6], ReentryOut &o) {
    o.counts[0] = o.counts[1] = 0;
    if (!(B > 0.0) || !isfinite(B)) return reentry_fail(o, kReNonphysical);
    for (int q = 0; q < 6; ++q) y[q] = y0[q];
    if (reentry_height(y[0], y[1], y[2]) <= c.hi) return reentry_footprint(y, epochJd, 0.0, o);
    const ReentryForces F{c.mu, c.rEq, c.j2, c.omega, B * f * c.scale};
    const NumParams p{c.mu, c.j2, c.rEq, kReRtol, kReAtol};
    double t = 0.0, hCur = kDpHStart;
    while (t < c.horizon) {
        const double dt = fmin(c.step, c.horizon - t);
        double b[6];
        for (int q = 0; q < 6; ++q) b[q] = y[q];
        if (dp87_interval(b, hCur, dt, F, p, o.counts) != kNumOk || !all_finite(b))
            return reentry_fail(o, kReStopped);
        double s;
        if (reentry_locate(y, b, dt, c.hi, s)) {
            double q[6];
            reentry_hermite(y, b, dt, s, q);
            return reentry_footprint(q, epochJd, t + s * dt, o);
        }
        for (int q = 0; q < 6; ++q) y[q] = b[q];
        t += dt;
    }
    reentry_fail(o, kReAbove);
    o.dt = std::numeric_limits<double>::infinity();
}

// A request's row as the trajectories read it: K14's nominal variables and factor, B_row, the epoch and model
struct ReentryRow {
    double xh[kFitVars];
    McFactor F;
    double B, epoch;
    uint32_t model;
    uint32_t status;    // kRe* request status
};

// Request status and row words from the row's columns, P words, model byte and B (given: ballistic, else NaN)
AZ_HD uint8_t reentry_row(const double (&el)[8], const double *P, int model, const Gravity &grav, bool hasB,
                          double ballistic, ReentryRow &R) {
    const uint8_t st = mc_row(el, P, model, grav, R.xh, R.F);
    R.B = hasB ? ballistic : kReBstarToB * el[7];
    R.epoch = el[0];
    R.model = (uint32_t)model;
    R.status = st == kConjOk ? kReOk : st == kConjNotPsd ? kReNotPsd : kReInitFailed;
    return (uint8_t)R.status;
}

// Sample k's seven element normals (K14's primary normals 0..6) and normal 7 under seed
AZ_HD void reentry_normals(uint64_t seed, uint64_t k, double (&z)[kFitVars], double &z7) {
    double all[8];
    for (int j = 0; j < 4; ++j) mc_normal_pair(seed, k, j, all[2 * j], all[2 * j + 1]);
    for (int v = 0; v < kFitVars; ++v) z[v] = all[v];
    z7 = all[7];
}

// Trajectory variables x, B and f: the nominal (sample = false) or sample k
AZ_HD void reentry_params(const ReentryRow &R, bool sample, uint64_t seed, uint64_t k, double sigma,
                          double (&x)[kFitVars], double &B, double &f) {
    if (!sample) {
        for (int v = 0; v < kFitVars; ++v) x[v] = R.xh[v];
        B = R.B;
        f = 1.0;
        return;
    }
    double z[kFitVars], z7;
    reentry_normals(seed, k, z, z7);
    mc_draw(R.F, R.xh, z, x);
    B = R.B + kReBstarToB * (x[6] - R.xh[6]);
    f = exp(sigma * z7);
}

// The TEME state at epoch (tsince 0) of the set of x: near-earth, its columns built into cols ...
AZ_HD bool reentry_epoch_near(const double (&x)[kFitVars], double epochJd, const Gravity &grav, const GravConsts &g,
                              double *cols, double (&y)[6]) {
    double inv;
    if (!fit_build_set_of<FitNearEarth>(x, 0, epochJd, grav, cols, inv)) return false;
    conj_eval_near([cols](int c) { return cols[c]; }, 0.0, g, y);
    return all_finite(y);
}
// ... and deep space, its record built into set (pairs_sdp4_at at tsince 0: the lattice's node 0 is (xlamo, no))
AZ_HD bool reentry_epoch_deep(const double (&x)[kFitVars], double epochJd, const Gravity &grav, const GravConsts &g,
                              Sdp4Sat &set, double (&y)[6]) {
    double inv;
    if (!fit_build_set_of<FitDeepSpace>(x, 0, epochJd, grav, set, inv)) return false;
    CellOut o;
    if (sdp4_cell(set, 0.0, set.xlamo, set.no, 0.0, g, o) != 0) return false;
    y[0] = o.rx, y[1] = o.ry, y[2] = o.rz, y[3] = o.vx, y[4] = o.vy, y[5] = o.vz;
    return all_finite(y);
}

// Failed trajectories: INIT_FAILED, NONPHYSICAL, STOPPED
AZ_HD bool reentry_failed(uint8_t st) { return st != kReReentered && st != kReAbove; }

}  // namespace az
