// az_iod.cuh -- K13: initial orbits for tracks that match no catalogue row.  __host__ __device__, so the kernels
// (az_iod.cu) and the host emulation (tests/host_emul/emul_iod.cu) run this source.
//
// Track j is the observations [offsets[j], offsets[j + 1]) in K8's observation layout (az_obs.cuh), in time order.
// Its epoch is the time of its middle observation, index floor(m / 2); it depends on the track alone.
//
// Geometry (the exact inverses of obs_model, with its GMST, station and omega):
//   TEME state   r, v as given;
//   ECEF state   r = Rz(GMST)^T r_ecef, v = Rz(GMST)^T (v_ecef + omega x r_ecef);
//   radar        r = Rz(GMST)^T (r_station + range (E sin az cos el + N cos az cos el + U sin el)); range-rate is
//                scored, never built from;
//   optical      the TEME line of sight L of (ra, dec) and the station's TEME position R = Rz(GMST)^T r_station.
// A method builds only from the observations whose geometry components are all used (sigma < inf): all six of a
// state, range / azimuth / elevation of a radar observation, both angles of an optical one.
//
// Candidates, from every method the track's observations allow (no threshold picks a method):
//   state        every state observation (TEME or ECEF), at its own time;
//   Gibbs, Herrick-Gibbs   >= 3 radar positions: both, for the middle position of every triplet of the table;
//   Lambert      exactly 2 radar positions: K9's lambert_solve, zero revolutions, normal +z (prograde) and -z
//                (retrograde), at the first position's time;
//   Gauss        >= 3 optical observations: every triplet of the table with |D0| = |L1 . (L2 x L3)| >= kIodGaussD0.
//                Every real root of the 8th-degree polynomial in r2 above 1 earth radius (bracketed on a geometric
//                grid of kIodGaussGrid points up to Fujiwara's bound, then bisected), each refined by Curtis'
//                Algorithm 5.6 (universal-variable f and g, averaged with the previous iterate) until every slant
//                range moves by at most kIodGaussTol of itself; a root whose refinement does not converge in
//                kIodGaussIter steps, or whose slant ranges turn negative, gives no candidate.
// Triplets: a fixed table of kIodTriplets fractional triplets (iod_triplet), mapped onto the method's observation
// count c by rounding; entry 0 is (first, middle, last), entries that collapse or repeat an earlier one are skipped.
// A candidate is rejected when it is not finite, e >= 1, or its perigee radius is below the model's earth radius.
//
// Score: each candidate is propagated two-body (universal variables, iod_kepler) from its reference time to every
// observation of the track and passed through obs_residual_rows (K8's residual rules: azimuth and right ascension
// wrapped and scaled by the cosine of the observed partner, sigma = inf not used); F = the sum of the squared weighted
// residuals.  The winner is the least (F, method, triplet, root); wrms = sqrt(F / used residuals).
//
// Conversion: the winner propagated two-body to the epoch, then its osculating elements (iod_coe: n in rev/day, the
// track's B*) are the initial set of K8's own fit (launch_fit, then launch_fit_deep) to one TEME state at the epoch
// with B* held: 6 residuals for 6 variables.  The class follows the initial set, as in the mixed fit.  The fit's final
// position and velocity residuals are the conversion residuals; above kIodConvDr / kIodConvDv, or a fit that did not
// converge, the track is CONVERSION_FAILED.
#pragma once

#include "az_correlate.cuh"
#include "az_lambert.cuh"

namespace az {

// per-track status bytes (ASTROZ_IOD_*) and methods (ASTROZ_IOD_METHOD_*)
enum IodStatus : uint8_t { kIodOk = 0, kIodTooFew = 1, kIodNoCandidate = 2, kIodConversionFailed = 3, kIodBadTrack = 4 };
enum IodMethod : uint8_t {
    kIodState = 0, kIodGibbs = 1, kIodHerrickGibbs = 2, kIodLambert = 3, kIodGauss = 4, kIodNone = 255
};
constexpr uint32_t kIodMaxTrack = 256;      // observations per track, K12's limit
constexpr int kIodTriplets = 30;            // entries of the triplet table
constexpr double kIodGaussD0 = 1e-12;       // the least |L1 . (L2 x L3)| a Gauss triplet may have
constexpr int kIodGaussGrid = 512;          // bracketing grid of the octic
constexpr int kIodGaussIter = 200;          // refinement steps
constexpr double kIodGaussTol = 1e-10;      // relative slant-range change that ends the refinement: 100x
                                            // above the rounding of the slant ranges at |D0| ~ 1e-4
constexpr int kIodKeplerIter = 50;          // Newton steps of the universal Kepler equation
constexpr double kIodConvDr = 1e-6;         // km
constexpr double kIodConvDv = 1e-9;         // km/s
constexpr uint32_t kIodFitIter = 50;        // the conversion fit's iteration limit
constexpr double kIodFitPosSigma = 1.0, kIodFitVelSigma = 1e-3;   // its weights (km, km/s)

AZ_HD double iod_dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
AZ_HD double iod_norm(const double *a) { return std::sqrt(iod_dot(a, a)); }
AZ_HD void iod_cross(const double *a, const double *b, double *o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
// x = Rz(GMST)^T X in place (the inverse of eci_to_ecef)
AZ_HD void iod_to_teme(double &x, double &y, double sg, double cg) {
    const double X = x, Y = y;
    x = cg * X - sg * Y;
    y = sg * X + cg * Y;
}

// ---- two-body propagation by universal variables (Curtis, Algorithms 3.3 and 3.4) ----------------------------------
AZ_HD void iod_stumpff(double z, double &C, double &S) {
    if (std::fabs(z) < 0.1) {   // the series: the closed forms cancel near z = 0
        C = 1.0 / 2 - z * (1.0 / 24 - z * (1.0 / 720 - z * (1.0 / 40320 - z * (1.0 / 3628800 - z / 479001600.0))));
        S = 1.0 / 6 - z * (1.0 / 120 - z * (1.0 / 5040 - z * (1.0 / 362880 - z * (1.0 / 39916800 - z / 6227020800.0))));
    } else if (z > 0.0) {
        const double s = std::sqrt(z);
        C = (1.0 - std::cos(s)) / z;
        S = (s - std::sin(s)) / (z * s);
    } else {
        const double s = std::sqrt(-z);
        C = (std::cosh(s) - 1.0) / -z;
        S = (std::sinh(s) - s) / (-z * s);
    }
}

// The universal anomaly chi of a flight of dt seconds from (r0, v0): Newton from Curtis' guess until a step is at most
// 1e-13 of chi.  False when it does not converge.
AZ_HD bool iod_chi(double r0n, double vr0, double alpha, double dt, double mu, double &chi) {
    const double smu = std::sqrt(mu);
    chi = smu * std::fabs(alpha) * dt;
    for (int it = 0; it < kIodKeplerIter; ++it) {
        double C, S;
        const double z = alpha * chi * chi;
        iod_stumpff(z, C, S);
        const double F = r0n * vr0 / smu * chi * chi * C + (1.0 - alpha * r0n) * chi * chi * chi * S + r0n * chi -
                         smu * dt;
        const double dF = r0n * vr0 / smu * chi * (1.0 - z * S) + (1.0 - alpha * r0n) * chi * chi * C + r0n;
        const double d = F / dF;
        chi -= d;
        if (!(std::fabs(chi) < INFINITY)) return false;
        if (std::fabs(d) <= 1e-13 * std::fabs(chi) || d == 0.0) return true;
    }
    return false;
}

// f, g (and their rates) of a flight of dt seconds from (r0, v0), and the state (r, v) it reaches.
AZ_HD bool iod_kepler(const double *r0, const double *v0, double dt, double mu, double *r, double *v) {
    if (dt == 0.0) {
        for (int c = 0; c < 3; ++c) r[c] = r0[c], v[c] = v0[c];
        return true;
    }
    const double r0n = iod_norm(r0), vr0 = iod_dot(r0, v0) / r0n, alpha = 2.0 / r0n - iod_dot(v0, v0) / mu;
    double chi;
    if (!iod_chi(r0n, vr0, alpha, dt, mu, chi)) return false;
    double C, S;
    const double z = alpha * chi * chi;
    iod_stumpff(z, C, S);
    const double f = 1.0 - chi * chi / r0n * C, g = dt - chi * chi * chi * S / std::sqrt(mu);
    double rr[3];
    for (int c = 0; c < 3; ++c) rr[c] = f * r0[c] + g * v0[c];
    const double rn = iod_norm(rr);
    const double fd = std::sqrt(mu) / (rn * r0n) * (z * chi * S - chi), gd = 1.0 - chi * chi / rn * C;
    for (int c = 0; c < 3; ++c) {
        v[c] = fd * r0[c] + gd * v0[c];
        r[c] = rr[c];
    }
    return rn > 0.0 && rn < INFINITY;
}

// Seconds from tRef to jdFull (both jd + fr sums, as every kernel of the library forms them)
AZ_HD double iod_seconds(double jdFull, double tRef) { return mul_rn(sub_rn(jdFull, tRef), 86400.0); }

// ---- osculating elements ---------------------------------------------------------------------------------------------
// e and the perigee radius of (r, v); false when the orbit is not a closed one SGP4 can carry (not finite, e >= 1, or
// perigee below rE).
AZ_HD bool iod_admissible(const double *s, double mu, double rE) {
    for (int c = 0; c < 6; ++c)
        if (!(std::fabs(s[c]) < INFINITY)) return false;
    const double rn = iod_norm(s), v2 = iod_dot(s + 3, s + 3), rv = iod_dot(s, s + 3);
    if (!(rn > 0.0)) return false;
    const double alpha = 2.0 / rn - v2 / mu;   // 1 / a
    double ev[3];
    for (int c = 0; c < 3; ++c) ev[c] = ((v2 - mu / rn) * s[c] - rv * s[3 + c]) / mu;
    const double e = iod_norm(ev);
    return alpha > 0.0 && e < 1.0 && (1.0 - e) / alpha >= rE;
}

// (r, v) -> the eight element columns (epoch JD, n rev/day, e, i, node, w, M deg, B*), osculating.  The node is 0 when
// the orbit is equatorial, w is 0 when it is circular; u = w + nu is measured from the node in either case.
AZ_HD void iod_coe(const double *s, double mu, double epochJd, double bstar, double (&el)[8]) {
    const double r2d = 1.0 / detail::kDeg;
    const double *r = s, *v = s + 3;
    double h[3];
    iod_cross(r, v, h);
    const double hn = iod_norm(h), hxy = std::sqrt(h[0] * h[0] + h[1] * h[1]);
    const double rn = iod_norm(r), v2 = iod_dot(v, v), rv = iod_dot(r, v);
    const double a = 1.0 / (2.0 / rn - v2 / mu);
    double ev[3];
    for (int c = 0; c < 3; ++c) ev[c] = ((v2 - mu / rn) * r[c] - rv * v[c]) / mu;
    const double inc = std::atan2(hxy, h[2]);
    const double node = hxy > 1e-14 * hn ? std::atan2(h[0], -h[1]) : 0.0;
    const double p[3] = {std::cos(node), std::sin(node), 0.0};   // the node's unit vector
    double hu[3], q[3];
    for (int c = 0; c < 3; ++c) hu[c] = h[c] / hn;
    iod_cross(hu, p, q);
    const double u = std::atan2(iod_dot(r, q), iod_dot(r, p));
    const double ex = iod_dot(ev, p), ey = iod_dot(ev, q);
    const double e = std::sqrt(ex * ex + ey * ey);
    const double w = std::atan2(ey, ex);
    const double nu = u - w;
    const double E = std::atan2(std::sqrt(1.0 - e * e) * std::sin(nu), e + std::cos(nu));
    const double M = E - e * std::sin(E);
    el[0] = epochJd;
    el[1] = std::sqrt(mu / (a * a * a)) * 86400.0 / kTwoPi;
    el[2] = e;
    el[3] = inc * r2d;
    el[4] = detail::wrap(node * r2d, 360.0);
    el[5] = detail::wrap(w * r2d, 360.0);
    el[6] = detail::wrap(M * r2d, 360.0);
    el[7] = bstar;
}

// ---- the methods ------------------------------------------------------------------------------------------------------
// Gibbs (Curtis, Algorithm 5.1): v2 of three positions
AZ_HD void iod_gibbs(const double *r1, const double *r2, const double *r3, double mu, double *v2) {
    const double a = iod_norm(r1), b = iod_norm(r2), c = iod_norm(r3);
    double c12[3], c23[3], c31[3], N[3], D[3], S[3], Dr[3];
    iod_cross(r1, r2, c12);
    iod_cross(r2, r3, c23);
    iod_cross(r3, r1, c31);
    for (int k = 0; k < 3; ++k) {
        N[k] = a * c23[k] + b * c31[k] + c * c12[k];
        D[k] = c12[k] + c23[k] + c31[k];
        S[k] = (b - c) * r1[k] + (c - a) * r2[k] + (a - b) * r3[k];
    }
    iod_cross(D, r2, Dr);
    const double f = std::sqrt(mu / (iod_norm(N) * iod_norm(D)));
    for (int k = 0; k < 3; ++k) v2[k] = f * (Dr[k] / b + S[k]);
}

// Herrick-Gibbs (Vallado, Algorithm 55): v2 of three positions at t1, t2, t3 seconds
AZ_HD void iod_herrick_gibbs(const double *r1, const double *r2, const double *r3, double t1, double t2, double t3,
                             double mu, double *v2) {
    const double d31 = t3 - t1, d32 = t3 - t2, d21 = t2 - t1;
    const double a = iod_norm(r1), b = iod_norm(r2), c = iod_norm(r3);
    const double k1 = -d32 * (1.0 / (d21 * d31) + mu / (12.0 * a * a * a));
    const double k2 = (d32 - d21) * (1.0 / (d21 * d32) + mu / (12.0 * b * b * b));
    const double k3 = d21 * (1.0 / (d32 * d31) + mu / (12.0 * c * c * c));
    for (int k = 0; k < 3; ++k) v2[k] = k1 * r1[k] + k2 * r2[k] + k3 * r3[k];
}

// The octic x^8 + a x^6 + b x^3 + c of Gauss' method
AZ_HD double iod_octic(double x, double a, double b, double c) {
    const double x3 = x * x * x;
    return ((x * x + a) * x3 + b) * x3 + c;
}

// Its real roots above rE, ascending, into roots[3]: sign changes on a geometric grid from rE to Fujiwara's bound,
// each bisected to adjacent doubles.  Returns the count.
AZ_HD int iod_octic_roots(double a, double b, double c, double rE, double (&roots)[3]) {
    const double hi = 2.0 * fmax(fmax(std::sqrt(std::fabs(a)), std::pow(std::fabs(b), 0.2)),
                                 std::pow(0.5 * std::fabs(c), 0.125));
    int n = 0;
    if (!(hi > rE) || !(hi < INFINITY)) return 0;
    const double step = std::log(hi / rE) / (kIodGaussGrid - 1);
    double x0 = rE, f0 = iod_octic(x0, a, b, c);
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int k = 1; k < kIodGaussGrid && n < 3; ++k) {
        const double x1 = k == kIodGaussGrid - 1 ? hi : rE * std::exp(step * k);
        const double f1 = iod_octic(x1, a, b, c);
        if (f0 == 0.0) {
            roots[n++] = x0;
        } else if ((f0 < 0.0) != (f1 < 0.0) && f1 != 0.0) {
            double lo = x0, up = x1, flo = f0;
            for (int it = 0; it < 200; ++it) {
                const double mid = 0.5 * (lo + up);
                if (mid <= lo || mid >= up) break;
                const double fm = iod_octic(mid, a, b, c);
                if ((fm < 0.0) == (flo < 0.0)) lo = mid, flo = fm;
                else up = mid;
            }
            roots[n++] = 0.5 * (lo + up);
        }
        x0 = x1;
        f0 = f1;
    }
    return n;
}

// Gauss' method on one optical triplet: L[3][3] lines of sight, R[3][3] station positions (TEME), t[3] seconds.
// emit(state at t[1], root) for every root that refines; returns the number of roots (before refinement).
// Curtis, Algorithms 5.5 and 5.6.
template <typename Emit>
AZ_HD int iod_gauss(const double (&L)[3][3], const double (&R)[3][3], const double (&t)[3], double mu, double rE,
                    Emit &&emit) {
    const double tau1 = t[0] - t[1], tau3 = t[2] - t[1], tau = tau3 - tau1;
    double p1[3], p2[3], p3[3];
    iod_cross(L[1], L[2], p1);
    iod_cross(L[0], L[2], p2);
    iod_cross(L[0], L[1], p3);
    const double D0 = iod_dot(L[0], p1);
    if (!(std::fabs(D0) >= kIodGaussD0) || !(tau1 < 0.0) || !(tau3 > 0.0)) return 0;
    double D[3][3];   // D[i][j] = R_i . p_j
    for (int i = 0; i < 3; ++i) {
        D[i][0] = iod_dot(R[i], p1);
        D[i][1] = iod_dot(R[i], p2);
        D[i][2] = iod_dot(R[i], p3);
    }
    const double A = (-D[0][1] * tau3 / tau + D[1][1] + D[2][1] * tau1 / tau) / D0;
    const double B = (D[0][1] * (tau3 * tau3 - tau * tau) * tau3 / tau + D[2][1] * (tau * tau - tau1 * tau1) * tau1 / tau) /
                     (6.0 * D0);
    const double E = iod_dot(L[1], R[1]), R22 = iod_dot(R[1], R[1]);
    const double a = -(A * A + 2.0 * A * E + R22), b = -2.0 * mu * B * (A + E), c = -mu * mu * B * B;
    double roots[3];
    const int nr = iod_octic_roots(a, b, c, rE, roots);
    for (int q = 0; q < nr; ++q) {
        const double x = roots[q], x3 = x * x * x;
        double rho[3];
        rho[0] = ((6.0 * (D[2][0] * tau1 / tau3 + D[1][0] * tau / tau3) * x3 + mu * D[2][0] * (tau * tau - tau1 * tau1) *
                   tau1 / tau3) / (6.0 * x3 + mu * (tau * tau - tau3 * tau3)) - D[0][0]) / D0;
        rho[1] = A + mu * B / x3;
        rho[2] = ((6.0 * (D[0][2] * tau3 / tau1 - D[1][2] * tau / tau1) * x3 + mu * D[0][2] * (tau * tau - tau3 * tau3) *
                   tau3 / tau1) / (6.0 * x3 + mu * (tau * tau - tau1 * tau1)) - D[2][2]) / D0;
        double f1 = 1.0 - 0.5 * mu * tau1 * tau1 / x3, f3 = 1.0 - 0.5 * mu * tau3 * tau3 / x3;
        double g1 = tau1 - mu * tau1 * tau1 * tau1 / (6.0 * x3), g3 = tau3 - mu * tau3 * tau3 * tau3 / (6.0 * x3);
        double r[3][3], v2[3];
        auto positions = [&]() {
            for (int i = 0; i < 3; ++i)
                for (int k = 0; k < 3; ++k) r[i][k] = R[i][k] + rho[i] * L[i][k];
            const double den = f1 * g3 - f3 * g1;
            for (int k = 0; k < 3; ++k) v2[k] = (-f3 * r[0][k] + f1 * r[2][k]) / den;
        };
        positions();
        bool ok = rho[0] > 0.0 && rho[1] > 0.0 && rho[2] > 0.0, done = false;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
        for (int it = 0; ok && !done && it < kIodGaussIter; ++it) {
            const double r2n = iod_norm(r[1]), vr2 = iod_dot(v2, r[1]) / r2n;
            const double alpha = 2.0 / r2n - iod_dot(v2, v2) / mu;
            double chi1, chi3, C1, S1, C3, S3;
            if (!iod_chi(r2n, vr2, alpha, tau1, mu, chi1) || !iod_chi(r2n, vr2, alpha, tau3, mu, chi3)) {
                ok = false;
                break;
            }
            iod_stumpff(alpha * chi1 * chi1, C1, S1);
            iod_stumpff(alpha * chi3 * chi3, C3, S3);
            const double smu = std::sqrt(mu);
            f1 = 0.5 * (f1 + 1.0 - chi1 * chi1 / r2n * C1);
            g1 = 0.5 * (g1 + tau1 - chi1 * chi1 * chi1 * S1 / smu);
            f3 = 0.5 * (f3 + 1.0 - chi3 * chi3 / r2n * C3);
            g3 = 0.5 * (g3 + tau3 - chi3 * chi3 * chi3 * S3 / smu);
            const double den = f1 * g3 - f3 * g1, c1 = g3 / den, c3 = -g1 / den;
            const double nrho[3] = {(-D[0][0] + D[1][0] / c1 - c3 / c1 * D[2][0]) / D0,
                                    (-c1 * D[0][1] + D[1][1] - c3 * D[2][1]) / D0,
                                    (-c1 / c3 * D[0][2] + D[1][2] / c3 - D[2][2]) / D0};
            done = true;
            for (int i = 0; i < 3; ++i) {
                done = done && std::fabs(nrho[i] - rho[i]) <= kIodGaussTol * std::fabs(nrho[i]);
                rho[i] = nrho[i];
            }
            ok = rho[0] > 0.0 && rho[1] > 0.0 && rho[2] > 0.0 && std::fabs(den) < INFINITY;
            positions();
        }
        if (ok && done) {
            const double s[6] = {r[1][0], r[1][1], r[1][2], v2[0], v2[1], v2[2]};
            emit(s, q);
        }
    }
    return nr;
}

// ---- a track ------------------------------------------------------------------------------------------------------------
// The geometry class of observation i: 1 a state with all six components used, 2 a radar observation with range,
// azimuth and elevation used, 3 an optical one with both angles used, 0 none.
AZ_HD int iod_class(const CorrObsArrays &a, uint32_t i) {
    const int kind = a.kind[i];
    const double *sg = a.sigma + (size_t)i * 6;
    const int need = kind <= kObsEcefState ? 6 : kind == kObsRadar ? 3 : 2;
    for (int c = 0; c < need; ++c)
        if (!(sg[c] < INFINITY)) return 0;
    return kind <= kObsEcefState ? 1 : kind == kObsRadar ? 2 : 3;
}

struct IodTrack {
    uint32_t begin, end, used;
    uint32_t count[4];    // observations of each geometry class (index 0 unused)
    double epoch;         // jdFull of the middle observation
    uint8_t status;       // kIodOk, kIodTooFew or kIodBadTrack
};

// A track's summary.  sorted = false: the device call's rule, an observation earlier than its predecessor makes the
// track BAD_TRACK.
AZ_HD void iod_track(const CorrObsArrays &a, uint32_t begin, uint32_t end, IodTrack &tr) {
    tr.begin = begin;
    tr.end = end;
    tr.used = 0;
    tr.count[0] = tr.count[1] = tr.count[2] = tr.count[3] = 0;
    tr.epoch = 0.0;
    tr.status = kIodBadTrack;
    if (end <= begin || end - begin > kIodMaxTrack) return;
    tr.used = corr_used(a, begin, end);
    bool sorted = true;
    double prev = -INFINITY;
    for (uint32_t i = begin; i < end; ++i) {
        const double t = add_rn(a.jd[i], a.fr[i]);
        sorted = sorted && !(t < prev);
        prev = t;
        ++tr.count[iod_class(a, i)];
    }
    if (!sorted || tr.used == 0) return;
    const uint32_t mid = begin + (end - begin) / 2;
    tr.epoch = add_rn(a.jd[mid], a.fr[mid]);
    tr.status = tr.count[1] == 0 && tr.count[2] < 2 && tr.count[3] < 3 ? kIodTooFew : kIodOk;
}

// Triplet q of the table in sixteenths of the way through c observations: 0 the whole span, 1-3 halves, 4-10
// quarters, 11-25 eighths (each middle at the midpoint), 26-29 long spans with an off-centre middle.
AZ_HD bool iod_triplet_raw(int q, uint32_t c, uint32_t (&ix)[3]) {
    int u0, span;
    int mid = -1;
    if (q == 0) u0 = 0, span = 16;
    else if (q < 4) u0 = 4 * (q - 1), span = 8;
    else if (q < 11) u0 = 2 * (q - 4), span = 4;
    else if (q < 26) u0 = q - 11, span = 2;
    else {
        const int m[4] = {4, 12, 2, 14};
        u0 = 0, span = 16, mid = m[q - 26];
    }
    const uint32_t u[3] = {(uint32_t)u0, (uint32_t)(mid >= 0 ? mid : u0 + span / 2), (uint32_t)(u0 + span)};
    for (int p = 0; p < 3; ++p) ix[p] = (u[p] * (c - 1) + 8) / 16;
    return ix[0] < ix[1] && ix[1] < ix[2];
}

// Triplet q of a method with c observations: false when it collapses or repeats an earlier entry
AZ_HD bool iod_triplet(int q, uint32_t c, uint32_t (&ix)[3]) {
    if (c < 3 || !iod_triplet_raw(q, c, ix)) return false;
    for (int p = 0; p < q; ++p) {
        uint32_t o[3];
        if (iod_triplet_raw(p, c, o) && o[0] == ix[0] && o[1] == ix[1] && o[2] == ix[2]) return false;
    }
    return true;
}

// The index of the k-th observation of geometry class cls in the track
AZ_HD uint32_t iod_nth(const CorrObsArrays &a, const IodTrack &tr, int cls, uint32_t k) {
    for (uint32_t i = tr.begin; i < tr.end; ++i)
        if (iod_class(a, i) == cls && k-- == 0) return i;
    return tr.end;
}

// Observation i's geometry: its time, and the TEME state (class 1), position (class 2) or line of sight L and station
// position R (class 3).
struct IodGeom {
    double t;
    double s[6];
    double L[3], R[3];
};

AZ_HD void iod_geom(const CorrObsArrays &a, uint32_t i, IodGeom &g) {
    CorrObs o;
    corr_obs(a, i, o);
    g.t = o.jdFull;
    for (int c = 0; c < 6; ++c) g.s[c] = 0.0;
    for (int c = 0; c < 3; ++c) g.L[c] = g.R[c] = 0.0;
    const double *v = o.value;
    if (o.kind == kObsTemeState) {
        for (int c = 0; c < 6; ++c) g.s[c] = v[c];
    } else if (o.kind == kObsEcefState) {
        g.s[0] = v[0], g.s[1] = v[1], g.s[2] = v[2];
        g.s[3] = v[3] - kObsOmega * v[1], g.s[4] = v[4] + kObsOmega * v[0], g.s[5] = v[5];
        iod_to_teme(g.s[0], g.s[1], o.sg, o.cg);
        iod_to_teme(g.s[3], g.s[4], o.sg, o.cg);
    } else if (o.kind == kObsRadar) {
        const double ce = std::cos(v[2]), se = std::sin(v[2]), ca = std::cos(v[1]), sa = std::sin(v[1]);
        const double E = v[0] * ce * sa, N = v[0] * ce * ca, U = v[0] * se;
        for (int c = 0; c < 3; ++c) g.s[c] = o.st.r[c] + E * o.st.e[c] + N * o.st.n[c] + U * o.st.u[c];
        iod_to_teme(g.s[0], g.s[1], o.sg, o.cg);
    } else {
        const double cd = std::cos(v[1]);
        g.L[0] = cd * std::cos(v[0]), g.L[1] = cd * std::sin(v[0]), g.L[2] = std::sin(v[1]);
        for (int c = 0; c < 3; ++c) g.R[c] = o.st.r[c];
        iod_to_teme(g.R[0], g.R[1], o.sg, o.cg);
    }
}

// F of a candidate state s at tRef over the whole track: two-body to each observation, K8's residual rows.  +inf when
// a propagation fails or F is not finite.
AZ_HD double iod_score(const CorrObsArrays &a, const IodTrack &tr, const double (&s)[6], double tRef, double mu) {
    double F = 0.0;
    for (uint32_t i = tr.begin; i < tr.end; ++i) {
        CorrObs o;
        corr_obs(a, i, o);
        auto eval = [&](int, double jdFull, const double (&)[1], double (&f)[6]) {
            return iod_kepler(s, s + 3, iod_seconds(jdFull, tRef), mu, f, f + 3);
        };
        double obs[6], sc[6], r[6];
        if (!obs_residual_rows(eval, 0, nullptr, o.jdFull, tRef, o.kind, o.value, o.w, o.sg, o.cg, o.st, obs, sc, r,
                               nullptr, 1))
            return INFINITY;
        for (int c = 0; c < 6; ++c) F += r[c] * r[c];
    }
    return F < INFINITY ? F : INFINITY;
}

// The running best of a lane: least (F, key), key = method << 16 | triplet << 2 | root
struct IodBest {
    double F;
    uint32_t key;
    double s[6];
    double tRef;
};

AZ_HD void iod_best_init(IodBest &b) {
    b.F = INFINITY;
    b.key = 0xFFFFFFFFu;
    for (int c = 0; c < 6; ++c) b.s[c] = 0.0;
    b.tRef = 0.0;
}
AZ_HD bool iod_better(double F, uint32_t key, double bF, uint32_t bKey) { return F < bF || (F == bF && key < bKey); }
AZ_HD uint32_t iod_key(int method, uint32_t index, int root) { return (uint32_t)method << 16 | index << 2 | root; }

// Generators of a track: its state observations, then 2 x kIodTriplets Gibbs / Herrick-Gibbs slots (>= 3 radar
// positions) or 2 Lambert slots (exactly 2), then kIodTriplets Gauss slots (>= 3 optical observations).
AZ_HD uint32_t iod_slots(const IodTrack &tr) {
    const uint32_t radar = tr.count[2] >= 3 ? 2 * kIodTriplets : tr.count[2] == 2 ? 2 : 0;
    return tr.count[1] + radar + (tr.count[3] >= 3 ? kIodTriplets : 0);
}

// Slot g: build its candidates, reject, score the rest into best.  Returns the candidates scored.
AZ_HD uint32_t iod_slot(const CorrObsArrays &a, const IodTrack &tr, uint32_t g, double mu, double rE, IodBest &best) {
    uint32_t scored = 0;
    auto offer = [&](const double (&s)[6], double tRef, uint32_t key) {
        if (!iod_admissible(s, mu, rE)) return;
        ++scored;
        const double F = iod_score(a, tr, s, tRef, mu);
        if (F < INFINITY && iod_better(F, key, best.F, best.key)) {
            best.F = F;
            best.key = key;
            for (int c = 0; c < 6; ++c) best.s[c] = s[c];
            best.tRef = tRef;
        }
    };
    if (g < tr.count[1]) {
        IodGeom o;
        iod_geom(a, iod_nth(a, tr, 1, g), o);
        const double s[6] = {o.s[0], o.s[1], o.s[2], o.s[3], o.s[4], o.s[5]};
        offer(s, o.t, iod_key(kIodState, g, 0));
        return scored;
    }
    g -= tr.count[1];
    const uint32_t radar = tr.count[2] >= 3 ? 2 * kIodTriplets : tr.count[2] == 2 ? 2 : 0;
    if (g < radar) {
        if (tr.count[2] == 2) {
            IodGeom p, q;
            iod_geom(a, iod_nth(a, tr, 2, 0), p);
            iod_geom(a, iod_nth(a, tr, 2, 1), q);
            const double n[3] = {0.0, 0.0, g == 0 ? 1.0 : -1.0};
            double v1[3];
            bool found = false;
            lambert_solve(p.s, q.s, iod_seconds(q.t, p.t), mu, n, 0,
                          [&](uint32_t, uint8_t st, int, const double *va, const double *) {
                              if (st != kLamOk) return;
                              found = true;
                              for (int c = 0; c < 3; ++c) v1[c] = va[c];
                          });
            if (found) {
                const double s[6] = {p.s[0], p.s[1], p.s[2], v1[0], v1[1], v1[2]};
                offer(s, p.t, iod_key(kIodLambert, g, 0));
            }
            return scored;
        }
        const int q = (int)(g >> 1), method = g & 1 ? kIodHerrickGibbs : kIodGibbs;
        uint32_t ix[3];
        if (!iod_triplet(q, tr.count[2], ix)) return scored;
        IodGeom o[3];
        for (int k = 0; k < 3; ++k) iod_geom(a, iod_nth(a, tr, 2, ix[k]), o[k]);
        double v2[3];
        if (method == kIodGibbs) iod_gibbs(o[0].s, o[1].s, o[2].s, mu, v2);
        else iod_herrick_gibbs(o[0].s, o[1].s, o[2].s, 0.0, iod_seconds(o[1].t, o[0].t), iod_seconds(o[2].t, o[0].t),
                               mu, v2);
        const double s[6] = {o[1].s[0], o[1].s[1], o[1].s[2], v2[0], v2[1], v2[2]};
        offer(s, o[1].t, iod_key(method, (uint32_t)q, 0));
        return scored;
    }
    const int q = (int)(g - radar);
    uint32_t ix[3];
    if (!iod_triplet(q, tr.count[3], ix)) return scored;
    IodGeom o[3];
    for (int k = 0; k < 3; ++k) iod_geom(a, iod_nth(a, tr, 3, ix[k]), o[k]);
    const double tRef = o[1].t;
    double L[3][3], R[3][3], t[3];
    for (int k = 0; k < 3; ++k) {
        for (int c = 0; c < 3; ++c) L[k][c] = o[k].L[c], R[k][c] = o[k].R[c];
        t[k] = iod_seconds(o[k].t, tRef);
    }
    iod_gauss(L, R, t, mu, rE, [&](const double (&s)[6], int root) {
        offer(s, tRef, iod_key(kIodGauss, (uint32_t)q, root));
    });
    return scored;
}

// The winner's outputs: its state at the epoch and the osculating initial set; deep = the initial set's class under
// the mixed fit's rule (build_near_earth's kDeepSpace, period > 225 min).  False when the winner does not reach the
// epoch.
AZ_HD bool iod_epoch_state(const IodBest &b, double epoch, double mu, double bstar, const Gravity &grav,
                           double (&state)[6], double (&el)[8], uint8_t &deep) {
    if (!iod_kepler(b.s, b.s + 3, iod_seconds(epoch, b.tRef), mu, state, state + 3)) return false;
    iod_coe(state, mu, epoch, bstar, el);
    TleRecord t;
    t.epochJd = el[0]; t.revPerDay = el[1]; t.ecc = el[2]; t.inclDeg = el[3];
    t.raanDeg = el[4]; t.argpDeg = el[5]; t.maDeg = el[6]; t.bstar = el[7];
    NearEarth ne;
    deep = build_near_earth(t, grav, ne) == kDeepSpace;
    return true;
}

// The track's final status from the IOD status and the conversion fit's status and residuals
AZ_HD uint8_t iod_final_status(uint8_t iod, uint8_t fit, double dr, double dv) {
    if (iod != kIodOk) return iod;
    return fit == kFitConverged && dr <= kIodConvDr && dv <= kIodConvDv ? kIodOk : kIodConversionFailed;
}

}  // namespace az
