// az_lambert.cuh -- per-problem core of K9: Lambert's problem for one (r1, r2, tof) with multi-revolution solutions,
// by Izzo's algorithm (D. Izzo, "Revisiting Lambert's problem", Celest. Mech. Dyn. Astron. 121, 2015): Householder
// iterations on Izzo's x, velocities from his gamma / rho / sigma reconstruction.  __host__ __device__, so
// tests/host_emul runs the same arithmetic on the CPU.
//
// This replaces the reference's OrbitalMechanics.lambertSolverSimple (src/OrbitalMechanics.zig:122-183), whose
// departure velocity does not reach r2 (it uses a heuristic semi-major axis where the Lagrange coefficients need the
// semi-latus rectum; SURVEY.md appendix C).  The reference's argument and degeneracy rules are kept.
//
// Conventions:
//   direction: the unit normal n sets the sense of motion.  With ih = r1 x r2 / |r1 x r2|, ih . n > 0 is the short way
//              (transfer angle < pi), ih . n < 0 the long way: lambda < 0 and the tangential unit vectors flip.  A
//              retrograde transfer is a negated n;
//   slots:     S = 2 max_revs + 1 solutions per problem: slot 0 is M = 0, slot 2M - 1 the left and slot 2M the right
//              branch of M revolutions;
//   status:    a slot that is not kLamOk has zero velocities;
//   numerics:  Householder steps on x until |dx| < 1e-13, at most 15 (then kLamNotConverged); T_min(M) by Halley steps
//              on dT/dx = 0, only for the largest candidate M.  Square roots and cube roots stand in for fractional
//              powers except in the M = 0 initial guess, and the file is compiled without FMA contraction, so the host
//              build equals a scalar C statement of the same operations bit for bit.
#pragma once

#include "az_math.cuh"

namespace az {

// per-slot status bytes (ASTROZ_LAMBERT_*)
constexpr uint8_t kLamOk = 0, kLamNoSolution = 1, kLamDegenerate = 2, kLamNotConverged = 3, kLamStateFailed = 4;
constexpr int kLamMaxIter = 15;
constexpr double kLamTol = 1e-13;
constexpr uint32_t kLamMaxRevs = 127;   // slot indices stay inside a byte
constexpr double kLamPi = 3.141592653589793;

AZ_HD double lam_norm(const double a[3]) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }
AZ_HD void lam_cross(const double a[3], const double b[3], double o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// The non-dimensional geometry of one problem.
struct LambertGeom {
    double lam, T, s, c, r1n, r2n;
    double ir1[3], ir2[3], it1[3], it2[3];
};

// kLamOk and g filled, or the status every slot of the problem takes: kLamNoSolution for tof <= 0, kLamDegenerate for a
// zero radius, |r1 x r2| < 1e-12 |r1| |r2| (the reference's |sin dnu| < 1e-12, OrbitalMechanics.zig:158) or ih . n = 0.
AZ_HD uint8_t lambert_geometry(const double r1[3], const double r2[3], double tof, double mu, const double n[3],
                               LambertGeom &g) {
    if (!(tof > 0.0)) return kLamNoSolution;
    g.r1n = lam_norm(r1);
    g.r2n = lam_norm(r2);
    if (g.r1n == 0.0 || g.r2n == 0.0) return kLamDegenerate;
    double h[3];
    lam_cross(r1, r2, h);
    const double hn = lam_norm(h);
    if (hn < 1e-12 * (g.r1n * g.r2n)) return kLamDegenerate;
    const double ih[3] = {h[0] / hn, h[1] / hn, h[2] / hn};
    const double dn = ih[0] * n[0] + ih[1] * n[1] + ih[2] * n[2];
    if (dn == 0.0) return kLamDegenerate;
    const double d[3] = {r2[0] - r1[0], r2[1] - r1[1], r2[2] - r1[2]};
    g.c = lam_norm(d);
    g.s = (g.r1n + g.r2n + g.c) / 2.0;
    for (int k = 0; k < 3; ++k) {
        g.ir1[k] = r1[k] / g.r1n;
        g.ir2[k] = r2[k] / g.r2n;
    }
    g.lam = sqrt(1.0 - g.c / g.s);
    if (dn < 0.0) {
        g.lam = -g.lam;
        lam_cross(g.ir1, ih, g.it1);
        lam_cross(g.ir2, ih, g.it2);
    } else {
        lam_cross(ih, g.ir1, g.it1);
        lam_cross(ih, g.ir2, g.it2);
    }
    g.T = sqrt(2.0 * mu / (g.s * g.s * g.s)) * tof;
    return kLamOk;
}

// 2F1(3, 1; 5/2; z) by its series, for Battin's form near x = 1 (|z| is small there)
AZ_HD double lambert_hyp2f1(double z) {
    double sum = 1.0, term = 1.0;
    for (int j = 0; j < 100; ++j) {
        term = term * (3.0 + j) / (2.5 + j) * z;
        sum = sum + term;
        if (fabs(term) < 1e-17) break;
    }
    return sum;
}

// Non-dimensional time of flight T(x, M): Battin's series for |x - 1| < 0.01, Lagrange's form for 0.01 < |x - 1| < 0.2,
// Lancaster's form otherwise (the switch points themselves take Lancaster's).
AZ_HD double lambert_tof(double x, double lam, int M) {
    const double dist = fabs(x - 1.0);
    const double l2 = lam * lam;
    if (dist < 0.2 && dist > 0.01) {
        const double a = 1.0 / (1.0 - x * x);
        if (a > 0.0) {
            const double alfa = 2.0 * acos(x);
            double beta = 2.0 * asin(sqrt(l2 / a));
            if (lam < 0.0) beta = -beta;
            return a * sqrt(a) * ((alfa - sin(alfa)) - (beta - sin(beta)) + 2.0 * kLamPi * M) / 2.0;
        }
        const double alfa = 2.0 * acosh(x);
        double beta = 2.0 * asinh(sqrt(-l2 / a));
        if (lam < 0.0) beta = -beta;
        return -a * sqrt(-a) * ((beta - sinh(beta)) - (alfa - sinh(alfa))) / 2.0;
    }
    const double E = x * x - 1.0;
    const double z = sqrt(1.0 + l2 * E);
    if (dist < 0.01) {
        const double eta = z - lam * x;
        const double s1 = 0.5 * (1.0 - lam - x * eta);
        const double q = 4.0 / 3.0 * lambert_hyp2f1(s1);
        const double rho = fabs(E);
        const double rev = M ? M * kLamPi / (rho * sqrt(rho)) : 0.0;
        return (eta * eta * eta * q + 4.0 * lam * eta) / 2.0 + rev;
    }
    const double y = sqrt(fabs(E));
    const double g = x * z - lam * E;
    const double d = E < 0.0 ? M * kLamPi + acos(g) : log(y * (z - lam * x) + g);
    return (x - lam * z - d / y) / E;
}

// dT/dx, d2T/dx2, d3T/dx3 at x, given T = T(x)
AZ_HD void lambert_dtdx(double x, double T, double lam, double &d1, double &d2, double &d3) {
    const double l2 = lam * lam, l3 = l2 * lam;
    const double umx2 = 1.0 - x * x;
    const double y = sqrt(1.0 - l2 * umx2);
    const double y2 = y * y, y3 = y2 * y;
    d1 = (3.0 * T * x - 2.0 + 2.0 * l3 * x / y) / umx2;
    d2 = (3.0 * T + 5.0 * x * d1 + 2.0 * (1.0 - l2) * l3 / y3) / umx2;
    d3 = (7.0 * x * d2 + 8.0 * d1 - 6.0 * (1.0 - l2) * l2 * l3 * x / (y3 * y2)) / umx2;
}

// T_min(M), M >= 1: Halley steps on dT/dx = 0 from x = 0
AZ_HD double lambert_tmin(double lam, int M) {
    double x = 0.0;
    double t = acos(lam) + lam * sqrt(1.0 - lam * lam) + M * kLamPi;
    for (int it = 0; it < kLamMaxIter; ++it) {
        double d1, d2, d3;
        lambert_dtdx(x, t, lam, d1, d2, d3);
        const double xn = x - d1 * d2 / (d2 * d2 - d1 * d3 / 2.0);
        const double err = fabs(x - xn);
        x = xn;
        t = lambert_tof(x, lam, M);
        if (err < kLamTol) break;
    }
    return t;
}

// M_max: the largest M <= maxRevs with T >= T_min(M)
AZ_HD int lambert_mmax(double T, double lam, uint32_t maxRevs) {
    const double mt = floor(T / kLamPi);
    int M = mt < (double)maxRevs ? (int)mt : (int)maxRevs;
    // below floor(T / pi) revolutions T > T00 + M pi >= T_min(M): only the largest candidate needs T_min
    if (M > 0 && T < acos(lam) + lam * sqrt(1.0 - lam * lam) + M * kLamPi && lambert_tmin(lam, M) > T) --M;
    return M;
}

// Izzo's initial guess for slot `slot` (M = (slot + 1) / 2; odd slots the left branch)
AZ_HD double lambert_guess(double T, double lam, uint32_t slot) {
    const int M = (int)((slot + 1) / 2);
    if (M == 0) {
        const double l2 = lam * lam, l3 = l2 * lam;
        const double t00 = acos(lam) + lam * sqrt(1.0 - l2);
        const double t1 = 2.0 / 3.0 * (1.0 - l3);
        if (T >= t00) return -(T - t00) / (T - t00 + 4.0);
        if (T <= t1) return t1 * (t1 - T) / (2.0 / 5.0 * (1.0 - l2 * l3) * T) + 1.0;
        return pow(T / t00, 0.69314718055994529 / log(t1 / t00)) - 1.0;
    }
    const double v = (slot & 1) ? (M + 1) * kLamPi / (8.0 * T) : 8.0 * T / (M * kLamPi);
    const double q = cbrt(v * v);
    return (q - 1.0) / (q + 1.0);
}

// Householder iterations on x towards T(x, M) = T.  The number of steps taken, or 0 when |dx| stayed >= 1e-13 for
// kLamMaxIter steps (a NaN included).
AZ_HD int lambert_householder(double T, double lam, int M, double &x) {
    for (int it = 1; it <= kLamMaxIter; ++it) {
        const double t = lambert_tof(x, lam, M);
        double d1, d2, d3;
        lambert_dtdx(x, t, lam, d1, d2, d3);
        const double delta = t - T;
        const double d1s = d1 * d1;
        const double xn = x - delta * (d1s - delta * d2 / 2.0) / (d1 * (d1s - delta * d2) + d3 * delta * delta / 6.0);
        const double err = fabs(x - xn);
        x = xn;
        if (err < kLamTol) return it;
    }
    return 0;
}

// v1, v2 of the solution x
AZ_HD void lambert_velocities(const LambertGeom &g, double mu, double x, double v1[3], double v2[3]) {
    const double lam = g.lam;
    const double gamma = sqrt(mu * g.s / 2.0);
    const double rho = (g.r1n - g.r2n) / g.c;
    const double sigma = sqrt(fmax(0.0, 1.0 - rho * rho));
    const double y = sqrt(1.0 - lam * lam * (1.0 - x * x));
    const double vr1 = gamma * ((lam * y - x) - rho * (lam * y + x)) / g.r1n;
    const double vr2 = -gamma * ((lam * y - x) + rho * (lam * y + x)) / g.r2n;
    const double vt = gamma * sigma * (y + lam * x);
    const double vt1 = vt / g.r1n, vt2 = vt / g.r2n;
    for (int k = 0; k < 3; ++k) {
        v1[k] = vr1 * g.ir1[k] + vt1 * g.it1[k];
        v2[k] = vr2 * g.ir2[k] + vt2 * g.it2[k];
    }
}

// Solve one problem: emit(slot, status, iterations, v1, v2) for slots 0 .. 2 maxRevs in order.  A problem's results
// depend on its own inputs alone.
template <class Emit>
AZ_HD void lambert_solve(const double r1[3], const double r2[3], double tof, double mu, const double n[3],
                         uint32_t maxRevs, Emit &&emit) {
    const double zero[3] = {0.0, 0.0, 0.0};
    const uint32_t S = 2 * maxRevs + 1;
    LambertGeom g;
    const uint8_t st = lambert_geometry(r1, r2, tof, mu, n, g);
    if (st != kLamOk) {
        for (uint32_t slot = 0; slot < S; ++slot) emit(slot, st, 0, zero, zero);
        return;
    }
    const int mMax = lambert_mmax(g.T, g.lam, maxRevs);
    for (uint32_t slot = 0; slot < S; ++slot) {
        const int M = (int)((slot + 1) / 2);
        if (M > mMax) {
            emit(slot, kLamNoSolution, 0, zero, zero);
            continue;
        }
        double x = lambert_guess(g.T, g.lam, slot);
        const int it = lambert_householder(g.T, g.lam, M, x);
        if (!it) {
            emit(slot, kLamNotConverged, kLamMaxIter, zero, zero);
            continue;
        }
        double v1[3], v2[3];
        lambert_velocities(g, mu, x, v1, v2);
        emit(slot, kLamOk, it, v1, v2);
    }
}

// One porkchop cell: the chaser at (rc, vc) departs, the target is at (rt, vt) on arrival tof later.  The transfer is
// prograde relative to the chaser (n = rc x vc); every feasible slot is solved and the one with the least
// |v1 - vc| + |vt - v2| kept, the lowest slot on a tie.  No OK slot: dv = 0, slot 0 and slot 0's status.
AZ_HD void lambert_porkchop_cell(const double rc[3], const double vc[3], const double rt[3], const double vt[3],
                                 double tof, double mu, uint32_t maxRevs, double dv[2], uint8_t &slot,
                                 uint8_t &status) {
    double n[3];
    lam_cross(rc, vc, n);
    double best = 0.0, b0 = 0.0, b1 = 0.0;
    uint8_t bestSlot = 0, st0 = kLamNoSolution;
    bool found = false;
    lambert_solve(rc, rt, tof, mu, n, maxRevs,
                  [&](uint32_t s, uint8_t st, int, const double v1[3], const double v2[3]) {
                      if (s == 0) st0 = st;
                      if (st != kLamOk) return;
                      const double d1[3] = {v1[0] - vc[0], v1[1] - vc[1], v1[2] - vc[2]};
                      const double d2[3] = {vt[0] - v2[0], vt[1] - v2[1], vt[2] - v2[2]};
                      const double a = lam_norm(d1), b = lam_norm(d2);
                      if (!found || a + b < best) {
                          found = true;
                          best = a + b;
                          b0 = a;
                          b1 = b;
                          bestSlot = (uint8_t)s;
                      }
                  });
    dv[0] = b0;
    dv[1] = b1;
    slot = bestSlot;
    status = found ? kLamOk : st0;
}

}  // namespace az

#ifndef AZ_LAMBERT_CORES_ONLY
namespace az {
struct LambertArgs {
    const double *r1, *r2, *tof, *normal;   // [n][3], [n][3], [n], [n][3] (nullable: +z)
    uint32_t n, maxRevs;
    double mu;
    double *v1, *v2;                        // [n][S][3]
    uint8_t *status, *iterations;           // [n][S] (iterations nullable)
};
// Porkchop grid: P pairs x D departures x A arrivals, one cell per thread, arrival index fastest.  Endpoint k of pair p
// at departure d has position depPos + (p D + d) stride and velocity depVel + (p D + d) stride (stride 6 for [.][6]
// states, 3 for separate position and velocity blocks), likewise for arrivals.
struct PorkchopArgs {
    const double *depPos, *depVel, *arrPos, *arrVel;
    uint32_t stride;
    const uint8_t *depStatus, *arrStatus;   // nullable: every state valid
    const double *depJd, *depFr, *arrJd, *arrFr;
    uint32_t P, D, A, maxRevs;
    double mu;
    double *dv;                             // [P][D][A][2]
    uint8_t *slot, *status;                 // [P][D][A]
};
cudaError_t launch_lambert(const LambertArgs &a, cudaStream_t stream);
cudaError_t launch_porkchop(const PorkchopArgs &a, cudaStream_t stream);
}  // namespace az
#endif
