// az_obs.cuh -- the measurement layer of the K8 observation fits (az_fit_obs.cu) and of astroz_cuda_observe: from a
// TEME state at an observation's time to what a sensor reports.  __host__ __device__, so the kernels and the host
// emulation (tests/host_emul/emul_fit_obs.cu) run this source.
//
// Kinds (ASTROZ_OBS_*), values h[obs_count(kind)]:
//   0 TEME state    x y z [km], vx vy vz [km/s]: the state itself (the observation of astroz_cuda_fit_elements);
//   1 ECEF state    r_ecef = Rz(GMST) r, the rotation propagate_pairs applies for its ECEF output, with GMST = pairs_gmst
//                   of the observation's own jd + fr; v_ecef = Rz(GMST) v - omega x r_ecef, the Earth-fixed velocity a
//                   GPS receiver reports.  The library's ECEF output mode follows the reference and leaves omega x r out;
//                   this kind does not.  omega = 360.98564736629 deg/day, the rate of the GMST polynomial;
//   2 radar         range [km], azimuth [rad, from north through east, in [0, 2 pi)], elevation [rad], range-rate
//                   [km/s], in the geodetic horizon frame of the station: rho = r_ecef - r_station, range-rate =
//                   rho . rho_dot / |rho| with rho_dot = v_ecef of kind 1;
//   3 optical       topocentric right ascension [rad, in [0, 2 pi)] and declination [rad] in TEME: rho = r_teme -
//                   Rz(GMST)^T r_station.
// Stations are (geodetic latitude deg, longitude deg, height km) on WGS84, the ellipsoid ecef_to_geodetic uses.
// Observations are geometric and instantaneous: no light time, no aberration, no refraction.  Polar motion and the
// TEME -> GCRF rotation are the caller's: optical angles must already be in TEME.
//
// Residuals are (observed - model) / sigma per component.  The azimuth and right-ascension differences are wrapped to
// (-pi, pi] and multiplied by the cosine of the OBSERVED elevation / declination, so their sigma is an arc on the sky
// and the weight does not move with the trial set; the Jacobian's differences are wrapped the same way.  A component
// with sigma = +inf carries no information: it adds nothing to the cost, the sums, the residual count or the floor.
#pragma once

#include "az_fit.cuh"

namespace az {

enum ObsKind : uint8_t { kObsTemeState = 0, kObsEcefState = 1, kObsRadar = 2, kObsOptical = 3 };
constexpr int kObsKinds = 4;
constexpr int kObsValues = 6;   // value[m][6], sigma[m][6]: components past a kind's count are ignored

// Earth rotation rate of pairs_gmst's polynomial: 360.98564736629 deg/day in rad/s
constexpr double kObsOmega = 360.98564736629 * detail::kDeg / 86400.0;

AZ_HD int obs_count(int kind) { return kind <= kObsEcefState ? 6 : kind == kObsRadar ? 4 : 2; }
AZ_HD bool obs_uses_station(int kind) { return kind == kObsRadar || kind == kObsOptical; }
// The wrapped angle of a kind (radar azimuth, optical right ascension) and the component whose cosine scales it
// (elevation, declination); -1 for the state kinds.
AZ_HD int obs_wrapped(int kind) { return kind == kObsRadar ? 1 : kind == kObsOptical ? 0 : -1; }
AZ_HD int obs_partner(int kind) { return kind == kObsRadar ? 2 : 1; }

// d reduced to (-pi, pi]
AZ_HD double obs_wrap(double d) { return d - kTwoPi * std::ceil((d - kPi) / kTwoPi); }

// A station's ECEF position and the east / north / up unit vectors of its geodetic horizon.
struct ObsStation {
    double r[3];
    double e[3], n[3], u[3];
};

AZ_HD void obs_station(const double *llh, ObsStation &st) {
    constexpr double a = 6378.137;
    constexpr double f = 1.0 / 298.257223563;
    constexpr double e2 = 2.0 * f - f * f;
    const double lat = llh[0] * detail::kDeg, lon = llh[1] * detail::kDeg, h = llh[2];
    const double sp = std::sin(lat), cp = std::cos(lat), sl = std::sin(lon), cl = std::cos(lon);
    const double N = a / std::sqrt(1.0 - e2 * sp * sp);
    st.r[0] = (N + h) * cp * cl;
    st.r[1] = (N + h) * cp * sl;
    st.r[2] = (N * (1.0 - e2) + h) * sp;
    st.e[0] = -sl;      st.e[1] = cl;       st.e[2] = 0.0;
    st.n[0] = -sp * cl; st.n[1] = -sp * sl; st.n[2] = cp;
    st.u[0] = cp * cl;  st.u[1] = cp * sl;  st.u[2] = sp;
}

AZ_HD double obs_dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
AZ_HD double obs_angle(double y, double x) {   // atan2 in [0, 2 pi)
    const double t = std::atan2(y, x);
    return t < 0.0 ? t + kTwoPi : t;
}

// h(kind, TEME state f, GMST sine / cosine, station) -> h[obs_count(kind)] (the rest zero).  sc[c] is the scale of
// component c's rounding floor where it is not |observed value|: |rho dot| for the range-rate, and |r| / |rho| rad for
// the angles -- the angle through which a position rounding of kFitNoise |r| turns the line of sight.
AZ_HD void obs_model(int kind, const double (&f)[6], double sg, double cg, const ObsStation &st, double (&h)[6],
                     double (&sc)[6]) {
    for (int c = 0; c < 6; ++c) h[c] = sc[c] = 0.0;
    if (kind == kObsTemeState) {
        for (int c = 0; c < 6; ++c) h[c] = f[c];
        return;
    }
    if (kind == kObsOptical) {
        const double sx = cg * st.r[0] - sg * st.r[1], sy = sg * st.r[0] + cg * st.r[1];
        const double rho[3] = {f[0] - sx, f[1] - sy, f[2] - st.r[2]};
        const double q = std::sqrt(rho[0] * rho[0] + rho[1] * rho[1]);
        h[0] = obs_angle(rho[1], rho[0]);
        h[1] = std::atan2(rho[2], q);
        sc[0] = sc[1] = std::sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]) / std::sqrt(obs_dot(rho, rho));
        return;
    }
    double x = f[0], y = f[1], vx = f[3], vy = f[4];
    eci_to_ecef(x, y, sg, cg);
    eci_to_ecef(vx, vy, sg, cg);
    vx += kObsOmega * y;   // - omega x r_ecef, omega along +z
    vy -= kObsOmega * x;
    if (kind == kObsEcefState) {
        h[0] = x; h[1] = y; h[2] = f[2];
        h[3] = vx; h[4] = vy; h[5] = f[5];
        return;
    }
    const double rho[3] = {x - st.r[0], y - st.r[1], f[2] - st.r[2]};
    const double rd[3] = {vx, vy, f[5]};
    const double E = obs_dot(rho, st.e), N = obs_dot(rho, st.n), U = obs_dot(rho, st.u);
    const double range = std::sqrt(obs_dot(rho, rho));
    h[0] = range;
    h[1] = obs_angle(E, N);
    h[2] = std::atan2(U, std::sqrt(E * E + N * N));
    h[3] = obs_dot(rho, rd) / range;
    sc[1] = sc[2] = std::sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]) / range;
    sc[3] = std::sqrt(obs_dot(rd, rd));
}

// One observation's weights: w[c] = 1 / sigma[c], times the cosine of the observed elevation / declination for the
// wrapped angle; 0 for a component that is not used (sigma = +inf, or past the kind's count).  Returns the number of
// used components.
AZ_HD int obs_weights(int kind, const double *value, const double *sigma, double (&w)[6]) {
    const int count = obs_count(kind), wr = obs_wrapped(kind);
    int used = 0;
    for (int c = 0; c < 6; ++c) {
        w[c] = 0.0;
        if (c < count && sigma[c] < INFINITY) {
            w[c] = 1.0 / sigma[c];
            if (c == wr) w[c] *= std::cos(value[obs_partner(kind)]);
            ++used;
        }
    }
    return used;
}

// The frame quantities of one observation: the sine and cosine of GMST at jdFull (kinds 1-3) and its station
// (kinds 2, 3; stations[3 * k] = lat, lon, h of station k).
AZ_HD void obs_frame(int kind, double jdFull, const double *llh, double &sg, double &cg, ObsStation &st) {
    sg = 0.0;
    cg = 1.0;
    if (kind != kObsTemeState) sincos_full(pairs_gmst(jdFull), sg, cg);
    if (obs_uses_station(kind)) obs_station(llh, st);
    else st = ObsStation{};
}

// One observation's weighted residual row and weighted Jacobian rows: observation (kind, value[6], w[6] from
// obs_weights, frame) against the model under set 0 and sets 1..nvar (eval as fit_accumulate_model's).  r[c] =
// (observed - model) w[c], the azimuth / right-ascension difference wrapped; J entry (j, c) at J[(j * 6 + c) * stride]
// = the same difference between set 1 + j and set 0, times w[c] inv[1 + j].  obs receives the used observed values and
// sc the nominal model's floor scales (obs_model).  The element fit's rows (fit_accumulate_obs) and K12's pair rows
// (az_correlate.cuh) are these.  Returns false when a cell failed.
template <typename EvalFn>
AZ_HD bool obs_residual_rows(EvalFn eval, int nvar, const double *inv, double jdFull, double epochJd, int kind,
                             const double *value, const double (&w)[6], double sg, double cg, const ObsStation &st,
                             double (&obs)[6], double (&sc)[6], double (&r)[6], double *J, int stride) {
    const double ts[1] = {mul_rn(sub_rn(jdFull, epochJd), 1440.0)};
    bool ok = true;
    const int wr = obs_wrapped(kind);
    double f0[6], h0[6];
    for (int c = 0; c < 6; ++c) obs[c] = w[c] != 0.0 ? value[c] : 0.0;
    ok = eval(0, jdFull, ts, f0) && ok;
    obs_model(kind, f0, sg, cg, st, h0, sc);
    for (int c = 0; c < 6; ++c) {
        const double d = c == wr ? obs_wrap(obs[c] - h0[c]) : obs[c] - h0[c];
        r[c] = w[c] != 0.0 ? d * w[c] : 0.0;
    }
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < nvar; ++j) {
        double f[6], h[6], scj[6];
        ok = eval(1 + j, jdFull, ts, f) && ok;
        obs_model(kind, f, sg, cg, st, h, scj);
        for (int c = 0; c < 6; ++c) {
            const double d = c == wr ? obs_wrap(h[c] - h0[c]) : h[c] - h0[c];
            J[(j * 6 + c) * stride] = w[c] != 0.0 ? d * w[c] * inv[1 + j] : 0.0;
        }
    }
    return ok;
}

// fit_accumulate_model with the measurement layer: obs_residual_rows, then the cost, floor and normal sums.
// Components are summed in fit_accumulate_model's order, (0, 3), (1, 4), (2, 5); pos2 and vel2 are formed only on the
// K8 path below.
template <typename EvalFn>
AZ_HD bool fit_accumulate_obs(EvalFn eval, int nvar, const double *inv, double jdFull, double epochJd, int kind,
                              const double *value, const double (&w)[6], double sg, double cg, const ObsStation &st,
                              double *J, double *acc, int stride) {
    // A TEME state with one position sigma and one velocity sigma (or none) is K8's observation: its own code, so
    // such a fit is astroz_cuda_fit_elements' to the bit whatever the compiler contracts.
    if (kind == kObsTemeState && w[0] != 0.0 && w[0] == w[1] && w[1] == w[2] && w[3] == w[4] && w[4] == w[5])
        return fit_accumulate_model(eval, nvar, inv, jdFull, epochJd, value, w[3] != 0.0 ? value + 3 : nullptr, w[0],
                                    w[3], J, acc, stride);
    double obs[6], sc[6], r[6];
    const bool ok = obs_residual_rows(eval, nvar, inv, jdFull, epochJd, kind, value, w, sg, cg, st, obs, sc, r, J,
                                      stride);
    {
        double F = acc[0], fl = acc[3 * stride];
        for (int c = 0; c < 3; ++c) {   // components in the order (0, 3), (1, 4), (2, 5): fit_accumulate_model's sums
            for (int q = c; q < 6; q += 3) {
                if (w[q] == 0.0) continue;
                F += r[q] * r[q];
                const bool scaled = sc[q] != 0.0;
                const double fq = (scaled ? sc[q] : obs[q]) * w[q] * kFitNoise;
                fl += fq * fq;
            }
        }
        acc[0] = F;
        acc[3 * stride] = fl;
    }
    fit_accumulate_normal(nvar, r, J, acc, stride);
    return ok;
}

// Covariance of the fitted variables at the final iterate: (J^T W J)^-1 over the nvar variables, by Cholesky on the
// unit-diagonal scaling fit_solve uses.  cov = its upper triangle in fit_tri order (kFitN words), the held B* row and
// column zero.  Returns false, with cov all zeros, when the normal matrix is not positive definite.
AZ_HD bool fit_covariance(const FitSums &s, int nvar, double (&cov)[kFitN]) {
    double sc[kFitVars], L[kFitVars][kFitVars], Li[kFitVars][kFitVars];
    for (int q = 0; q < kFitN; ++q) cov[q] = 0.0;
    for (int j = 0; j < nvar; ++j) {
        const double njj = s.N[fit_tri(j, j)];
        if (!(njj > 0.0) || !(njj < INFINITY)) return false;
        sc[j] = 1.0 / std::sqrt(njj);
    }
    for (int j = 0; j < nvar; ++j) {
        for (int k = 0; k <= j; ++k) {
            double a = (k == j) ? 1.0 : s.N[fit_tri(k, j)] * sc[j] * sc[k];
            for (int q = 0; q < k; ++q) a -= L[j][q] * L[k][q];
            if (k == j) {
                if (!(a > 0.0) || !(a < INFINITY)) return false;
                L[j][j] = std::sqrt(a);
            } else {
                L[j][k] = a / L[k][k];
            }
        }
    }
    for (int j = 0; j < nvar; ++j) {   // Li = L^-1, lower triangular
        Li[j][j] = 1.0 / L[j][j];
        for (int k = 0; k < j; ++k) {
            double b = 0.0;
            for (int q = k; q < j; ++q) b -= L[j][q] * Li[q][k];
            Li[j][k] = b / L[j][j];
        }
    }
    for (int j = 0; j < nvar; ++j)     // (D N D)^-1 = Li^T Li, then scaled back by D
        for (int k = j; k < nvar; ++k) {
            double a = 0.0;
            for (int q = k; q < nvar; ++q) a += Li[q][j] * Li[q][k];
            cov[fit_tri(j, k)] = a * sc[j] * sc[k];
        }
    return true;
}

}  // namespace az
