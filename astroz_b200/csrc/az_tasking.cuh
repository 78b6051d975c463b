// az_tasking.cuh -- K18: sensor tasking.  Every catalogue row is scored at every sensor slot by visibility and by the
// information one observation would give about its elements, and a greedy schedule carries each tasked row's
// covariance.  __host__ __device__, so the kernels (az_tasking.cu) and the host emulation (tests/host_emul/emul_tasking.cu)
// run this source.
//
// The catalogue is K10's: element columns, a 7 x 7 covariance P in the element fit's variables (28 words) and the model
// byte.  Sensor k is (kind radar / optical, station, sigma[4], limits[4] indexed by kTaskLimit*).  For one cell (row s,
// sensor k, slot t), at K10's tsince and jdFull = add_rn(jd, fr):
//   sets        fit_build_set_of under the row's model as K10 builds them, nvar = corr_nvar of the row's INPUT
//               covariance (the posterior keeps its zero pattern); the nominal set is propagated at every slot, the
//               stepped sets only at slots where the row is visible to at least one sensor;
//   visible     the radar elevation of obs_model above the station's geodetic horizon >= el_min and the radar range
//               <= range_max (both kinds, no refraction); optical sensors also need the object sunlit under a
//               cylindrical shadow of radius kTaskEarthRadius (r.s >= 0 or |r - (r.s) s| > R), the Sun's elevation at
//               the station (Rz(GMST) s).u <= sun_el_max, and the angle between the line of sight and s >= exclusion;
//   rows        h = obs_model of the sensor's kind under the nominal set, w = obs_weights(kind, h, sigma) (the
//               predicted elevation / declination is the partner), G[c][j] the weighted Jacobian rows of
//               obs_residual_rows with the prediction as the observation (so z = 0);
//   gain        g = 1/2 log det(I + L^T N L) = sum log diag(C), N = G^T G, P = L L^T the semi-definite Cholesky of K12
//               (corr_d2), I + L^T N L = C C^T.  It equals 1/2 log det(I + G P G^T), the mutual information of the
//               observation and the row's variables; P = 0 gives 0 exactly;
//   spread      sqrt((G P G^T)_cc) sigma_c: the predicted 1-sigma of each measured component, the azimuth / right
//               ascension as an arc on the sky;
//   posterior   P+ = L (I + L^T N L)^-1 L^T = A A^T, A = L C^-T: exactly symmetric and positive semi-definite;
//   failure     a cell whose nominal or stepped propagation fails (deep space: decay, eccentricity), or whose gain is not
//               finite, is not visible and is counted.
// The schedule: slot by slot, sensor k = 0 .. S-1 takes the row of largest g (then lowest row index) among the rows
// visible to it with g > gain_min and not taken by a lower sensor in the slot; each taken row's P becomes its P+ before
// the next slot is scored.
#pragma once

#include "az_correlate.cuh"

namespace az {

constexpr int kTaskMaxSensors = 32;
constexpr uint32_t kTaskIdle = 0xFFFFFFFFu;        // task_row of an idle sensor
constexpr double kTaskEarthRadius = 6378.137;      // km, the shadow cylinder
enum TaskLimit { kTaskElMin = 0, kTaskRangeMax = 1, kTaskSunElMax = 2, kTaskExclusion = 3 };
constexpr int kTaskCellWords = 4 + 4 + 4 * kFitVars;   // value[4], spread[4], G[4][7] of one visible cell

// One sensor, its station's frame resolved.
struct TaskSensor {
    int kind;
    ObsStation st;
    double sigma[6];   // [4..5] = +inf
    double lim[4];
};

AZ_HD void task_sensor(const uint8_t *kind, const uint32_t *station, const double *stations, const double *sigma,
                       const double *limits, int k, TaskSensor &s) {
    s.kind = kind[k];
    obs_station(stations + (size_t)station[k] * 3, s.st);
    for (int c = 0; c < 6; ++c) s.sigma[c] = c < 4 ? sigma[(size_t)k * 4 + c] : INFINITY;
    for (int c = 0; c < 4; ++c) s.lim[c] = limits[(size_t)k * 4 + c];
}

// The unit Sun direction of a slot (sun[3] of any length)
AZ_HD void task_sun(const double *sun, double (&u)[3]) {
    const double r = std::sqrt(sun[0] * sun[0] + sun[1] * sun[1] + sun[2] * sun[2]);
    for (int c = 0; c < 3; ++c) u[c] = sun[c] / r;
}

// Whether sensor s sees the nominal TEME state f0 at GMST (sg, cg), Sun direction u (optical only); h receives the
// prediction of the sensor's kind.
AZ_HD bool task_visible(const TaskSensor &s, const double (&f0)[6], double sg, double cg, const double (&u)[3],
                        double (&h)[6]) {
    double sc[6];
    obs_model(kObsRadar, f0, sg, cg, s.st, h, sc);
    if (!(h[2] >= s.lim[kTaskElMin] && h[0] <= s.lim[kTaskRangeMax])) return false;
    if (s.kind != kObsOptical) return true;
    const double r[3] = {f0[0], f0[1], f0[2]};
    const double rs = obs_dot(r, u);
    const double px = r[0] - rs * u[0], py = r[1] - rs * u[1], pz = r[2] - rs * u[2];
    if (!(rs >= 0.0 || std::sqrt(px * px + py * py + pz * pz) > kTaskEarthRadius)) return false;
    double ux = u[0], uy = u[1];
    eci_to_ecef(ux, uy, sg, cg);
    const double ue[3] = {ux, uy, u[2]};
    if (!(obs_dot(ue, s.st.u) <= std::sin(s.lim[kTaskSunElMax]))) return false;
    // the line of sight in TEME: rho = r - Rz(GMST)^T r_station
    const double sx = cg * s.st.r[0] - sg * s.st.r[1], sy = sg * s.st.r[0] + cg * s.st.r[1];
    const double rho[3] = {r[0] - sx, r[1] - sy, r[2] - s.st.r[2]};
    const double cx = rho[1] * u[2] - rho[2] * u[1], cy = rho[2] * u[0] - rho[0] * u[2],
                 cz = rho[0] * u[1] - rho[1] * u[0];
    if (!(std::atan2(std::sqrt(cx * cx + cy * cy + cz * cz), obs_dot(rho, u)) >= s.lim[kTaskExclusion])) return false;
    obs_model(kObsOptical, f0, sg, cg, s.st, h, sc);
    return true;
}

// The weighted Jacobian rows of a visible cell: G[c][j] of obs_residual_rows with h0 as the observation, from the
// stepped states f[1 .. nvar]; columns past nvar zero.
AZ_HD void task_jacobian(const TaskSensor &s, const double (*f)[6], int nvar, const double *inv, double sg, double cg,
                         const double (&h0)[6], double (&w)[6], double (&G)[4][kFitVars]) {
    obs_weights(s.kind, h0, s.sigma, w);
    const int wr = obs_wrapped(s.kind);
    for (int c = 0; c < 4; ++c)
        for (int j = 0; j < kFitVars; ++j) G[c][j] = 0.0;
    for (int j = 0; j < nvar; ++j) {
        double h[6], sc[6];
        obs_model(s.kind, f[1 + j], sg, cg, s.st, h, sc);
        for (int c = 0; c < 4; ++c) {
            const double d = c == wr ? obs_wrap(h[c] - h0[c]) : h[c] - h0[c];
            G[c][j] = w[c] != 0.0 ? d * w[c] * inv[1 + j] : 0.0;
        }
    }
}

// P = L L^T, the semi-definite Cholesky of corr_d2 (a column whose pivot is not positive is zero)
AZ_HD void task_cholesky(const double *P, double (&L)[kFitVars][kFitVars]) {
    auto Pw = [P](int j, int k) { return j <= k ? P[fit_tri(j, k)] : P[fit_tri(k, j)]; };
    for (int j = 0; j < kFitVars; ++j) {
        for (int i = 0; i < kFitVars; ++i) L[i][j] = 0.0;
        double d = Pw(j, j);
        for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
        if (d > 0.0) {
            const double ljj = std::sqrt(d);
            L[j][j] = ljj;
            for (int i = j + 1; i < kFitVars; ++i) {
                double s = Pw(j, i);
                for (int q = 0; q < j; ++q) s -= L[i][q] * L[j][q];
                L[i][j] = s / ljj;
            }
        }
    }
}

// Gain, spread and (Pplus non-null) the posterior words of one cell: G its weighted rows, L the row's Cholesky factor,
// sigma the sensor's.  False when the factorisation of I + L^T N L fails or the gain is not finite.
AZ_HD bool task_update(const double (&G)[4][kFitVars], const double (&L)[kFitVars][kFitVars], const double *sigma,
                       double &g, double (&spread)[4], double *Pplus) {
    double B[4][kFitVars];   // G L
    for (int c = 0; c < 4; ++c) {
        double v = 0.0;
        for (int q = 0; q < kFitVars; ++q) {
            double s = 0.0;
            for (int p = q; p < kFitVars; ++p) s += G[c][p] * L[p][q];
            B[c][q] = s;
            v += s * s;
        }
        spread[c] = sigma[c] < INFINITY ? std::sqrt(v) * sigma[c] : 0.0;
    }
    // I + B^T B = C C^T
    double C[kFitVars][kFitVars];
    g = 0.0;
    for (int j = 0; j < kFitVars; ++j) {
        for (int i = 0; i < kFitVars; ++i) C[i][j] = 0.0;
        for (int i = j; i < kFitVars; ++i) {
            double s = i == j ? 1.0 : 0.0;
            for (int c = 0; c < 4; ++c) s += B[c][i] * B[c][j];
            for (int q = 0; q < j; ++q) s -= C[i][q] * C[j][q];
            if (i == j) {
                if (!(s > 0.0)) return false;
                C[j][j] = std::sqrt(s);
            } else {
                C[i][j] = s / C[j][j];
            }
        }
        g += std::log(C[j][j]);
    }
    if (!(std::fabs(g) < INFINITY)) return false;
    if (!Pplus) return true;
    double A[kFitVars][kFitVars];   // row i: C^-1 (row i of L)
    for (int i = 0; i < kFitVars; ++i)
        for (int j = 0; j < kFitVars; ++j) {
            double s = L[i][j];
            for (int q = 0; q < j; ++q) s -= C[j][q] * A[i][q];
            A[i][j] = s / C[j][j];
        }
    for (int i = 0; i < kFitVars; ++i)
        for (int k = i; k < kFitVars; ++k) {
            double s = 0.0;
            for (int q = 0; q < kFitVars; ++q) s += A[i][q] * A[k][q];
            Pplus[fit_tri(i, k)] = s;
        }
    return true;
}

// One (row, slot) against every sensor: eval the row's set evaluator (fit_accumulate_model's), P the row's current
// covariance words, u the slot's unit Sun direction (read by optical sensors only).  emit(k, gain, h, spread, G) for
// each visible cell; the return value's bit k is set when cell k is visible.  failed receives the failed cells.
template <typename EvalFn, typename EmitFn>
AZ_HD uint32_t task_score(EvalFn eval, int nvar, const double *inv, double epochJd, double jdFull,
                          const TaskSensor *sensors, int S, const double (&u)[3], const double *P, EmitFn emit,
                          uint32_t &failed) {
    const double ts[1] = {mul_rn(sub_rn(jdFull, epochJd), 1440.0)};
    double f[kFitSets][6];
    failed = 0;
    if (!eval(0, jdFull, ts, f[0])) {
        failed = (uint32_t)S;
        return 0;
    }
    double sg, cg;
    sincos_full(pairs_gmst(jdFull), sg, cg);
    uint32_t seen = 0;
    for (int k = 0; k < S; ++k) {
        double h[6];
        if (task_visible(sensors[k], f[0], sg, cg, u, h)) seen |= 1u << k;
    }
    if (!seen) return 0;
    bool ok = true;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < nvar; ++j) ok = eval(1 + j, jdFull, ts, f[1 + j]) && ok;
    if (!ok) {
        for (uint32_t b = seen; b; b &= b - 1) ++failed;
        return 0;
    }
    double L[kFitVars][kFitVars];
    task_cholesky(P, L);
    uint32_t visible = 0;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int k = 0; k < S; ++k) {
        if (!(seen >> k & 1u)) continue;
        double h[6], w[6], G[4][kFitVars], spread[4], g;
        task_visible(sensors[k], f[0], sg, cg, u, h);
        task_jacobian(sensors[k], f, nvar, inv, sg, cg, h, w, G);
        if (!task_update(G, L, sensors[k].sigma, g, spread, nullptr)) {
            ++failed;
            continue;
        }
        visible |= 1u << k;
        emit(k, g, h, spread, G);
    }
    return visible;
}

// Device scratch of the call: the sensors, each row's built sets (a near-earth or a deep-space record in one slot of
// kTaskRowBytes), inv and nvar, per (sensor, row) the gain and the cell words, per row the slot that last took it.
AZ_HD size_t task_row_bytes() {
    const size_t near = sizeof(double) * kFitSets * kSgp4Cols;
    const size_t deep = sizeof(Sdp4Sat) * kFitSets + sizeof(double2) * kFitSets * 2 * kFitLatticeNodes;
    return ((near > deep ? near : deep) + 15) & ~size_t(15);
}

AZ_HD size_t task_scratch_bytes(uint32_t n, uint32_t S) {
    const size_t sensors = ((sizeof(TaskSensor) * S) + 15) & ~size_t(15);
    return sensors + (size_t)n * task_row_bytes() + (size_t)n * kFitSets * 8 + (size_t)n * 4 + (size_t)S * n * 8 +
           (size_t)S * n * kTaskCellWords * 8 + (size_t)n * 4 + 16;
}

}  // namespace az
