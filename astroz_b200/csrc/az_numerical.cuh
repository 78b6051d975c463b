// az_numerical.cuh -- per-state cores of K7, numerical propagation of a batch of initial states: what
// propagate_numerical(state, t0, duration, dt, mu, ...) computes for one state (bindings/python/src/propagator.zig:13-193),
// one state per thread.  __host__ __device__, so tests/host_emul runs the same arithmetic on the CPU.
//
// The integrator (RK4 / Dormand-Prince 8(7)) and the force set (two-body, + J2, + drag, + J2 + drag) are template
// parameters: each of the eight specialisations carries only its own stages and force terms.  Every operation follows
// the reference's order (the file is compiled without FMA contraction), so a two-body or J2 trajectory equals the
// scalar restatement bit for bit; the step-growth factor (errNorm^-1/8, three square roots here, pow in the reference)
// and exp (drag) round differently.
#pragma once

#include "az_math.cuh"

namespace az {

// force-set bits (ASTROZ_FORCE_*); two-body is always on
constexpr int kForceJ2 = 1, kForceDrag = 2;
// integrators (ASTROZ_INTEGRATOR_*)
constexpr int kIntRk4 = 0, kIntDp87 = 1;
// per-state status bytes (ASTROZ_NUMERICAL_*)
constexpr uint8_t kNumOk = 0, kNumStopped = 1, kNumSubstepLimit = 2, kNumNonFinite = 3;

// Exponential atmosphere of the binding: earth's sea-level density and scale height (src/constants.zig:163-164) and the
// 1500 km cutoff (bindings/python/src/propagator.zig:11)
constexpr double kDragRho0 = 1.225, kDragScaleHeight = 7.249, kDragMaxAltitude = 1500.0;
// DormandPrince87 step control (src/propagators/Integrator.zig:62-69)
constexpr double kDpHMin = 0.001, kDpHMax = 3600.0, kDpSafety = 0.9, kDpHStart = 60.0;
constexpr uint32_t kDpMaxSubsteps = 10000;

// Prince & Dormand (1981), RK8(7)13M: nodes c, stage weights a (row i uses stages j < i), the 8th-order weights b8
// (the propagated solution) and the 7th-order weights b7 (the error estimate).
struct Dp87Tableau {
    double c[13];
    double a[13][12];
    double b8[13];
    double b7[13];
};
// clang-format off
#define AZ_DP87_TABLEAU {                                                                                              \
    {0.0, 1.0 / 18.0, 1.0 / 12.0, 1.0 / 8.0, 5.0 / 16.0, 3.0 / 8.0, 59.0 / 400.0, 93.0 / 200.0,                        \
     5490023248.0 / 9719169821.0, 13.0 / 20.0, 1201146811.0 / 1299019798.0, 1.0, 1.0},                                 \
    {{0},                                                                                                              \
     {1.0 / 18.0},                                                                                                     \
     {1.0 / 48.0, 1.0 / 16.0},                                                                                         \
     {1.0 / 32.0, 0, 3.0 / 32.0},                                                                                      \
     {5.0 / 16.0, 0, -75.0 / 64.0, 75.0 / 64.0},                                                                       \
     {3.0 / 80.0, 0, 0, 3.0 / 16.0, 3.0 / 20.0},                                                                       \
     {29443841.0 / 614563906.0, 0, 0, 77736538.0 / 692538347.0, -28693883.0 / 1125000000.0,                           \
      23124283.0 / 1800000000.0},                                                                                      \
     {16016141.0 / 946692911.0, 0, 0, 61564180.0 / 158732637.0, 22789713.0 / 633445777.0,                             \
      545815736.0 / 2771057229.0, -180193667.0 / 1043307555.0},                                                        \
     {39632708.0 / 573591083.0, 0, 0, -433636366.0 / 683701615.0, -421739975.0 / 2616292301.0,                        \
      100302831.0 / 723423059.0, 790204164.0 / 839813087.0, 800635310.0 / 3783071287.0},                               \
     {246121993.0 / 1340847787.0, 0, 0, -37695042795.0 / 15268766246.0, -309121744.0 / 1061227803.0,                  \
      -12992083.0 / 490766935.0, 6005943493.0 / 2108947869.0, 393006217.0 / 1396673457.0,                              \
      123872331.0 / 1001029789.0},                                                                                     \
     {-1028468189.0 / 846180014.0, 0, 0, 8478235783.0 / 508512852.0, 1311729495.0 / 1432422823.0,                     \
      -10304129995.0 / 1701304382.0, -48777925059.0 / 3047939560.0, 15336726248.0 / 1032824649.0,                      \
      -45442868181.0 / 3398467696.0, 3065993473.0 / 597172653.0},                                                      \
     {185892177.0 / 718116043.0, 0, 0, -3185094517.0 / 667107341.0, -477755414.0 / 1098053517.0,                      \
      -703635378.0 / 230739211.0, 5731566787.0 / 1027545527.0, 5232866602.0 / 850066563.0,                             \
      -4093664535.0 / 808688257.0, 3962137247.0 / 1805957418.0, 65686358.0 / 487910083.0},                             \
     {403863854.0 / 491063109.0, 0, 0, -5068492393.0 / 434740067.0, -411421997.0 / 543043805.0,                       \
      652783627.0 / 914296604.0, 11173962825.0 / 925320556.0, -13158990841.0 / 6184727034.0,                           \
      3936647629.0 / 1978049680.0, -160528059.0 / 685178525.0, 248638103.0 / 1413531060.0, 0}},                        \
    {14005451.0 / 335480064.0, 0, 0, 0, 0, -59238493.0 / 1068277825.0, 181606767.0 / 758867731.0,                      \
     561292985.0 / 797845732.0, -1041891430.0 / 1371343529.0, 760417239.0 / 1151165299.0,                              \
     118820643.0 / 751138087.0, -528747749.0 / 2220607170.0, 1.0 / 4.0},                                               \
    {13451932.0 / 455176623.0, 0, 0, 0, 0, -808719846.0 / 976000145.0, 1757004468.0 / 5645159321.0,                    \
     656045339.0 / 265891186.0, -3867574721.0 / 1518517206.0, 465885868.0 / 322736535.0,                               \
     53011238.0 / 667516719.0, 2.0 / 45.0, 0}}
// clang-format on
// Almost every weight has a non-zero low word: they are read from constant memory, warp-uniform broadcasts that the
// DFMA / DMUL takes as a c[bank][offset] operand (the K1 rule, az_math.cuh).
static __constant__ Dp87Tableau kDp87Dev = AZ_DP87_TABLEAU;
static const Dp87Tableau kDp87Host = AZ_DP87_TABLEAU;
#ifdef __CUDA_ARCH__
#define AZ_DP87(field) (::az::kDp87Dev.field)
#else
#define AZ_DP87(field) (::az::kDp87Host.field)
#endif

// The tableau's zero pattern, as compile-time facts for the unrolled stage loops (a zero weight is skipped, as the
// reference skips it): stages 1 and 2 feed only rows 2-4, a[12][11] = 0, b8 and b7 have no weight on stages 1-4, b7
// none on stage 12.  tests/test_numerical_host_emulation.py checks these against the table.
AZ_HD constexpr bool dp87_a_nz(int i, int j) {
    return j < i && !(j == 1 && i != 2) && !(j == 2 && i != 3 && i != 4) && !(i == 3 && j == 1) &&
           !(i == 12 && j == 11);
}
AZ_HD constexpr bool dp87_b8_nz(int i) { return i == 0 || i >= 5; }
AZ_HD constexpr bool dp87_b7_nz(int i) { return i == 0 || (i >= 5 && i <= 11); }

struct NumParams {
    double mu, j2, rEq;  // km^3/s^2, -, km
    double rtol, atol;   // DP87 tolerances
};
struct DragBody {
    double cd, area, mass;  // -, m^2, kg
};

// Accelerations in the order of the binding's force list (propagator.zig:119-146): TwoBody (ForceModel.zig:49-55), J2
// (:67-79), Drag (:95-110).  Several models are summed by Composite (:365-374) into a total that starts at zero;
// a single model is returned as it is.
template <int kForces>
AZ_HD void accel(const double s[6], const NumParams &p, const DragBody &d, double acc[3]) {
    const double x = s[0], y = s[1], z = s[2];
    const double r = sqrt(x * x + y * y + z * z);
    const double f = -p.mu / (r * r * r);
    if (kForces == 0) {
        acc[0] = f * x;
        acc[1] = f * y;
        acc[2] = f * z;
        return;
    }
    acc[0] = 0.0 + f * x;
    acc[1] = 0.0 + f * y;
    acc[2] = 0.0 + f * z;
    if (kForces & kForceJ2) {
        const double r2 = x * x + y * y + z * z;
        const double rj = sqrt(r2);
        const double fj = -1.5 * p.j2 * p.mu * p.rEq * p.rEq / (r2 * r2 * rj);
        const double z2r2 = (z * z) / r2;
        acc[0] += fj * x * (5.0 * z2r2 - 1.0);
        acc[1] += fj * y * (5.0 * z2r2 - 1.0);
        acc[2] += fj * z * (5.0 * z2r2 - 3.0);
    }
    if (kForces & kForceDrag) {
        // a model returning zeros adds nothing to a total that is never -0
        const double alt = r - p.rEq;
        if (!(alt > kDragMaxAltitude)) {
            const double vx = s[3], vy = s[4], vz = s[5];
            const double v = sqrt(vx * vx + vy * vy + vz * vz);
            if (!(v < 1e-10)) {
                const double rho = kDragRho0 * exp(-alt / kDragScaleHeight);
                const double fd = -0.5 * d.cd * d.area * rho * v * 1e3 / d.mass;
                acc[0] += fd * vx / v;
                acc[1] += fd * vy / v;
                acc[2] += fd * vz / v;
            }
        }
    }
}

// The integrators below take the force as a policy F: f(s, acc) writes the acceleration at state s, and
// f.interval(k) is called before output interval k is integrated.  FixedForces is the binding's force list of the
// eight fixed specialisations; ListForces (further down) is a caller's ordered model list.
template <int kForces>
struct FixedForces {
    const NumParams &p;
    const DragBody &d;
    AZ_HD void operator()(const double s[6], double acc[3]) const { accel<kForces>(s, p, d, acc); }
    AZ_HD void interval(uint32_t) {}
};

// derivative of Integrator.zig:47-50 / :261-264: (velocity, acceleration)
template <class F>
AZ_HD void deriv(const double s[6], const F &f, double k[6]) {
    double a[3];
    f(s, a);
    k[0] = s[3];
    k[1] = s[4];
    k[2] = s[5];
    k[3] = a[0];
    k[4] = a[1];
    k[5] = a[2];
}

// Rk4.step (Integrator.zig:28-45); y is replaced by the state after dt
template <class F>
AZ_HD void rk4_step(double y[6], double dt, const F &f) {
    double k1[6], k2[6], k3[6], k4[6], s[6];
    const double half = 0.5 * dt;
    deriv(y, f, k1);
#pragma unroll
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k1[c] * half;
    deriv(s, f, k2);
#pragma unroll
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k2[c] * half;
    deriv(s, f, k3);
#pragma unroll
    for (int c = 0; c < 6; ++c) s[c] = y[c] + k3[c] * dt;
    deriv(s, f, k4);
    const double factor = dt / 6.0;
#pragma unroll
    for (int c = 0; c < 6; ++c) y[c] = y[c] + factor * (k1[c] + 2.0 * k2[c] + 2.0 * k3[c] + k4[c]);
}

// One attempt of DormandPrince87.adaptiveStep (Integrator.zig:190-259) from y with step h: y8 receives the 8th-order
// solution, the return value is errNorm.  The 8th- and 7th-order sums are accumulated as each stage is formed; that is
// the reference's order of additions (stage by stage, zero weights skipped), so only stages still read by later rows
// stay live.
template <class F>
AZ_HD double dp87_attempt(const double y[6], double h, const F &f, const NumParams &p, double y8[6]) {
    double k[13][6];
    double y7[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) y8[c] = y7[c] = y[c];
#pragma unroll
    for (int i = 0; i < 13; ++i) {
        double ys[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) ys[c] = y[c];
#pragma unroll
        for (int j = 0; j < 12; ++j) {
            if (dp87_a_nz(i, j)) {
                const double ah = AZ_DP87(a[i][j]) * h;
#pragma unroll
                for (int c = 0; c < 6; ++c) ys[c] = ys[c] + ah * k[j][c];
            }
        }
        deriv(ys, f, k[i]);
        if (dp87_b8_nz(i)) {
            const double bh = AZ_DP87(b8[i]) * h;
#pragma unroll
            for (int c = 0; c < 6; ++c) y8[c] = y8[c] + bh * k[i][c];
        }
        if (dp87_b7_nz(i)) {
            const double bh = AZ_DP87(b7[i]) * h;
#pragma unroll
            for (int c = 0; c < 6; ++c) y7[c] = y7[c] + bh * k[i][c];
        }
    }
    double e = 0.0;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const double scale = p.atol + p.rtol * fmax(fabs(y[c]), fabs(y8[c]));
        const double se = (y8[c] - y7[c]) / scale;
        e += se * se;
    }
    return sqrt(e / 6.0);
}

// hNew of adaptiveStep (Integrator.zig:244-252).  errNorm^(-1/8) is formed as three correctly rounded square roots
// (the same bits on host and device; the reference's pow differs from it in the last place).  fmin / fmax return the
// non-NaN operand, as Zig's @min / @max do, so a NaN errNorm shrinks the step tenfold.
AZ_HD double dp87_next_h(double h, double errNorm) {
    double hNew;
    if (errNorm < 1e-10) {
        hNew = h * 5.0;
    } else {
        const double factor = kDpSafety * sqrt(sqrt(sqrt(1.0 / errNorm)));
        hNew = h * fmin(5.0, fmax(0.1, factor));
    }
    hNew = fmin(hNew, kDpHMax);
    return fmax(hNew, kDpHMin);
}

// DormandPrince87.step (Integrator.zig:154-182) over one output interval of length dt, carrying hCur from interval to
// interval.  Returns kNumOk, kNumSubstepLimit (10,000 accepted substeps and the interval not finished: y is where the
// reference leaves it) or kNumStopped: an attempt rejected at h == hMin, which the reference retries with the same y
// and h forever (this is also where a non-finite errNorm ends).  counts[0] / counts[1] add accepted / rejected attempts.
template <class F>
AZ_HD uint8_t dp87_interval(double y[6], double &hCur, double dt, const F &f, const NumParams &p,
                            uint64_t counts[2]) {
    double remaining = dt;
    uint32_t substeps = 0;
    double h = fmin(hCur, remaining);
    while (remaining > 1e-14 && substeps < kDpMaxSubsteps) {
        h = fmin(h, remaining);
        h = fmax(h, kDpHMin);
        double y8[6];
        const double errNorm = dp87_attempt(y, h, f, p, y8);
        const double hNew = dp87_next_h(h, errNorm);
        if (errNorm <= 1.0) {
#pragma unroll
            for (int c = 0; c < 6; ++c) y[c] = y8[c];
            remaining -= h;
            ++substeps;
            ++counts[0];
        } else {
            ++counts[1];
            if (h == kDpHMin) {
                hCur = hNew;
                return kNumStopped;
            }
        }
        h = hNew;
    }
    hCur = h;
    return (remaining > 1e-14) ? kNumSubstepLimit : kNumOk;
}

AZ_HD bool all_finite(const double y[6]) {
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 6; ++c) ok = ok && isfinite(y[c]);
    return ok;
}

// The step sizes of the sampling loop `while (t < t_end) { step = min(dt, t_end - t); ...; t += step; }`
// (src/propagators/Propagator.zig:39-45), as the host's loop produced them: every step is dt until t_end - t < dt, then a
// tail of short steps.  The tail is one step, or two when t_end - t was rounded (after one short step t is within an ulp
// of t_end, and the next difference is exact); kMaxTail leaves room.  Small enough to travel as a kernel parameter, so no
// table has to be uploaded before a launch.
constexpr uint32_t kMaxTail = 4;
struct StepTable {
    double dt;
    uint32_t nFull, nTail;    // K = nFull + nTail steps
    double tail[kMaxTail];
    AZ_HD double step(uint32_t k) const { return k < nFull ? dt : tail[k - nFull]; }
};
// Append the loop's next step to t (start from StepTable{dt, 0, 0, {}}); false when the steps do not have the shape above.
inline bool step_table_push(StepTable &t, double step) {
    if (step == t.dt && t.nTail == 0) return ++t.nFull != 0;  // 32-bit wrap: more steps than K7 counts
    if (t.nTail == kMaxTail) return false;
    t.tail[t.nTail++] = step;
    return true;
}

// One state's trajectory (Propagator.propagate, src/propagators/Propagator.zig:22-48): y0 at out[0..6), then the state
// after each of the K intervals of `steps` (the sampling loop's step sizes, built once on the host) at out[6 (k + 1)).
// A stopped state's later samples are zero-filled.  Returns the status byte; counts[2] receives accepted / rejected
// steps (RK4: one accepted step per interval).  f is the force policy; f.interval(k) runs before interval k.
template <int kInt, class F>
AZ_HD uint8_t propagate_with(const double y0[6], F &f, const NumParams &p, const StepTable &steps, double *out,
                             uint64_t counts[2]) {
    const uint32_t K = steps.nFull + steps.nTail;
    double y[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) out[c] = y[c] = y0[c];
    counts[0] = counts[1] = 0;
    uint8_t status = kNumOk;
    double hCur = kDpHStart;
    for (uint32_t k = 0; k < K; ++k) {
        const double dt = steps.step(k);
        f.interval(k);
        if (kInt == kIntRk4) {
            rk4_step(y, dt, f);
            ++counts[0];
            if (status == kNumOk && !all_finite(y)) status = kNumNonFinite;
        } else {
            const uint8_t st = dp87_interval(y, hCur, dt, f, p, counts);
            if (st == kNumStopped) {
                for (size_t w = (size_t)(k + 1) * 6; w < (size_t)(K + 1) * 6; ++w) out[w] = 0.0;
                return kNumStopped;
            }
            if (st == kNumSubstepLimit) status = kNumSubstepLimit;
        }
        double *o = out + (size_t)(k + 1) * 6;
#pragma unroll
        for (int c = 0; c < 6; ++c) o[c] = y[c];
    }
    return status;
}

// The fixed force sets of the eight K7 kernels
template <int kInt, int kForces>
AZ_HD uint8_t propagate_state(const double y0[6], const DragBody &d, const NumParams &p, const StepTable &steps,
                              double *out, uint64_t counts[2]) {
    FixedForces<kForces> f{p, d};
    return propagate_with<kInt>(y0, f, p, steps, out, counts);
}

// ---- model lists: the force models of the reference's propagators module (src/propagators/ForceModel.zig) ----------
// kinds (ASTROZ_MODEL_*) and descriptor flags (ASTROZ_MODEL_PER_STATE_*, ASTROZ_MODEL_POS_TABLE)
constexpr int32_t kModelTwoBody = 0, kModelJ2 = 1, kModelJ3 = 2, kModelJ4 = 3, kModelDrag = 4, kModelImprovedDrag = 5,
                  kModelSrp = 6, kModelThirdBody = 7, kModelKinds = 8;
constexpr uint32_t kModelPerStateC = 1, kModelPerStateArea = 2, kModelPerStateMass = 4, kModelPosTable = 8;
constexpr uint32_t kMaxModels = 16;
// SolarRadiationPressure: pressure at 1 AU [N/m^2] and the AU [km] (src/constants.zig:27-28); ImprovedDrag: the
// atmosphere's rotation rate [rad/s] (ForceModel.zig:292)
constexpr double kSrpPressure = 4.56e-6, kAuKm = 1.495978707e8, kEarthOmega = 7.2921150e-5;

// One model of a list, the layout of astroz_force_model_t.  c is cd (Drag, ImprovedDrag) or cr (SRP); c_arr / area_arr /
// mass_arr, when set, replace the scalar by one value per state; pos is SRP's sunPos or ThirdBody's pos, and pos_table,
// when set, replaces it by one row per output interval ([K][3]).
struct ForceModel {
    int32_t kind;
    uint32_t flags;
    double mu, coef, r_eq;
    double rho0, scale_height, max_altitude, f107;
    double c, area, mass;
    double pos[3];
    const double *c_arr, *area_arr, *mass_arr;
    const double *pos_table;
};
struct ModelList {
    uint32_t count;  // 1..kMaxModels
    ForceModel m[kMaxModels];
};

AZ_HD double per_state(const double *arr, double scalar, uint32_t i) { return arr ? arr[i] : scalar; }

// ImprovedDrag.getDensity (ForceModel.zig:283-320): the last of the five layers with altitude >= baseAlt (the first
// below 200 km), exponential decay from its base, scaled by f107 / 150
AZ_HD double improved_density(double altitude, double f107) {
    double base = 100.0, rho = 5.297e-7, H = 5.877;
    if (altitude >= 200.0) base = 200.0, rho = 2.789e-10, H = 37.105;
    if (altitude >= 400.0) base = 400.0, rho = 3.725e-12, H = 62.822;
    if (altitude >= 600.0) base = 600.0, rho = 2.418e-13, H = 79.864;
    if (altitude >= 1000.0) base = 1000.0, rho = 3.561e-15, H = 200.0;
    const double deltaH = altitude - base;
    double r = rho * exp(-deltaH / H);
    const double f107Scale = f107 / 150.0;
    r *= f107Scale;
    return r;
}

// One model's acceleration at state s of batch item i during output interval k, line for line as the reference's
// acceleration() of that kind; a guard that returns zeros there writes zeros here.
AZ_HD void model_accel(const ForceModel &m, const double s[6], uint32_t i, uint32_t k, double a[3]) {
    const double x = s[0], y = s[1], z = s[2];
    a[0] = a[1] = a[2] = 0.0;
    switch (m.kind) {
        case kModelTwoBody: {  // :49-55
            const double r = sqrt(x * x + y * y + z * z);
            const double factor = -m.mu / (r * r * r);
            a[0] = factor * x, a[1] = factor * y, a[2] = factor * z;
            break;
        }
        case kModelJ2: {  // :67-79
            const double r2 = x * x + y * y + z * z;
            const double r = sqrt(r2);
            const double factor = -1.5 * m.coef * m.mu * m.r_eq * m.r_eq / (r2 * r2 * r);
            const double z2R2 = (z * z) / r2;
            a[0] = factor * x * (5.0 * z2R2 - 1.0);
            a[1] = factor * y * (5.0 * z2R2 - 1.0);
            a[2] = factor * z * (5.0 * z2R2 - 3.0);
            break;
        }
        case kModelJ3: {  // :122-142; the x / y coefficient carries a 1/r its z term does not (kept)
            const double r2 = x * x + y * y + z * z;
            const double r = sqrt(r2);
            const double rEq3 = m.r_eq * m.r_eq * m.r_eq;
            const double factor = 2.5 * m.coef * m.mu * rEq3 / (r2 * r2 * r2 * r);
            const double z2R2 = (z * z) / r2;
            const double xyCoeff = 3.0 * z / r - 7.0 * z * z2R2 / r;
            const double zCoeff = 6.0 * z * z - 7.0 * z * z * z2R2 - 0.6 * r2;
            a[0] = factor * x * xyCoeff, a[1] = factor * y * xyCoeff, a[2] = factor * zCoeff;
            break;
        }
        case kModelJ4: {  // :154-175; divides by r^9 (kept)
            const double r2 = x * x + y * y + z * z;
            const double r = sqrt(r2);
            const double r4 = r2 * r2;
            const double z2 = z * z;
            const double z4 = z2 * z2;
            const double z2R2 = z2 / r2;
            const double z4R4 = z4 / r4;
            const double rEq4 = m.r_eq * m.r_eq * m.r_eq * m.r_eq;
            const double factor = 1.875 * m.coef * m.mu * rEq4 / (r4 * r4 * r);
            const double xyTerm = 3.0 - 42.0 * z2R2 + 63.0 * z4R4;
            const double zTerm = 15.0 - 70.0 * z2R2 + 63.0 * z4R4;
            a[0] = factor * x * xyTerm, a[1] = factor * y * xyTerm, a[2] = factor * z * zTerm;
            break;
        }
        case kModelDrag: {  // :95-110
            const double vx = s[3], vy = s[4], vz = s[5];
            const double r = sqrt(x * x + y * y + z * z);
            const double altitude = r - m.r_eq;
            if (altitude > m.max_altitude) break;
            const double v = sqrt(vx * vx + vy * vy + vz * vz);
            if (v < 1e-10) break;
            const double rho = m.rho0 * exp(-altitude / m.scale_height);
            const double factor = -0.5 * per_state(m.c_arr, m.c, i) * per_state(m.area_arr, m.area, i) * rho * v * 1e3 /
                                  per_state(m.mass_arr, m.mass, i);
            a[0] = factor * vx / v, a[1] = factor * vy / v, a[2] = factor * vz / v;
            break;
        }
        case kModelImprovedDrag: {  // :322-348; zero below 100 km (kept)
            const double vx = s[3], vy = s[4], vz = s[5];
            const double r = sqrt(x * x + y * y + z * z);
            const double altitude = r - m.r_eq;
            if (altitude > m.max_altitude || altitude < 100.0) break;
            const double vrelX = vx + kEarthOmega * y;
            const double vrelY = vy - kEarthOmega * x;
            const double vrelZ = vz;
            const double vrel = sqrt(vrelX * vrelX + vrelY * vrelY + vrelZ * vrelZ);
            if (vrel < 1e-10) break;
            const double rho = improved_density(altitude, m.f107);
            const double factor = -0.5 * per_state(m.c_arr, m.c, i) * per_state(m.area_arr, m.area, i) * rho * vrel *
                                  1e3 / per_state(m.mass_arr, m.mass, i);
            a[0] = factor * vrelX / vrel, a[1] = factor * vrelY / vrel, a[2] = factor * vrelZ / vrel;
            break;
        }
        case kModelSrp: {  // :197-227
            double sx, sy, sz;
            if (m.pos_table) {
                const double *q = m.pos_table + (size_t)k * 3;
                sx = q[0], sy = q[1], sz = q[2];
            } else {
                sx = m.pos[0], sy = m.pos[1], sz = m.pos[2];
            }
            const double dx = sx - x, dy = sy - y, dz = sz - z;
            const double dist = sqrt(dx * dx + dy * dy + dz * dz);
            if (dist < 1e-10) break;
            const double sunDirX = dx / dist, sunDirY = dy / dist, sunDirZ = dz / dist;
            const double sunDist = sqrt(sx * sx + sy * sy + sz * sz);
            if (sunDist < 1e-10) break;
            const double hx = sx / sunDist, hy = sy / sunDist, hz = sz / sunDist;
            const double proj = x * hx + y * hy + z * hz;
            if (proj < 0) {
                const double perpX = x - proj * hx, perpY = y - proj * hy, perpZ = z - proj * hz;
                const double rho = sqrt(perpX * perpX + perpY * perpY + perpZ * perpZ);
                if (rho < m.r_eq) break;
            }
            const double scale = (kAuKm / dist) * (kAuKm / dist);
            const double factor = -per_state(m.c_arr, m.c, i) * kSrpPressure * scale * per_state(m.area_arr, m.area, i) /
                                  per_state(m.mass_arr, m.mass, i) * 1e-3;
            a[0] = factor * sunDirX, a[1] = factor * sunDirY, a[2] = factor * sunDirZ;
            break;
        }
        case kModelThirdBody: {  // :244-265
            double qx, qy, qz;
            if (m.pos_table) {
                const double *q = m.pos_table + (size_t)k * 3;
                qx = q[0], qy = q[1], qz = q[2];
            } else {
                qx = m.pos[0], qy = m.pos[1], qz = m.pos[2];
            }
            const double qMag = sqrt(qx * qx + qy * qy + qz * qz);
            if (qMag < 1e-10) break;
            const double qMag3 = qMag * qMag * qMag;
            const double dx = qx - x, dy = qy - y, dz = qz - z;
            const double dMag = sqrt(dx * dx + dy * dy + dz * dz);
            if (dMag < 1e-10) break;
            const double dMag3 = dMag * dMag * dMag;
            a[0] = m.mu * (dx / dMag3 - qx / qMag3);
            a[1] = m.mu * (dy / dMag3 - qy / qMag3);
            a[2] = m.mu * (dz / dMag3 - qz / qMag3);
            break;
        }
        default: break;
    }
}

// A caller's model list for batch item i: one model's acceleration as it is (the binding's rule,
// bindings/python/src/propagator.zig:138-146), several summed by Composite (ForceModel.zig:365-374) into a total that
// starts at zero, in list order.  L stays where the launch put it (a __grid_constant__ parameter on the device), and the
// list is walked by a loop that is not unrolled, so neither it nor a per-model array is copied into local memory.
struct ListForces {
    const ModelList &L;
    uint32_t i;      // batch item: its per-state coefficients
    uint32_t k = 0;  // output interval: its row of every position table
    AZ_HD void interval(uint32_t kk) { k = kk; }
    AZ_HD void operator()(const double s[6], double acc[3]) const {
        if (L.count == 1) {
            model_accel(L.m[0], s, i, k, acc);
            return;
        }
        acc[0] = acc[1] = acc[2] = 0.0;
#pragma unroll 1
        for (uint32_t j = 0; j < L.count; ++j) {
            double a[3];
            model_accel(L.m[j], s, i, k, a);
            acc[0] += a[0];
            acc[1] += a[1];
            acc[2] += a[2];
        }
    }
};

template <int kInt>
AZ_HD uint8_t propagate_state_models(const double y0[6], const ModelList &L, uint32_t i, const NumParams &p,
                                     const StepTable &steps, double *out, uint64_t counts[2]) {
    ListForces f{L, i};
    return propagate_with<kInt>(y0, f, p, steps, out, counts);
}

// ---- impulsive maneuvers: Spacecraft.propagate's loop (src/Spacecraft.zig:172-323) over a model list -----------------
// impulse kinds (ASTROZ_IMPULSE_*) and the status bytes of the maneuver calls beyond K7's (ASTROZ_MANEUVER_*)
constexpr int32_t kImpAbsolute = 0, kImpPrograde = 1, kImpPhase = 2, kImpPlaneChange = 3;
constexpr uint8_t kManAbnormal = 4, kManTruncated = 5;
// a trajectory has at most this many samples; one more stops the state (bounds a phasing coast of huge `orbits`)
constexpr uint64_t kManMaxSamples = 0xfffffffeull;

// One impulse of a schedule, the layout of astroz_impulse_t.  p: ABSOLUTE dv[3] km/s; PROGRADE p[0] = dv km/s; PHASE
// p[0] = angle rad, p[1] = orbits; PLANE_CHANGE p[0] = delta inclination rad, p[1] = delta RAAN rad.
struct Impulse {
    double time;
    int32_t kind;
    uint32_t reserved;
    double p[3];
};

// std.math.pow(f64, x, 3) as Zig evaluates an integral exponent (repeated squaring of the significand): x * (x * x)
AZ_HD double zig_pow3(double x) { return x * (x * x); }
// std.math.pow(f64, x, 2.0 / 3.0) as Zig evaluates it: the fractional part above 0.5 becomes 2/3 - 1 through exp(log),
// the integral part 1 multiplies the significand back in
AZ_HD double zig_pow_two_thirds(double x) { return exp((2.0 / 3.0 - 1.0) * log(x)) * x; }

// calculatePhaseChange (Spacecraft.zig:310-323): the prograde dv of a phasing orbit from radius r
AZ_HD double phase_dv(double radius, double phaseAngle, double transferOrbits, double mu) {
    const double vCircular = sqrt(mu / radius);
    const double period = 2.0 * kPi * sqrt(zig_pow3(radius) / mu);
    const double deltaT = phaseAngle * period / (2.0 * kPi * transferOrbits);
    const double transferPeriod = period + deltaT;
    const double aTransfer = zig_pow_two_thirds(transferPeriod * sqrt(mu) / (2.0 * kPi));
    const double vTransfer = sqrt(mu * (2.0 / radius - 1.0 / aTransfer));
    return vTransfer - vCircular;
}

// progradeVec (Spacecraft.zig:260-263)
AZ_HD void prograde_vec(const double y[6], double dvMag, double dv[3]) {
    const double vMag = sqrt(y[3] * y[3] + y[4] * y[4] + y[5] * y[5]);
    dv[0] = y[3] / vMag * dvMag, dv[1] = y[4] / vMag * dvMag, dv[2] = y[5] / vMag * dvMag;
}

// calculations.impulse (calculations.zig:480-485)
AZ_HD void apply_dv(double y[6], double dx, double dy, double dz) {
    y[3] = y[3] + dx, y[4] = y[4] + dy, y[5] = y[5] + dz;
}

// applyPlaneChange (Spacecraft.zig:272-307), its "simplified" direction kept: dv = (hx sin di, hy sin di, hz cos di) *
// dvMag / |h|, which is the reference's result and not the textbook plane change
AZ_HD void plane_change(double y[6], double deltaInclination, double deltaRaan) {
    const double vMag = sqrt(y[3] * y[3] + y[4] * y[4] + y[5] * y[5]);
    const double totalAngle = sqrt(deltaInclination * deltaInclination + deltaRaan * deltaRaan);
    if (totalAngle < 1e-10) return;
    const double dvMag = 2.0 * vMag * sin(totalAngle / 2.0);
    const double hx = y[1] * y[5] - y[2] * y[4];
    const double hy = y[2] * y[3] - y[0] * y[5];
    const double hz = y[0] * y[4] - y[1] * y[3];
    const double hMag = sqrt(hx * hx + hy * hy + hz * hz);
    const double si = sin(deltaInclination), ci = cos(deltaInclination);
    apply_dv(y, hx / hMag * dvMag * si, hy / hMag * dvMag * si, hz / hMag * dvMag * ci);
}

// One state's row of a maneuver call: sample j's time at times[j] and state at out[6 j] while j < cap; count counts
// every sample, written or not.
struct ManeuverRow {
    double *times, *out;
    uint64_t cap, count;
    // false when the sample would pass kManMaxSamples
    AZ_HD bool append(double t, const double y[6]) {
        if (count == kManMaxSamples) return false;
        if (count < cap) {
            times[count] = t;
#pragma unroll
            for (int c = 0; c < 6; ++c) out[count * 6 + c] = y[c];
        }
        ++count;
        return true;
    }
};

// Spacecraft.propagate (Spacecraft.zig:172-270) for one state, line for line, with the force f, the integrator kInt and
// the impulses imp[m] in list order:
//   append (t0, y0); while t < tf { fire every impulse with time <= t + h (a partial step to it when it lies ahead, the
//   burn, a sample); a regular step of min(h, tf - t); a sample; stop when the orbit is abnormal }.
// A DP87 step carries hCur through every call (partial steps, phasing coasts, regular steps).  Writes row.count
// samples (the first row.cap of them) and zero-fills the rest of the row.  Status: kManTruncated when count > cap, else
// kNumStopped (a DP87 rejection at hMin, or a sample past kManMaxSamples), kNumSubstepLimit, kNumNonFinite,
// kManAbnormal (the reference's abnormal-orbit stop), kNumOk.
template <int kInt, class F>
AZ_HD uint8_t maneuver_with(const double y0[6], F &f, const NumParams &p, double t0, double tf, double h,
                            const Impulse *imp, uint32_t m, ManeuverRow &row, uint64_t counts[2]) {
    double y[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) y[c] = y0[c];
    counts[0] = counts[1] = 0;
    row.count = 0;
    uint8_t status = kNumOk;
    bool stopped = false, abnormal = false;
    double hCur = kDpHStart;
    double t = t0;
    // Integrator.step of length dt from y; false when the state stops
    auto step = [&](double dt) -> bool {
        if (kInt == kIntRk4) {
            rk4_step(y, dt, f);
            ++counts[0];
            if (status == kNumOk && !all_finite(y)) status = kNumNonFinite;
            return true;
        }
        const uint8_t st = dp87_interval(y, hCur, dt, f, p, counts);
        if (st == kNumSubstepLimit) status = kNumSubstepLimit;
        return st != kNumStopped;
    };
    row.append(t, y);
    uint32_t idx = 0;
    while (t < tf && !stopped) {
        while (idx < m && imp[idx].time <= t + h) {
            const Impulse &b = imp[idx];
            const double dt = b.time - t;
            if (dt > 0) {
                if (!step(dt)) { stopped = true; break; }
                t += dt;
                if (!row.append(t, y)) { stopped = true; break; }
            }
            if (b.kind == kImpAbsolute) {
                apply_dv(y, b.p[0], b.p[1], b.p[2]);
            } else if (b.kind == kImpPrograde) {
                double dv[3];
                prograde_vec(y, b.p[0], dv);
                apply_dv(y, dv[0], dv[1], dv[2]);
            } else if (b.kind == kImpPhase) {  // applyImpulse's .phase (Spacecraft.zig:237-252)
                const double r = sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
                double dv[3];
                prograde_vec(y, phase_dv(r, b.p[0], b.p[1], p.mu), dv);
                apply_dv(y, dv[0], dv[1], dv[2]);
                const double period = 2.0 * kPi * sqrt(zig_pow3(r) / p.mu);
                const double tEnd = t + period * b.p[1];
                for (; t < tEnd && !stopped; t += h)
                    stopped = !step(h) || !row.append(t + h, y);
                if (stopped) break;
                apply_dv(y, -dv[0], -dv[1], -dv[2]);
            } else {
                plane_change(y, b.p[0], b.p[1]);
            }
            if (!row.append(t, y)) { stopped = true; break; }
            ++idx;
        }
        if (stopped) break;
        const double s = fmin(h, tf - t);
        if (!step(s)) { stopped = true; break; }
        t += s;
        if (!row.append(t, y)) { stopped = true; break; }
        // the abnormal-orbit test (Spacecraft.zig:263-269, calculateEnergy :265-269)
        const double r = sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
        const double v = sqrt(y[3] * y[3] + y[4] * y[4] + y[5] * y[5]);
        const double energy = 0.5 * v * v - p.mu / r;
        if (energy > 0 || isnan(energy) || r > 100000) {
            abnormal = true;
            break;
        }
    }
    for (uint64_t j = row.count; j < row.cap; ++j) {
        row.times[j] = 0.0;
#pragma unroll
        for (int c = 0; c < 6; ++c) row.out[j * 6 + c] = 0.0;
    }
    if (row.count > row.cap) return kManTruncated;
    if (stopped) return kNumStopped;
    if (status != kNumOk) return status;
    return abnormal ? kManAbnormal : kNumOk;
}

template <int kInt>
AZ_HD uint8_t maneuver_state_models(const double y0[6], const ModelList &L, uint32_t i, const NumParams &p, double t0,
                                    double tf, double h, const Impulse *imp, uint32_t m, ManeuverRow &row,
                                    uint64_t counts[2]) {
    ListForces f{L, i};
    return maneuver_with<kInt>(y0, f, p, t0, tf, h, imp, m, row, counts);
}

}  // namespace az

#ifndef AZ_NUMERICAL_CORES_ONLY
namespace az {
struct NumArgs {
    const double *states;            // [n][6]
    const double *cd, *area, *mass;  // [n] each (drag force sets only)
    StepTable steps;                 // the sampling loop's step sizes
    uint32_t n;
    NumParams p;
    double *out;        // [n][K + 1][6]
    uint8_t *status;    // [n]
    uint64_t *counts;   // [n][2] or nullptr
};
// Queue K7 for `integrator` / `forces` on s.
cudaError_t launch_numerical(const NumArgs &a, int integrator, int forces, cudaStream_t s);
// K7 with a model list: a.cd / a.area / a.mass are unused (per-state coefficients come with the models); the list's
// pointers are device pointers.  The list travels in the launch's parameters.
struct ModelArgs {
    NumArgs a;
    ModelList models;
};
cudaError_t launch_numerical_models(const ModelArgs &a, int integrator, cudaStream_t s);
// K7 maneuvers: a model list (no position tables) and per-state impulse schedules.  State i (of this launch; `first` +
// i of the call) fires impulses[offsets[first + i] .. offsets[first + i + 1]).
struct ManeuverArgs {
    const double *states;      // [n][6]
    uint32_t n, first;
    double t0, tf, h;
    NumParams p;               // mu: the central body's; rtol / atol: DP87's
    const uint32_t *offsets;   // [call's n + 1]
    const Impulse *impulses;   // [m]
    uint32_t maxSamples;
    double *times;             // [n][maxSamples]
    double *out;               // [n][maxSamples][6]
    uint64_t *count;           // [n]
    uint8_t *status;           // [n]
    uint64_t *counts;          // [n][2] or nullptr
    ModelList models;
};
cudaError_t launch_maneuvers(const ManeuverArgs &a, int integrator, cudaStream_t s);
}  // namespace az
#endif
