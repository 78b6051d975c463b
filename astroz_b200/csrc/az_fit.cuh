// az_fit.cuh -- K8: least-squares fit of SGP4 mean elements to TEME ephemerides, one satellite at a time.
// __host__ __device__, so the kernel (az_fit.cu) and the host emulation (tests/host_emul/emul_fit.cu) run this source.
//
// The model is the library's near-earth path: a trial element set goes through build_near_earth and sgp4_columns, the
// way every near-earth table is built, and is propagated by sgp4_cell<1> at tsince = ((jd + fr) - epoch) * 1440,
// formed uncontracted like K6 and Satrec.sgp4.  Seven variables, six when B* is held:
//   x = [n (rev/day), e cos w, e sin w, i (rad), node (rad), lambda = M + w (rad), B* (1/ER)]
// The pairs (e cos w, e sin w) and lambda stay well conditioned as e -> 0, where (w, M) alone do not.  Levenberg-
// Marquardt over the weighted residuals (pos / pos_sigma, vel / vel_sigma): forward-difference Jacobian with the steps
// of fit_step(), Marquardt damping lambda diag(J^T J), the normal equations solved by Cholesky on their unit-diagonal
// scaling, lambda / 10 after an accepted step and x 10 after a rejected one.
//
// Deep-space sets (period > 225 min) have a second model, FitDeepSpace, under the same driver: equinoctial variables
//   x = [n (rev/day), k = e cos pi, h = e sin pi, q = tan(i/2) cos node, p = tan(i/2) sin node, lambda = M + pi, B*],
// pi = w + node, which stay well conditioned as i -> 0 (GEO), where node and M + w alone do not (their Jacobian columns
// coincide).  They diverge as i -> 180 deg: retrograde deep-space sets near i = 180 deg are not fitted well.  A trial set
// goes through build_deep_space and sdp4_record and is propagated by pairs_sdp4_query, the K6 deep-space query; the class
// is held (a trial set whose period drops to 225 min or below cannot be built), and an observation whose cell status is
// not 0 makes the pass fail.
#pragma once

#include "az_pairs.cuh"
#include "az_tables.hpp"

namespace az {

// per-satellite status bytes (ASTROZ_FIT_*)
enum FitStatus : uint8_t { kFitConverged = 0, kFitIterLimit = 1, kFitInitFailed = 2, kFitDeepSpace = 3, kFitTooFew = 4 };

constexpr int kFitVars = 7;              // variables with B* free
constexpr int kFitSets = 1 + kFitVars;   // nominal set + one perturbed set per variable
constexpr int kFitN = kFitVars * (kFitVars + 1) / 2;  // J^T J upper triangle, row-major
constexpr double kFitTol = 1e-10;        // the fit stops when a step changes the cost by at most this fraction of it
constexpr double kFitNoise = 1e-12;      // ... or when every residual is at the rounding floor: kFitNoise x |state|
constexpr double kFitLambda0 = 1e-3;     // initial Marquardt damping

// Forward-difference step of variable j: 1e-8 rev/day, 1e-8 on e cos w / e sin w, 1e-8 rad on the angles, 1e-8 / ER
// on B*.  Each moves a LEO position by 1e-4 .. 1e-3 km over a day: some 1e8 times the propagation's rounding, and small
// enough that the truncation error of the difference (~ step / value) stays below 1e-8 of the column.  When the
// forward set is not a near-earth element set (the period would cross 225 min, the perigee 1 earth radius) the
// backward step is taken instead.
AZ_HD double fit_step(int) { return 1e-8; }

struct FitSums {             // one pass over a satellite's observations under the nominal set and its perturbations
    double F;                // weighted cost: sum of r^2, r = (observed - model) / sigma
    double pos2, vel2;       // unweighted sums of |dr|^2 [km^2] and |dv|^2 [km^2/s^2]
    double floor;            // kFitNoise^2 sum of (|r_obs| / pos_sigma)^2 + (|v_obs| / vel_sigma)^2: the rounding floor of F
    double N[kFitN];         // J^T J, J = d(model)/dx weighted
    double g[kFitVars];      // J^T r
};
constexpr int kFitSumWords = 4 + kFitN + kFitVars;

AZ_HD double *fit_words(FitSums &s) { return &s.F; }
static_assert(sizeof(FitSums) == kFitSumWords * sizeof(double), "FitSums is a flat array of doubles");

AZ_HD int fit_tri(int j, int k) { return j * kFitVars - j * (j - 1) / 2 + (k - j); }  // entry (j, k), j <= k

// Variables -> the eight element columns (epoch, n, e, i, node, w, M in degrees, B*): w = atan2(e sin w, e cos w) and
// M = lambda - w, node, w and M reduced to [0, 360).  The fit's output is this conversion of its final iterate.
AZ_HD void fit_elements_of(const double (&x)[kFitVars], double epochJd, TleRecord &t) {
    using detail::kDeg;
    const double r2d = 1.0 / kDeg;
    t = TleRecord{};
    t.epochJd = epochJd;
    t.revPerDay = x[0];
    t.ecc = std::sqrt(x[1] * x[1] + x[2] * x[2]);
    const double w = std::atan2(x[2], x[1]);
    t.argpDeg = detail::wrap(w * r2d, 360.0);
    t.inclDeg = x[3] * r2d;
    t.raanDeg = detail::wrap(x[4] * r2d, 360.0);
    t.maDeg = detail::wrap((x[5] - w) * r2d, 360.0);
    t.bstar = x[6];
}

// el[c] = column c of the element set (epoch JD, n rev/day, e, i, node, w, M deg, B*) -> variables
AZ_HD void fit_vars_of(const double *el, double (&x)[kFitVars]) {
    using detail::kDeg;
    const double w = el[5] * kDeg;
    x[0] = el[1];
    x[1] = el[2] * std::cos(w);
    x[2] = el[2] * std::sin(w);
    x[3] = el[3] * kDeg;
    x[4] = el[4] * kDeg;
    x[5] = el[6] * kDeg + w;
    x[6] = el[7];
}

AZ_HD int fit_columns(const TleRecord &t, const Gravity &grav, double *cols) {
    NearEarth ne;
    const int rc = build_near_earth(t, grav, ne);
    if (rc == kOk) sgp4_columns(ne, cols);
    return rc;
}

// The near-earth model: variables above, sets as near-earth columns (kSgp4Cols doubles).  The class of the initial set
// decides the status of a set that is not fitted.
struct FitNearEarth {
    using Set = double[kSgp4Cols];
    AZ_HD static void vars_of(const double *el, double (&x)[kFitVars]) { fit_vars_of(el, x); }
    AZ_HD static void elements_of(const double (&x)[kFitVars], double epochJd, TleRecord &t) {
        fit_elements_of(x, epochJd, t);
    }
    AZ_HD static bool build(const TleRecord &t, const Gravity &grav, double *cols) {
        return fit_columns(t, grav, cols) == kOk;
    }
    // from build_near_earth's code for the initial set: is it fitted, and if not, its status
    AZ_HD static bool fits(int rc) { return rc == kOk; }
    AZ_HD static uint8_t not_fitted(int rc) { return rc == kDeepSpace ? kFitDeepSpace : kFitInitFailed; }
};

// The deep-space model: equinoctial variables (file comment), sets as Sdp4Sat records.
struct FitDeepSpace {
    using Set = Sdp4Sat;
    // el[c] = the eight element columns -> x
    AZ_HD static void vars_of(const double *el, double (&x)[kFitVars]) {
        using detail::kDeg;
        const double node = el[4] * kDeg, peri = el[5] * kDeg + node, ti = std::tan(0.5 * el[3] * kDeg);
        x[0] = el[1];
        x[1] = el[2] * std::cos(peri);
        x[2] = el[2] * std::sin(peri);
        x[3] = ti * std::cos(node);
        x[4] = ti * std::sin(node);
        x[5] = el[6] * kDeg + peri;
        x[6] = el[7];
    }
    // x -> element set: e = |(k, h)|, pi = atan2(h, k), i = 2 atan |(p, q)|, node = atan2(p, q), w = pi - node,
    // M = lambda - pi; node, w and M reduced to [0, 360)
    AZ_HD static void elements_of(const double (&x)[kFitVars], double epochJd, TleRecord &t) {
        using detail::kDeg;
        const double r2d = 1.0 / kDeg;
        t = TleRecord{};
        t.epochJd = epochJd;
        t.revPerDay = x[0];
        t.ecc = std::sqrt(x[1] * x[1] + x[2] * x[2]);
        const double peri = std::atan2(x[2], x[1]);
        const double node = std::atan2(x[4], x[3]);
        t.inclDeg = 2.0 * std::atan(std::sqrt(x[3] * x[3] + x[4] * x[4])) * r2d;
        t.raanDeg = detail::wrap(node * r2d, 360.0);
        t.argpDeg = detail::wrap((peri - node) * r2d, 360.0);
        t.maDeg = detail::wrap((x[5] - peri) * r2d, 360.0);
        t.bstar = x[6];
    }
    // the class is held: a set that fails init or whose period is 225 min or less cannot be built
    AZ_HD static bool build(const TleRecord &t, const Gravity &grav, Sdp4Sat &rec) {
        DeepSpace ds;
        if (build_deep_space(t, grav, ds) != kOk || !(detail::kHTwoPi / ds.ne.no > 225.0)) return false;
        rec = sdp4_record(ds);
        return true;
    }
    AZ_HD static bool fits(int rc) { return rc == kDeepSpace; }
    AZ_HD static uint8_t not_fitted(int) { return kFitInitFailed; }   // callers route near-earth sets to FitNearEarth
};

// Set k of an iteration into set: k = 0 the nominal set x, k = 1 + j the set with variable j stepped (forward, or
// backward when the forward set cannot be built).  inv[0] = 0, inv[k] = 1 / (the step actually taken, x'[j] - x[j] in
// fp64).  Returns false when the set cannot be built.
template <typename Model, typename SetT>
AZ_HD bool fit_build_set_of(const double (&x)[kFitVars], int k, double epochJd, const Gravity &grav, SetT &set,
                            double &inv) {
    TleRecord t;
    inv = 0.0;
    if (k == 0) {
        Model::elements_of(x, epochJd, t);
        return Model::build(t, grav, set);
    }
    const int j = k - 1;
    double xs[kFitVars];
    for (int q = 0; q < kFitVars; ++q) xs[q] = x[q];
    for (int dir = 0; dir < 2; ++dir) {
        xs[j] = dir == 0 ? x[j] + fit_step(j) : x[j] - fit_step(j);
        Model::elements_of(xs, epochJd, t);
        if (Model::build(t, grav, set)) {
            inv = 1.0 / (xs[j] - x[j]);
            return true;
        }
    }
    return false;
}

// the near-earth sets into cols[kSgp4Cols]
AZ_HD bool fit_build_set(const double (&x)[kFitVars], int k, double epochJd, const Gravity &grav, double *cols,
                         double &inv) {
    return fit_build_set_of<FitNearEarth>(x, k, epochJd, grav, cols, inv);
}

// One observation's share of J^T r and J^T J: r[6] its weighted residuals, J its 6 x nvar Jacobian, entry (j, c) at
// J[(j * 6 + c) * stride]; word q of the FitSums being accumulated is acc[q * stride].
AZ_HD void fit_accumulate_normal(int nvar, const double (&r)[6], const double *J, double *acc, int stride) {
    // all kFitVars columns, the held B* column as zeros, so the sums keep static indices (registers on the device)
#pragma unroll
    for (int j = 0; j < kFitVars; ++j) {
        double jc[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) jc[c] = j < nvar ? J[(j * 6 + c) * stride] : 0.0;
        double gj = 0.0;
#pragma unroll
        for (int c = 0; c < 6; ++c) gj += jc[c] * r[c];
        acc[(4 + kFitN + j) * stride] += gj;
#pragma unroll
        for (int k = j; k < kFitVars; ++k) {
            double njk = 0.0;
#pragma unroll
            for (int c = 0; c < 6; ++c) njk += jc[c] * (k < nvar ? J[(k * 6 + c) * stride] : 0.0);
            acc[(4 + fit_tri(j, k)) * stride] += njk;
        }
    }
}

// One observation's contribution to s: the model under set 0 and under sets 1..nvar (eval(k, jdFull, ts, f) = the TEME
// state f[6] of set k at the observation, false when that set's cell fails), the weighted residual and the difference
// columns of the Jacobian.  J is scratch for the 6 x nvar Jacobian of this observation, entry (j, c) at
// J[(j * 6 + c) * stride]; word q of the FitSums being accumulated is acc[q * stride].  vel = nullptr: positions only.
// Returns false when a cell failed (the sums are then meaningless).
template <typename EvalFn>
AZ_HD bool fit_accumulate_model(EvalFn eval, int nvar, const double *inv, double jdFull, double epochJd,
                                const double *pos, const double *vel, double wp, double wv, double *J, double *acc,
                                int stride) {
    const double ts[1] = {mul_rn(sub_rn(jdFull, epochJd), 1440.0)};
    bool ok = true;
    const int nc = vel ? 6 : 3;
    double obs[6], w[6], f0[6];
    for (int c = 0; c < 3; ++c) {
        obs[c] = pos[c];
        w[c] = wp;
        obs[3 + c] = vel ? vel[c] : 0.0;
        w[3 + c] = wv;
    }
    ok = eval(0, jdFull, ts, f0) && ok;
    double r[6];
    for (int c = 0; c < 6; ++c) r[c] = c < nc ? (obs[c] - f0[c]) * w[c] : 0.0;
    {
        double F = acc[0], pos2 = acc[stride], vel2 = acc[2 * stride], fl = acc[3 * stride];
        for (int c = 0; c < 3; ++c) {
            const double dp = obs[c] - f0[c], dv = obs[3 + c] - f0[3 + c];
            pos2 += dp * dp;
            if (vel) vel2 += dv * dv;
            F += r[c] * r[c];
            if (vel) F += r[3 + c] * r[3 + c];
            const double fp = obs[c] * wp * kFitNoise, fv = obs[3 + c] * wv * kFitNoise;
            fl += fp * fp;
            if (vel) fl += fv * fv;
        }
        acc[0] = F;
        acc[stride] = pos2;
        acc[2 * stride] = vel2;
        acc[3 * stride] = fl;
    }
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < nvar; ++j) {
        double f[6];
        ok = eval(1 + j, jdFull, ts, f) && ok;
        for (int c = 0; c < 6; ++c) J[(j * 6 + c) * stride] = c < nc ? (f[c] - f0[c]) * w[c] * inv[1 + j] : 0.0;
    }
    fit_accumulate_normal(nvar, r, J, acc, stride);
    return ok;
}

// The near-earth model's observation: set(k) = column accessor of near-earth set k, propagated by sgp4_cell<1>.
template <typename SetFn>
AZ_HD void fit_accumulate(SetFn set, int nvar, const double *inv, double jdFull, double epochJd, const double *pos,
                          const double *vel, double wp, double wv, const GravConsts &g, double *J, double *acc,
                          int stride) {
    auto eval = [&](int k, double, const double (&ts)[1], double (&f)[6]) {
        CellOut o[1];
        sgp4_cell<1>(set(k), ts, g, o);
        f[0] = o[0].rx; f[1] = o[0].ry; f[2] = o[0].rz;
        f[3] = o[0].vx; f[4] = o[0].vy; f[5] = o[0].vz;
        return true;
    };
    fit_accumulate_model(eval, nvar, inv, jdFull, epochJd, pos, vel, wp, wv, J, acc, stride);
}

// ---- deep space: the K2a resonance lattice of one record, and its query --------------------------------------------
constexpr int kFitLatticeNodes = 16;   // nodes per direction: the lattice's extent (speed only; see fit_deep_eval)

// Nodes of one direction that cover |tsince| <= maxAbsTs: node k is the state after k 720-min steps from atime = 0.
AZ_HD int fit_lattice_nodes(double maxAbsTs) {
    const int need = resonance_node(maxAbsTs) + 1;
    return need < kFitLatticeNodes ? need : kFitLatticeNodes;
}

// Direction dir (0 forward, 1 backward) of e's lattice, nodes 0 .. nodes - 1 into out (a [2][kFitLatticeNodes] lattice
// of pairs_sdp4_query's layout).  Only node 0 for a non-resonant record (irez 0 never reads the lattice).
AZ_HD void fit_deep_lattice(const Sdp4Sat &e, int dir, int nodes, double2 *out) {
    const double delt = dir == 0 ? kStepp : -kStepp;
    double xli = e.xlamo, xni = e.no, atime = 0.0;
    out += dir * kFitLatticeNodes;
    out[0] = make_double2(xli, xni);
    if (e.irez == 0) return;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int k = 1; k < nodes; ++k) {
        resonance_step(e, xli, xni, atime, delt);
        out[k] = make_double2(xli, xni);
    }
}

// The deep-space model's observation: pairs_sdp4_query in TEME, the state at the lattice node below |tsince| stepped on
// to the query, so a time beyond the lattice is stepped from its last node and the result never depends on the
// lattice's extent.  False when the cell's status is not 0.
AZ_HD bool fit_deep_eval(const Sdp4Sat &e, const double2 *lattice, double jdFull, const GravConsts &g,
                         double (&f)[6]) {
    CellOut o;
    const uint8_t st = pairs_sdp4_query<0, true>(e, lattice, kFitLatticeNodes, jdFull, g, o);
    f[0] = o.rx; f[1] = o.ry; f[2] = o.rz;
    f[3] = o.vx; f[4] = o.vy; f[5] = o.vz;
    return st == 0;
}

// Solve (N + lambda diag N) d = g for the nvar variables, on the unit-diagonal scaling of N (a variable whose column
// is zero gets d = 0).  Returns false when the Cholesky factorisation meets a pivot that is not positive and finite.
AZ_HD bool fit_solve(const FitSums &s, int nvar, double lambda, double (&d)[kFitVars]) {
    double sc[kFitVars], L[kFitVars][kFitVars], y[kFitVars];
    for (int j = 0; j < kFitVars; ++j) {
        const double njj = j < nvar ? s.N[fit_tri(j, j)] : 0.0;
        sc[j] = njj > 0.0 ? 1.0 / std::sqrt(njj) : 0.0;
        d[j] = 0.0;
    }
    for (int j = 0; j < nvar; ++j) {
        for (int k = 0; k <= j; ++k) {
            double a = (k == j) ? (sc[j] > 0.0 ? 1.0 + lambda : 1.0) : s.N[fit_tri(k, j)] * sc[j] * sc[k];
            for (int q = 0; q < k; ++q) a -= L[j][q] * L[k][q];
            if (k == j) {
                if (!(a > 0.0) || !(a < INFINITY)) return false;
                L[j][j] = std::sqrt(a);
            } else {
                L[j][k] = a / L[k][k];
            }
        }
    }
    for (int j = 0; j < nvar; ++j) {
        double b = s.g[j] * sc[j];
        for (int q = 0; q < j; ++q) b -= L[j][q] * y[q];
        y[j] = b / L[j][j];
    }
    for (int j = nvar - 1; j >= 0; --j) {
        double b = y[j];
        for (int q = j + 1; q < nvar; ++q) b -= L[q][j] * d[q];
        d[j] = b / L[j][j];
    }
    for (int j = 0; j < nvar; ++j) d[j] *= sc[j];
    return true;
}

struct FitResult {
    double el[8];            // fitted columns (epoch, n, e, i, node, w, M, B*)
    double rmsPos, rmsVel;   // sqrt(mean |dr|^2) [km], sqrt(mean |dv|^2) [km/s] (0 without velocities)
    uint32_t iters;          // LM steps tried (accepted or rejected)
    uint8_t status;
};

// The whole fit of one satellite.  pass(x, s) evaluates the nominal set x and its nvar perturbed sets over the
// satellite's observations into s (zeroed by the caller) and returns false when a set cannot be built; it must
// return the same bits wherever it is called for the same x.  nResiduals is the number of scalar residuals the
// observations carry.  Failing satellites (init, deep space, too few residuals) return their initial columns with
// zero RMS and no iterations; for a fitted satellite final(s) receives the sums at its final iterate.
// Model (FitNearEarth, FitDeepSpace) gives the variables and the class rule of the initial set.
template <typename PassFn, typename FinalFn, typename Model>
AZ_HD void fit_satellite_run(const double *el0, const Gravity &grav, bool fitBstar, uint32_t maxIter,
                             uint64_t nResiduals, PassFn pass, FinalFn final, FitResult &out, Model) {
    const int nvar = fitBstar ? kFitVars : kFitVars - 1;
    for (int c = 0; c < 8; ++c) out.el[c] = el0[c];
    out.rmsPos = out.rmsVel = 0.0;
    out.iters = 0;
    {
        TleRecord t;
        t.epochJd = el0[0]; t.revPerDay = el0[1]; t.ecc = el0[2]; t.inclDeg = el0[3];
        t.raanDeg = el0[4]; t.argpDeg = el0[5]; t.maDeg = el0[6]; t.bstar = el0[7];
        NearEarth ne;
        const int rc = build_near_earth(t, grav, ne);
        if (!Model::fits(rc)) {
            out.status = Model::not_fitted(rc);
            return;
        }
    }
    if (nResiduals < (uint64_t)nvar) {
        out.status = kFitTooFew;
        return;
    }
    double x[kFitVars];
    Model::vars_of(el0, x);
    FitSums s = {};
    if (!pass(x, s)) {
        out.status = kFitInitFailed;
        return;
    }
    uint8_t status = kFitIterLimit;
    double lambda = kFitLambda0;
    uint32_t it = 0;
    if (s.F <= s.floor) status = kFitConverged;
    while (status != kFitConverged && it < maxIter) {
        ++it;
        double d[kFitVars], xt[kFitVars];
        FitSums t = {};
        bool ok = fit_solve(s, nvar, lambda, d);
        if (ok) {
            for (int j = 0; j < kFitVars; ++j) xt[j] = x[j] + d[j];
            ok = pass(xt, t);
        }
        if (!ok || !(t.F < s.F)) {   // rejected (also a non-finite cost)
            if (ok && t.F - s.F <= kFitTol * s.F) status = kFitConverged;
            lambda *= 10.0;
            continue;
        }
        const bool small = s.F - t.F <= kFitTol * s.F;
        for (int j = 0; j < kFitVars; ++j) x[j] = xt[j];
        s = t;
        lambda *= 0.1;
        if (small || s.F <= s.floor) status = kFitConverged;
    }
    TleRecord t;
    Model::elements_of(x, el0[0], t);
    out.el[0] = t.epochJd; out.el[1] = t.revPerDay; out.el[2] = t.ecc; out.el[3] = t.inclDeg;
    out.el[4] = t.raanDeg; out.el[5] = t.argpDeg; out.el[6] = t.maDeg; out.el[7] = t.bstar;
    final(s);
    out.iters = it;
    out.status = status;
}

// The fit of TEME ephemerides: nObs positions (and velocities with haveVel), RMS from the final iterate's sums.
template <typename PassFn, typename Model = FitNearEarth>
AZ_HD void fit_satellite(const double *el0, const Gravity &grav, bool fitBstar, uint32_t maxIter, uint32_t nObs,
                         bool haveVel, PassFn pass, FitResult &out, Model model = Model{}) {
    auto final = [&](const FitSums &s) {
        out.rmsPos = std::sqrt(s.pos2 / nObs);
        out.rmsVel = haveVel ? std::sqrt(s.vel2 / nObs) : 0.0;
    };
    fit_satellite_run(el0, grav, fitBstar, maxIter, (uint64_t)nObs * (haveVel ? 6 : 3), pass, final, out, model);
}

}  // namespace az
