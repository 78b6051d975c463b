// az_correlate.cuh -- K12: sensor tracks correlated with catalogue rows by the Mahalanobis distance of the track's
// stacked residuals under the row's covariance.  __host__ __device__, so the kernels (az_correlate.cu) and the host
// emulation (tests/host_emul/emul_correlate.cu) run this source.
//
// The catalogue is K10's: element columns, a 7 x 7 covariance P in the element fit's variables (28 words, NULL: every P
// zero) and the model byte (NULL: all 0).  Track j is the observations [offsets[j], offsets[j + 1]) in K8's observation
// layout (az_obs.cuh).  For one pair (track j, row s), x the variables of row s:
//   sets      fit_build_set_of under the row's model, as K10 builds them (forward step, the backward step when the forward
//             set cannot be built, inv = 1 / the step taken); B* held when P's B* row is zero; when P is all zero no
//             stepped set is built or propagated (nvar = 0);
//   rows      per observation, z (6) and G (6 x nvar) = obs_residual_rows: the weighted residual and weighted Jacobian
//             rows of the element fit (fit_accumulate_obs), at K10's tsince and jdFull = add_rn(jd, fr);
//   sums      |z|^2, b = G^T z and N = G^T G, accumulated over the track's observations in track order, each
//             observation's share formed by fit_accumulate_normal;
//   distance  d^2 = z^T (I + G P G^T)^-1 z over the stacked rows, evaluated by the push-through identity as
//             |z|^2 - b^T (I + P N)^-1 P b in its symmetric form: P = L L^T (a semi-definite Cholesky: a column whose
//             pivot is not positive is zero), u = L^T b, d^2 = |z|^2 - u^T (I + L^T N L)^-1 u, the 7 x 7 solve by
//             Cholesky (I + L^T N L has every eigenvalue >= 1).  Clamped at 0.  P = 0 gives |z|^2 exactly;
//   failure   a cell that fails (deep space: decay, eccentricity) or sums / d^2 that are not finite: the pair is skipped
//             and counted;
//   gate      the chi-square quantile of k degrees of freedom at the gate probability, k the track's used scalar
//             residuals (corr_chi2_quantile).
// Per track: the `best` smallest (d^2, row) over the evaluated pairs, ordered by d^2 and then row index (corr_insert),
// the rows with d^2 <= gate counted over every row, the failed pairs counted.  A track's bytes depend on its own
// observations and the catalogue alone.
#pragma once

#include "az_covariance.cuh"
#include "az_obs.cuh"

namespace az {

// per-track status bytes (ASTROZ_CORR_*)
enum CorrStatus : uint8_t { kCorrOk = 0, kCorrUncorrelated = 1, kCorrNoRow = 2, kCorrBadTrack = 3 };
constexpr int kCorrMaxBest = 8;                    // slots of the ordered list
constexpr uint32_t kCorrMaxTrack = 256;            // observations per track
constexpr uint32_t kCorrEmptyRow = 0xFFFFFFFFu;    // an empty slot's row

// The stepped sets of P: 0 when P is all zero, else cov_nvar (6 with the B* row zero, 7)
AZ_HD int corr_nvar(const double *P) {
    for (int q = 0; q < kFitN; ++q)
        if (P[q] != 0.0) return cov_nvar(P);
    return 0;
}

// The observation arrays of a batch of tracks (K8's layout)
struct CorrObsArrays {
    const double *jd, *fr;
    const uint8_t *kind;
    const double *value, *sigma;   // [m][6]
    const uint32_t *station;       // [m], read by the radar and optical kinds
    const double *stations;        // [k][3]
};

// Observation i: time, kind, values, weights, GMST and station.  Returns its used components.
struct CorrObs {
    int kind;
    double jdFull;
    double value[6], w[6];
    double sg, cg;
    ObsStation st;
};

AZ_HD int corr_obs(const CorrObsArrays &a, uint32_t i, CorrObs &o) {
    o.kind = a.kind[i];
    o.jdFull = add_rn(a.jd[i], a.fr[i]);
    double sigma[6], llh[3] = {0.0, 0.0, 0.0};
    for (int c = 0; c < 6; ++c) {
        o.value[c] = a.value[(size_t)i * 6 + c];
        sigma[c] = a.sigma[(size_t)i * 6 + c];
    }
    const int used = obs_weights(o.kind, o.value, sigma, o.w);
    if (obs_uses_station(o.kind)) {
        const uint32_t k = a.station[i];
        for (int c = 0; c < 3; ++c) llh[c] = a.stations[(size_t)k * 3 + c];
    }
    obs_frame(o.kind, o.jdFull, llh, o.sg, o.cg, o.st);
    return used;
}

// The used scalar residuals of a track (k), from the weights alone
AZ_HD uint32_t corr_used(const CorrObsArrays &a, uint32_t begin, uint32_t end) {
    uint32_t used = 0;
    for (uint32_t i = begin; i < end; ++i) {
        double value[6], sigma[6], w[6];
        for (int c = 0; c < 6; ++c) {
            value[c] = a.value[(size_t)i * 6 + c];
            sigma[c] = a.sigma[(size_t)i * 6 + c];
        }
        used += (uint32_t)obs_weights(a.kind[i], value, sigma, w);
    }
    return used;
}

// A track the device call refuses to score: empty, longer than kCorrMaxTrack, or with no used residual
AZ_HD bool corr_bad_track(uint32_t begin, uint32_t end, uint32_t used) {
    return end <= begin || end - begin > kCorrMaxTrack || used == 0;
}

// The pair sums of one (track, row): acc[0] = |z|^2, acc[4 + fit_tri(j, k)] = N, acc[4 + kFitN + j] = b (FitSums'
// word layout; words 1 .. 3 stay zero).  eval is the row's set evaluator (fit_accumulate_model's), J scratch for one
// observation's rows at stride 1.  False when a cell failed or a sum is not finite.
template <typename EvalFn>
AZ_HD bool corr_pair_sums(EvalFn eval, int nvar, const double *inv, double epochJd, const CorrObsArrays &a,
                          uint32_t begin, uint32_t end, double *J, double (&acc)[kFitSumWords]) {
#pragma unroll
    for (int q = 0; q < kFitSumWords; ++q) acc[q] = 0.0;
    for (uint32_t i = begin; i < end; ++i) {
        CorrObs o;
        corr_obs(a, i, o);
        double obs[6], sc[6], r[6];
        if (!obs_residual_rows(eval, nvar, inv, o.jdFull, epochJd, o.kind, o.value, o.w, o.sg, o.cg, o.st, obs, sc, r,
                               J, 1))
            return false;
#pragma unroll
        for (int c = 0; c < 6; ++c) acc[0] += r[c] * r[c];
        if (nvar > 0) fit_accumulate_normal(nvar, r, J, acc, 1);
    }
    bool finite = true;
#pragma unroll
    for (int q = 0; q < kFitSumWords; ++q) finite = finite && std::fabs(acc[q]) < INFINITY;
    return finite;
}

// d^2 = |z|^2 - u^T (I + L^T N L)^-1 u, u = L^T b, P = L L^T (file comment).  Not clamped; NaN when the solve fails.
AZ_HD double corr_d2(const double (&acc)[kFitSumWords], const double *P, int nvar) {
    const double zz = acc[0];
    if (nvar == 0) return zz;
    auto Pw = [P](int j, int k) { return j <= k ? P[fit_tri(j, k)] : P[fit_tri(k, j)]; };
    auto Nw = [&acc](int j, int k) { return j <= k ? acc[4 + fit_tri(j, k)] : acc[4 + fit_tri(k, j)]; };
    double L[kFitVars][kFitVars];
#pragma unroll
    for (int j = 0; j < kFitVars; ++j) {
#pragma unroll
        for (int i = 0; i < kFitVars; ++i) L[i][j] = 0.0;
        double d = Pw(j, j);
#pragma unroll
        for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
        if (d > 0.0) {
            const double ljj = std::sqrt(d);
            L[j][j] = ljj;
#pragma unroll
            for (int i = j + 1; i < kFitVars; ++i) {
                double s = Pw(j, i);
#pragma unroll
                for (int q = 0; q < j; ++q) s -= L[i][q] * L[j][q];
                L[i][j] = s / ljj;
            }
        }
    }
    double u[kFitVars], M[kFitVars][kFitVars];
#pragma unroll
    for (int k = 0; k < kFitVars; ++k) {
        double nl[kFitVars];   // column k of N L
#pragma unroll
        for (int q = 0; q < kFitVars; ++q) {
            double s = 0.0;
#pragma unroll
            for (int p = k; p < kFitVars; ++p) s += Nw(q, p) * L[p][k];
            nl[q] = s;
        }
#pragma unroll
        for (int j = 0; j <= k; ++j) {
            double s = 0.0;
#pragma unroll
            for (int q = j; q < kFitVars; ++q) s += L[q][j] * nl[q];
            M[j][k] = (j == k ? 1.0 : 0.0) + s;
        }
        double s = 0.0;
#pragma unroll
        for (int q = k; q < kFitVars; ++q) s += L[q][k] * acc[4 + kFitN + q];
        u[k] = s;
    }
    // M = C C^T (upper words M[j][k], j <= k), v = C^-1 u
    double C[kFitVars][kFitVars], v[kFitVars], vv = 0.0;
#pragma unroll
    for (int j = 0; j < kFitVars; ++j) {
        double d = M[j][j];
#pragma unroll
        for (int q = 0; q < j; ++q) d -= C[j][q] * C[j][q];
        if (!(d > 0.0)) return NAN;
        const double cjj = std::sqrt(d);
#pragma unroll
        for (int i = j + 1; i < kFitVars; ++i) {
            double s = M[j][i];
#pragma unroll
            for (int q = 0; q < j; ++q) s -= C[i][q] * C[j][q];
            C[i][j] = s / cjj;
        }
        double s = u[j];
#pragma unroll
        for (int q = 0; q < j; ++q) s -= C[j][q] * v[q];
        v[j] = s / cjj;
        vv += v[j] * v[j];
    }
    return zz - vv;
}

// ---- the gate: the chi-square quantile --------------------------------------------------------------------------------
// The regularised incomplete gamma functions P(a, y) and Q(a, y) = 1 - P: the series for y < a + 1, the continued
// fraction (modified Lentz) otherwise, each with the prefactor y^a e^-y / Gamma(a).
AZ_HD void corr_gamma_pq(double a, double y, double &P, double &Q) {
    if (!(y > 0.0)) {
        P = 0.0;
        Q = 1.0;
        return;
    }
    const double pre = std::exp(a * std::log(y) - y - std::lgamma(a));
    if (y < a + 1.0) {
        double ap = a, del = 1.0 / a, sum = del;
        for (int n = 0; n < 4000; ++n) {
            ap += 1.0;
            del *= y / ap;
            sum += del;
            if (del < sum * 1e-17) break;
        }
        P = sum * pre;
        Q = 1.0 - P;
        return;
    }
    constexpr double tiny = 1e-300;
    double b = y + 1.0 - a, c = 1.0 / tiny, d = 1.0 / b, h = d;
    for (int i = 1; i < 4000; ++i) {
        const double an = -i * (i - a);
        b += 2.0;
        d = an * d + b;
        if (std::fabs(d) < tiny) d = tiny;
        c = b + an / c;
        if (std::fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (std::fabs(del - 1.0) < 4e-16) break;
    }
    Q = pre * h;
    P = 1.0 - Q;
}

// The quantile x of the chi-square distribution of k >= 1 degrees of freedom at probability p in (0, 1): P(k/2, x/2)
// = p.  Newton's method on the log of the smaller tail (P for p <= 1/2, Q = 1 - p otherwise) in y = x / 2, from the
// Wilson-Hilferty approximation, kept inside the bracket it has established (a step that leaves it bisects).
AZ_HD double corr_chi2_quantile(uint32_t k, double p) {
    const double a = 0.5 * k;
    const bool upper = p > 0.5;
    const double t = upper ? 1.0 - p : p, lt = std::log(t);
    // normal quantile of p (Abramowitz & Stegun 26.2.23, |error| < 4.5e-4): the starting point only
    const double s = std::sqrt(-2.0 * lt);
    double z = s - (2.515517 + 0.802853 * s + 0.010328 * s * s) / (1.0 + 1.432788 * s + 0.189269 * s * s +
                                                                  0.001308 * s * s * s);
    if (!upper) z = -z;
    const double h = 2.0 / (9.0 * k), wh = 1.0 - h + z * std::sqrt(h);
    double y = wh > 0.1 ? 0.5 * k * wh * wh * wh : 0.5 * k * 1e-3;
    double lo = 0.0, hi = INFINITY;
    for (int it = 0; it < 200; ++it) {
        double P, Q;
        corr_gamma_pq(a, y, P, Q);
        const double F = upper ? Q : P;
        if ((F < t) != upper) lo = y;   // the quantile lies above y
        else hi = y;
        const double dens = std::exp((a - 1.0) * std::log(y) - y - std::lgamma(a));   // dP/dy
        const double g = std::log(F) - lt, dg = (upper ? -dens : dens) / F;
        double yn = y - g / dg;
        if (!(yn > lo && yn < hi)) yn = hi < INFINITY ? 0.5 * (lo + hi) : 2.0 * y;
        const double dy = yn - y;
        y = yn;
        if (std::fabs(dy) <= 1e-15 * y) break;
    }
    return 2.0 * y;
}

// ---- the ordered list --------------------------------------------------------------------------------------------------
AZ_HD bool corr_less(double d, uint32_t r, double bd, uint32_t br) { return d < bd || (d == bd && r < br); }

AZ_HD void corr_empty(double (&bd)[kCorrMaxBest], uint32_t (&br)[kCorrMaxBest]) {
#pragma unroll
    for (int q = 0; q < kCorrMaxBest; ++q) {
        bd[q] = INFINITY;
        br[q] = kCorrEmptyRow;
    }
}

// (d, r) into the list, kept ordered by (d^2, row); the last entry falls off
AZ_HD void corr_insert(double (&bd)[kCorrMaxBest], uint32_t (&br)[kCorrMaxBest], double d, uint32_t r) {
#pragma unroll
    for (int q = 0; q < kCorrMaxBest; ++q) {
        if (corr_less(d, r, bd[q], br[q])) {
            const double td = bd[q];
            const uint32_t tr = br[q];
            bd[q] = d;
            br[q] = r;
            d = td;
            r = tr;
        }
    }
}

// A track's status from its in-gate count and its best row (empty: no pair was evaluated)
AZ_HD uint8_t corr_status(uint32_t nGate, uint32_t bestRow) {
    return nGate > 0 ? kCorrOk : bestRow == kCorrEmptyRow ? kCorrNoRow : kCorrUncorrelated;
}

// ---- launch shape -----------------------------------------------------------------------------------------------------
// Tracks go in chunks of kCorrThreads (one thread each), rows in chunks of `rows` consecutive rows; a CTA scores one
// (track chunk, row chunk).  The row chunk is the smallest that still leaves about AZ_CORR_TARGET_CTAS CTAs per class,
// so one track against the catalogue spreads over the whole GPU and a dense batch keeps its set building amortised over
// 64 tracks.  No result depends on the shape.
constexpr int kCorrWarps = 2;
constexpr int kCorrThreads = kCorrWarps * 32;
#ifndef AZ_CORR_TARGET_CTAS
#define AZ_CORR_TARGET_CTAS 2048
#endif
struct CorrShape {
    uint32_t trackChunks, rowChunks, rows;
};

AZ_HD CorrShape corr_shape(uint32_t n, uint32_t t) {
    CorrShape s;
    s.trackChunks = (uint32_t)(((uint64_t)t + kCorrThreads - 1) / kCorrThreads);
    uint64_t want = s.trackChunks ? (AZ_CORR_TARGET_CTAS + s.trackChunks - 1) / s.trackChunks : 1;
    const uint64_t most = ((uint64_t)n + kCorrWarps - 1) / kCorrWarps;   // at least one stage of rows per chunk
    if (want > most) want = most;
    if (want > 65535) want = 65535;
    if (want < 1) want = 1;
    s.rows = (uint32_t)(((uint64_t)n + want - 1) / want);
    if (s.rows < 1) s.rows = 1;
    s.rowChunks = (uint32_t)(((uint64_t)n + s.rows - 1) / s.rows);
    if (s.rowChunks < 1) s.rowChunks = 1;
    return s;
}

// Scratch of the device call: gate[t] doubles, then per class (near-earth, deep space) and row chunk the partial lists
// d2[t][best] and rows[t][best] and the counts [t][2] (in gate, failed).
AZ_HD size_t corr_scratch_bytes(uint32_t n, uint32_t t, uint32_t best) {
    const CorrShape s = corr_shape(n, t);
    const size_t lists = (size_t)2 * s.rowChunks * t;
    return (size_t)8 * t + lists * best * 8 + lists * best * 4 + lists * 8;
}

}  // namespace az
