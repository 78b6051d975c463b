// az_covariance.cuh -- K10: a fitted element set's covariance carried to a TEME or RTN state covariance at any time.
// __host__ __device__, so the kernels (az_covariance.cu) and the host emulation (tests/host_emul/emul_covariance.cu)
// run this source.
//
// Satellite s has element columns el (epoch, n, e, i, node, w, M deg, B*), a 7 x 7 covariance P in the variables of
// the element fit (az_fit.cuh: FitNearEarth's for model 0, FitDeepSpace's equinoctial set for model 1) and queries at
// times jd + fr.  For each query:
//   nominal   f(x) with x = Model::vars_of(el): sgp4_cell<1> on fit_columns (model 0) or fit_deep_eval (model 1), at
//             tsince = ((jd + fr) - epoch) * 1440 formed uncontracted -- the models the fit propagates;
//   Jacobian  J = df/dx (6 x 7), forward differences over the sets fit_build_set_of builds (fit_step, the backward step
//             when the forward set cannot be built, divided by the step actually taken): the fit's own J;
//   B* held   P's B* row all zero: the B* set is neither built nor propagated and J's B* column is zero;
//   frame     TEME, or RTN of the nominal state: R = r / |r|, N = r x v / |r x v|, T = N x R; the one rotation is
//             applied to the position and to the velocity block (no omega x r term of a rotating frame);
//   outputs   the 21-word upper triangle of Sigma = J P J^T row by row, J in the output frame (row-major 6 x 7), the
//             nominal TEME state;
//   status    kCovInitFailed when a set cannot be built under the row's model, kCovCellFailed when a deep-space cell
//             of the nominal or a stepped set fails (near-earth cells never fail: their decay is a diagnostic, as in
//             the grid and the fit).  A failed query is zero in every output.
// A query's bytes depend on its satellite's inputs and its own time alone.
#pragma once

#include "az_fit.cuh"

namespace az {

// per-query status bytes (ASTROZ_COV_*) and frames (ASTROZ_COV_FRAME_*)
enum CovStatus : uint8_t { kCovOk = 0, kCovInitFailed = 1, kCovCellFailed = 2 };
enum CovFrame : int { kCovFrameTeme = 0, kCovFrameRtn = 1 };

constexpr int kCovWords = 21;                 // upper triangle of the 6 x 6 state covariance
constexpr int kCovJacWords = 6 * kFitVars;    // J[6][7]

// Work items are chunks of Q consecutive queries, one warp each.  Q is the largest power of two <= AZ_COV_MAX_CHUNK
// that still leaves AZ_COV_WORK_ITEMS work items (1 below that): a batch with few queries per satellite (one query per
// object at a common time) spreads its segments -- each a serial set build and a few queries -- over the whole GPU,
// and a dense batch amortises a segment's set building over up to AZ_COV_MAX_CHUNK queries.  The defaults are chosen
// by measurement (DESIGN.md section 3, K10); the macros exist for measurement builds.  No result depends on Q.
#ifndef AZ_COV_MAX_CHUNK
#define AZ_COV_MAX_CHUNK 256
#endif
#ifndef AZ_COV_WORK_ITEMS
#define AZ_COV_WORK_ITEMS 2048
#endif
AZ_HD uint32_t cov_chunk(uint32_t m) {
    uint32_t q = AZ_COV_MAX_CHUNK;
    while (q > 1 && ((uint64_t)m + q - 1) / q < (uint64_t)AZ_COV_WORK_ITEMS) q >>= 1;
    return q;
}

// The variables of P: 7, or 6 when its B* row is all zero
AZ_HD int cov_nvar(const double *P) {
    for (int j = 0; j < kFitVars; ++j)
        if (P[fit_tri(j, kFitVars - 1)] != 0.0) return kFitVars;
    return kFitVars - 1;
}

// The satellite whose queries contain query q: the largest s < n with offsets[s] <= q (offsets non-decreasing)
AZ_HD uint32_t cov_first_sat(const uint32_t *offsets, uint32_t n, uint32_t q) {
    uint32_t lo = 0, hi = n;   // offsets[hi] > q
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (offsets[mid] <= q) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The zeros of a failed query
AZ_HD void cov_zero(double *J, int stride, double (&f0)[6], double (&sig)[kCovWords]) {
    for (int c = 0; c < 6; ++c) f0[c] = 0.0;
    for (int q = 0; q < kCovWords; ++q) sig[q] = 0.0;
    for (int q = 0; q < kCovJacWords; ++q) J[q * stride] = 0.0;
}

// Rows R, T, N of the RTN frame of TEME state f: R = r / |r|, N = r x v / |r x v|, T = N x R
AZ_HD void cov_rtn(const double (&f)[6], double (&R)[3][3]) {
    const double rn = std::sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
    const double h[3] = {f[1] * f[5] - f[2] * f[4], f[2] * f[3] - f[0] * f[5], f[0] * f[4] - f[1] * f[3]};
    const double hn = std::sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    for (int c = 0; c < 3; ++c) {
        R[0][c] = f[c] / rn;
        R[2][c] = h[c] / hn;
    }
    R[1][0] = R[2][1] * R[0][2] - R[2][2] * R[0][1];
    R[1][1] = R[2][2] * R[0][0] - R[2][0] * R[0][2];
    R[1][2] = R[2][0] * R[0][1] - R[2][1] * R[0][0];
}

// One query whose sets are built: eval(k, jdFull, ts, f) = the TEME state f[6] of set k (false when its cell fails),
// inv[1 + j] = 1 / step of variable j, P the 28 covariance words.  J receives the 6 x 7 Jacobian in the output frame,
// entry (c, j) at J[(c * kFitVars + j) * stride]; f0 the nominal TEME state; sig the 21 words of Sigma.
template <typename EvalFn>
AZ_HD uint8_t cov_query(EvalFn eval, int nvar, const double *inv, const double *P, double jdFull, double epochJd,
                        int frame, double *J, int stride, double (&f0)[6], double (&sig)[kCovWords]) {
    const double ts[1] = {mul_rn(sub_rn(jdFull, epochJd), 1440.0)};
    bool ok = eval(0, jdFull, ts, f0);
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int j = 0; j < kFitVars; ++j) {
        double f[6];
        if (j < nvar) ok = eval(1 + j, jdFull, ts, f) && ok;
        for (int c = 0; c < 6; ++c) J[(c * kFitVars + j) * stride] = j < nvar ? (f[c] - f0[c]) * inv[1 + j] : 0.0;
    }
    if (!ok) {
        cov_zero(J, stride, f0, sig);
        return kCovCellFailed;
    }
    if (frame == kCovFrameRtn) {
        double R[3][3];
        cov_rtn(f0, R);
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
        for (int j = 0; j < kFitVars; ++j) {
            for (int b = 0; b < 6; b += 3) {
                double u[3];
                for (int c = 0; c < 3; ++c) u[c] = J[((b + c) * kFitVars + j) * stride];
                for (int c = 0; c < 3; ++c)
                    J[((b + c) * kFitVars + j) * stride] = R[c][0] * u[0] + R[c][1] * u[1] + R[c][2] * u[2];
            }
        }
    }
    // Sigma = J P J^T: row a of J P, then its products with rows b >= a of J
    int q = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        double jp[kFitVars];
#pragma unroll
        for (int k = 0; k < kFitVars; ++k) {
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < kFitVars; ++j)
                s += J[(a * kFitVars + j) * stride] * P[j <= k ? fit_tri(j, k) : fit_tri(k, j)];
            jp[k] = s;
        }
#pragma unroll
        for (int b = a; b < 6; ++b, ++q) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < kFitVars; ++k) s += jp[k] * J[(b * kFitVars + k) * stride];
            sig[q] = s;
        }
    }
    return kCovOk;
}

}  // namespace az
