// az_avoid.cuh -- K16: collision-avoidance manoeuvre trials.  __host__ __device__, so the kernels (az_avoid.cu) and the
// host emulation (tests/host_emul/emul_avoid.cu) run this source.
//
// The catalogue and candidates are K11's.  The primary of a candidate is the object that burns.  Trial k takes
// candidate c = candidate[k], a burn time burn_jd + burn_fr, an impulsive dv_rtn [km/s] in the primary's RTN frame at the
// burn and optionally sigma [km/s], the 1-sigma execution error per RTN axis (independent axes, uncorrelated with the
// orbit error):
//   burn        ts_b = ((burn_jd + burn_fr) - epoch) * 1440, formed as K10 forms tsince; it must come before the
//               window: ts_b <= ts0 - w (ts0 the candidate's guess tsince, w its half window), else BAD_TRIAL.  x(t_b)
//               and J (6 x 7, TEME) are K10's nominal and Jacobian of the primary's row at t_b (B* held when P's B* row
//               is zero); the post-burn state is x(t_b) + [0; R dv], R = [R^ T^ N^] of x(t_b) (cov_rtn);
//   conversion  K8's fit (launch_fit, then launch_fit_deep) from the primary's own words to the one TEME state at t_b,
//               B* held at the primary's B*, K13's weights and iteration limit; the epoch stays the primary's epoch, so
//               the new trajectory meets the post-burn state at t_b and shares the nominal's drag history (a re-epoched
//               set would restart SGP4's drag polynomials at the burn, and even a zero burn would drift from the
//               nominal).  The class follows the initial set.  A fit that does not converge, residuals above
//               kIodConvDr / kIodConvDv, or a new set that K10 cannot build or propagate under the primary's model
//               byte (a burn that moves the period across 225 min) is CONVERSION_FAILED;
//   zero burn   dv = (0, 0, 0): the new row is the primary's words, copied, J' = J and A = I; the fit is not run, so the
//               trial's record is K11's record of the nominal pair bit for bit (with sigma = 0);
//   transport   J' = K10's Jacobian of the new set at t_b, J'6 its six orbital columns; A (7 x 7): rows 0-5 are
//               J'6^-1 (J - J'(:, B*) e_B*^T), row 6 is e_B*^T (B* is carried over); P' = A P A^T + [J'6^-1 [0 0; 0
//               R diag(sigma^2) R^T] J'6^-T, 0; 0, 0].  A held B* stays held.  J'6^-1 by avoid_solve6: rows, then
//               columns, equilibrated to a largest |entry| of 1, LU with partial pivoting (the largest |entry| of the
//               column, the first row on a tie); a pivot |u| <= kAvoidPivot or a scale that is 0 or not finite is
//               singular: CONVERSION_FAILED;
//   reassess    K11 unchanged on (new row with P' and the primary's model byte, the secondary's row) with the
//               candidate's guess, window and radius.
// Statuses, first match: BAD_TRIAL / BAD_PAIR (candidate index >= m, burn not before the window / the candidate's rows);
// INIT_FAILED (a model byte > 1) or K10's INIT_FAILED / CELL_FAILED of the primary at t_b; CONVERSION_FAILED; K11's
// statuses of the post-burn pair.  A trial that is not assessed (stopped before K11, or K11's INIT_FAILED / CELL_FAILED
// of the post-burn pair) has every output zero.
// The returned row is an ordinary catalogue row: appended to the catalogue it gives the same K11 record bit for bit.
// A trial's bytes depend on its own inputs, its candidate and its two rows alone.
#pragma once

#include "az_conjunction.cuh"
#include "az_iod.cuh"

namespace az {

// the new status bytes, continuing ASTROZ_CONJ_*
constexpr uint8_t kConjConversionFailed = 7, kConjBadTrial = 8;
constexpr double kAvoidPivot = 1e-12;   // the least |pivot| of the equilibrated J'6

// Device pointers (host pointers in the emulation).
struct AvoidArgs {
    const double *elements = nullptr;    // [8][n]
    const double *covariance = nullptr;  // [n][28]
    const uint8_t *model = nullptr;      // [n], nullable (all 0)
    uint32_t n = 0;
    const uint32_t *primary = nullptr, *secondary = nullptr;  // [m] rows
    const double *jd = nullptr, *fr = nullptr;                 // [m] guess times
    const double *window = nullptr;      // [m] half window [min]
    const double *hbr = nullptr;         // [m] combined hard-body radius [km]
    uint32_t m = 0;
    const uint32_t *candidate = nullptr; // [t]
    const double *burnJd = nullptr, *burnFr = nullptr;         // [t]
    const double *dv = nullptr;          // [t][3] RTN [km/s]
    const double *dvSigma = nullptr;     // [t][3] RTN [km/s], nullable (all 0)
    uint32_t t = 0;
    int grav = 1;
    GravConsts g{};
    void *scratch = nullptr;             // avoid_scratch_bytes(t)
    double *record = nullptr;            // [t][13]
    double *newElements = nullptr;       // [t][8], nullable
    double *newCovariance = nullptr;     // [t][28], nullable
    double *residual = nullptr;          // [t][2], nullable
    uint8_t *status = nullptr;           // [t] ASTROZ_CONJ_*
};

// The scratch: the catalogue of K10's first pass (one primary copy per trial, queried at t_b), the conversion batch and
// the fit's outputs, K10's second pass, and K11's catalogue of two rows per trial (new row 2k, secondary copy 2k + 1)
struct AvoidScratch {
    double *el1;        // [8][t] primary copies
    double *P1;         // [t][28] their P
    double *state;      // [t][6] x(t_b)
    double *sig;        // [t][21] K10's Sigma (not used; both passes write it)
    double *J, *J2;     // [t][42] J, J'
    double *init;       // [8][t] the fit's initial sets
    double *pos, *vel;  // [t][3] the post-burn state
    double *fitted;     // [8][t]
    double *rms;        // [t][2]
    double *el2;        // [8][2t]
    double *P2;         // [2t][28]
    double *jd2, *fr2, *win2, *hbr2;   // [t] K11's candidates
    uint32_t *offsets;  // [t + 1] = 0, 1, ..., t
    uint32_t *iters;    // [t]
    uint32_t *pri2, *sec2;             // [t]
    uint8_t *model1;    // [t]
    uint8_t *model2;    // [2t]
    uint8_t *st;        // [t] the trial's status before K11 (kConjOk: still running)
    uint8_t *cov1St, *fitSt, *cov2St;  // [t]
};

constexpr size_t kAvoidDoubles = 8 + kFitN + 6 + kCovWords + 2 * kCovJacWords + 8 + 6 + 8 + 2 + 16 + 2 * kFitN + 4;

AZ_HD size_t avoid_scratch_bytes(uint32_t t) {
    return (size_t)t * kAvoidDoubles * 8 + ((size_t)4 * t + 1) * 4 + (size_t)8 * t;
}

AZ_HD AvoidScratch avoid_scratch(void *p, uint32_t t) {
    AvoidScratch s;
    double *d = static_cast<double *>(p);
    auto take = [&d](size_t words) {
        double *q = d;
        d += words;
        return q;
    };
    s.el1 = take((size_t)8 * t);
    s.P1 = take((size_t)kFitN * t);
    s.state = take((size_t)6 * t);
    s.sig = take((size_t)kCovWords * t);
    s.J = take((size_t)kCovJacWords * t);
    s.J2 = take((size_t)kCovJacWords * t);
    s.init = take((size_t)8 * t);
    s.pos = take((size_t)3 * t);
    s.vel = take((size_t)3 * t);
    s.fitted = take((size_t)8 * t);
    s.rms = take((size_t)2 * t);
    s.el2 = take((size_t)16 * t);
    s.P2 = take((size_t)2 * kFitN * t);
    s.jd2 = take(t);
    s.fr2 = take(t);
    s.win2 = take(t);
    s.hbr2 = take(t);
    s.offsets = reinterpret_cast<uint32_t *>(d);
    s.iters = s.offsets + t + 1;
    s.pri2 = s.iters + t;
    s.sec2 = s.pri2 + t;
    s.model1 = reinterpret_cast<uint8_t *>(s.sec2 + t);
    s.model2 = s.model1 + t;
    s.st = s.model2 + 2 * (size_t)t;
    s.cov1St = s.st + t;
    s.fitSt = s.cov1St + t;
    s.cov2St = s.fitSt + t;
    return s;
}

AZ_HD bool avoid_zero_burn(const double *dv) { return dv[0] == 0.0 && dv[1] == 0.0 && dv[2] == 0.0; }

// Step 1, trial k: the checks, then row k of K10's first catalogue (the primary's words and P, or an unbuildable set
// e = -1 when the trial is already decided) and its query offsets
AZ_HD void avoid_prepare(const AvoidArgs &a, const AvoidScratch &s, uint32_t k) {
    const uint32_t c = a.candidate[k];
    uint8_t st = kConjOk;
    uint32_t p = 0;
    if (c >= a.m) {
        st = kConjBadTrial;
    } else {
        p = a.primary[c];
        const uint32_t q = a.secondary[c];
        if (p >= a.n || q >= a.n || p == q) {
            st = kConjBadPair;
        } else {
            const double epoch = a.elements[p];
            const double tsb = pairs_tsince_deep(add_rn(a.burnJd[k], a.burnFr[k]), epoch);
            const double ts0 = pairs_tsince_deep(add_rn(a.jd[c], a.fr[c]), epoch);
            if (!(tsb <= ts0 - a.window[c])) st = kConjBadTrial;
            else if (a.model && a.model[p] > 1) st = kConjInitFailed;
            else if (a.model && a.model[q] > 1) st = kConjInitFailed;
        }
    }
    const bool ok = st == kConjOk;
    for (int w = 0; w < 8; ++w) s.el1[(size_t)w * a.t + k] = ok ? a.elements[(size_t)w * a.n + p] : (w == 2 ? -1.0 : 0.0);
    for (int w = 0; w < kFitN; ++w) s.P1[(size_t)k * kFitN + w] = ok ? a.covariance[(size_t)p * kFitN + w] : 0.0;
    s.model1[k] = ok && a.model ? a.model[p] : 0;
    s.st[k] = st;
    s.offsets[k] = k;
    if (k + 1 == a.t) s.offsets[a.t] = a.t;
}

// Step 3, trial k: the status after K10's first pass and the conversion batch: the post-burn state and the fit's initial
// set (the primary's words; e = -1 for a zero burn or a decided trial, which the fit refuses at once)
AZ_HD void avoid_burn(const AvoidArgs &a, const AvoidScratch &s, uint32_t k) {
    uint8_t st = s.st[k];
    if (st == kConjOk && s.cov1St[k] != kCovOk) st = s.cov1St[k] == kCovInitFailed ? kConjInitFailed : kConjCellFailed;
    s.st[k] = st;
    const double *dv = a.dv + (size_t)k * 3;
    const bool convert = st == kConjOk && !avoid_zero_burn(dv);
    double x[6], R[3][3];
    for (int c = 0; c < 6; ++c) x[c] = convert ? s.state[(size_t)k * 6 + c] : 0.0;
    if (convert) cov_rtn(x, R);
    for (int c = 0; c < 3; ++c) {
        s.pos[(size_t)k * 3 + c] = x[c];
        s.vel[(size_t)k * 3 + c] = convert ? x[3 + c] + (R[0][c] * dv[0] + R[1][c] * dv[1] + R[2][c] * dv[2]) : 0.0;
    }
    for (int w = 0; w < 8; ++w) s.init[(size_t)w * a.t + k] = convert ? s.el1[(size_t)w * a.t + k] : (w == 2 ? -1.0 : 0.0);
}

// X = J'6^-1 B in place (B: 6 x NB), J'6 = columns 0-5 of the row-major 6 x 7 words Jp (file comment); false: singular
template <int NB>
AZ_HD bool avoid_solve6(const double *Jp, double (&B)[6][NB]) {
    double S[6][6], dr[6], dc[6];
    for (int i = 0; i < 6; ++i) {
        double mx = 0.0;
        for (int j = 0; j < 6; ++j) mx = std::fmax(mx, std::fabs(Jp[i * kFitVars + j]));
        if (!(mx > 0.0) || !(mx < INFINITY)) return false;
        dr[i] = 1.0 / mx;
        for (int j = 0; j < 6; ++j) S[i][j] = Jp[i * kFitVars + j] * dr[i];
    }
    for (int j = 0; j < 6; ++j) {
        double mx = 0.0;
        for (int i = 0; i < 6; ++i) mx = std::fmax(mx, std::fabs(S[i][j]));
        if (!(mx > 0.0)) return false;
        dc[j] = 1.0 / mx;
        for (int i = 0; i < 6; ++i) S[i][j] *= dc[j];
    }
    for (int i = 0; i < 6; ++i)
        for (int b = 0; b < NB; ++b) B[i][b] *= dr[i];
    for (int j = 0; j < 6; ++j) {
        int piv = j;
        for (int i = j + 1; i < 6; ++i)
            if (std::fabs(S[i][j]) > std::fabs(S[piv][j])) piv = i;
        if (!(std::fabs(S[piv][j]) > kAvoidPivot)) return false;
        if (piv != j) {
            for (int q = 0; q < 6; ++q) {
                const double u = S[j][q];
                S[j][q] = S[piv][q];
                S[piv][q] = u;
            }
            for (int b = 0; b < NB; ++b) {
                const double u = B[j][b];
                B[j][b] = B[piv][b];
                B[piv][b] = u;
            }
        }
        for (int i = j + 1; i < 6; ++i) {
            const double l = S[i][j] / S[j][j];
            for (int q = j + 1; q < 6; ++q) S[i][q] -= l * S[j][q];
            for (int b = 0; b < NB; ++b) B[i][b] -= l * B[j][b];
        }
    }
    for (int j = 5; j >= 0; --j)
        for (int b = 0; b < NB; ++b) {
            double v = B[j][b];
            for (int q = j + 1; q < 6; ++q) v -= S[j][q] * B[q][b];
            B[j][b] = v / S[j][j];
        }
    for (int j = 0; j < 6; ++j)
        for (int b = 0; b < NB; ++b) B[j][b] *= dc[j];
    return true;
}

// P' words (28) of avoid_transport's rule.  J and Jp: row-major 6 x 7 words of J and J'; x the pre-burn TEME state;
// zero: the zero burn (A = I, P copied).  False: J'6 is singular.
AZ_HD bool avoid_covariance(const double *J, const double *Jp, const double *P, const double (&x)[6],
                            const double *sigma, bool zero, double *Pn) {
    const bool exec = sigma && (sigma[0] != 0.0 || sigma[1] != 0.0 || sigma[2] != 0.0);
    if (zero && !exec) {
        for (int w = 0; w < kFitN; ++w) Pn[w] = P[w];
        return true;
    }
    // B = [J - J'(:, B*) e_B*^T | [0; R^T diag(sigma)]], solved in place to [A(0:6, :) | G]
    double B[6][kFitVars + 3];
    double R[3][3];
    cov_rtn(x, R);
    for (int i = 0; i < 6; ++i) {
        for (int j = 0; j < kFitVars; ++j)
            B[i][j] = zero ? 0.0 : (j < 6 ? J[i * kFitVars + j] : J[i * kFitVars + j] - Jp[i * kFitVars + j]);
        for (int q = 0; q < 3; ++q) B[i][kFitVars + q] = i < 3 || !exec ? 0.0 : R[q][i - 3] * sigma[q];
    }
    if (!avoid_solve6(Jp, B)) return false;
    if (zero) {
        for (int w = 0; w < kFitN; ++w) Pn[w] = P[w];
    } else {   // A P A^T, A's row 6 = e_B*
        double AP[kFitVars][kFitVars];
        for (int i = 0; i < kFitVars; ++i)
            for (int q = 0; q < kFitVars; ++q) {
                double v = 0.0;
                for (int j = 0; j < kFitVars; ++j) {
                    const double aij = i < 6 ? B[i][j] : (j == 6 ? 1.0 : 0.0);
                    v += aij * P[j <= q ? fit_tri(j, q) : fit_tri(q, j)];
                }
                AP[i][q] = v;
            }
        for (int i = 0; i < kFitVars; ++i)
            for (int q = i; q < kFitVars; ++q) {
                double v = 0.0;
                for (int j = 0; j < kFitVars; ++j) v += AP[i][j] * (q < 6 ? B[q][j] : (j == 6 ? 1.0 : 0.0));
                Pn[fit_tri(i, q)] = v;
            }
    }
    if (exec)
        for (int i = 0; i < 6; ++i)
            for (int q = i; q < 6; ++q) {
                double v = 0.0;
                for (int b = 0; b < 3; ++b) v += B[i][kFitVars + b] * B[q][kFitVars + b];
                Pn[fit_tri(i, q)] += v;
            }
    return true;
}

// Step 6, trial k: the conversion's status, the new row and P', and K11's candidate k over rows (2k, 2k + 1) of its
// catalogue (a decided trial: the pair (2k, 2k), which K11 answers at once with BAD_PAIR)
AZ_HD void avoid_transport(const AvoidArgs &a, const AvoidScratch &s, uint32_t k) {
    uint8_t st = s.st[k];
    const double *dv = a.dv + (size_t)k * 3;
    const bool zero = avoid_zero_burn(dv);
    if (st == kConjOk && !zero) {
        const double dr = s.rms[2 * (size_t)k], dvr = s.rms[2 * (size_t)k + 1];
        if (!(s.fitSt[k] == kFitConverged && dr <= kIodConvDr && dvr <= kIodConvDv) || s.cov2St[k] != kCovOk)
            st = kConjConversionFailed;
    }
    const uint32_t c = st == kConjOk ? a.candidate[k] : 0;
    const uint32_t q = st == kConjOk ? a.secondary[c] : 0;
    double Pn[kFitN];
    if (st == kConjOk) {
        double x[6];
        for (int w = 0; w < 6; ++w) x[w] = s.state[(size_t)k * 6 + w];
        const double *J = s.J + (size_t)k * kCovJacWords;
        const double *Jp = zero ? J : s.J2 + (size_t)k * kCovJacWords;
        if (!avoid_covariance(J, Jp, s.P1 + (size_t)k * kFitN, x, a.dvSigma ? a.dvSigma + (size_t)k * 3 : nullptr, zero,
                              Pn))
            st = kConjConversionFailed;
    }
    const bool ok = st == kConjOk;
    const size_t n2 = 2 * (size_t)a.t, r0 = 2 * (size_t)k, r1 = r0 + 1;
    const double *nw = zero ? s.el1 : s.fitted;
    for (int w = 0; w < 8; ++w) {
        s.el2[w * n2 + r0] = ok ? nw[(size_t)w * a.t + k] : 0.0;
        s.el2[w * n2 + r1] = ok ? a.elements[(size_t)w * a.n + q] : 0.0;
    }
    for (int w = 0; w < kFitN; ++w) {
        s.P2[r0 * kFitN + w] = ok ? Pn[w] : 0.0;
        s.P2[r1 * kFitN + w] = ok ? a.covariance[(size_t)q * kFitN + w] : 0.0;
    }
    s.model2[r0] = s.model1[k];
    s.model2[r1] = ok && a.model ? a.model[q] : 0;
    s.pri2[k] = (uint32_t)r0;
    s.sec2[k] = ok ? (uint32_t)r1 : (uint32_t)r0;
    s.jd2[k] = ok ? a.jd[c] : 0.0;
    s.fr2[k] = ok ? a.fr[c] : 0.0;
    s.win2[k] = ok ? a.window[c] : 0.0;
    s.hbr2[k] = ok ? a.hbr[c] : 0.0;
    s.st[k] = st;
}

// Step 8, trial k: the status by precedence, zeros for a trial that is not assessed, the optional outputs.  K11 wrote
// record[k] and status[k].
AZ_HD void avoid_finish(const AvoidArgs &a, const AvoidScratch &s, uint32_t k) {
    const uint8_t st = s.st[k];
    const bool zero = avoid_zero_burn(a.dv + (size_t)k * 3);
    if (st != kConjOk) {
        a.status[k] = st;
        for (int w = 0; w < kConjRecordWords; ++w) a.record[(size_t)k * kConjRecordWords + w] = 0.0;
    }
    // assessed: K11 ran and did not fail on the post-burn pair (its INIT_FAILED / CELL_FAILED zero the record)
    const uint8_t k11 = st == kConjOk ? a.status[k] : st;
    const bool ok = st == kConjOk && k11 != kConjInitFailed && k11 != kConjCellFailed;
    const size_t n2 = 2 * (size_t)a.t, r0 = 2 * (size_t)k;
    if (a.newElements)
        for (int w = 0; w < 8; ++w) a.newElements[(size_t)k * 8 + w] = ok ? s.el2[w * n2 + r0] : 0.0;
    if (a.newCovariance)
        for (int w = 0; w < kFitN; ++w) a.newCovariance[(size_t)k * kFitN + w] = ok ? s.P2[r0 * kFitN + w] : 0.0;
    if (a.residual)
        for (int w = 0; w < 2; ++w) a.residual[(size_t)k * 2 + w] = ok && !zero ? s.rms[2 * (size_t)k + w] : 0.0;
}

}  // namespace az
