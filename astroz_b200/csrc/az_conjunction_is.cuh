// az_conjunction_is.cuh -- K15: importance-sampled collision probability of candidate conjunctions.  __host__
// __device__, so the kernels (az_conjunction_is.cu, the item loop of az_conjunction_mc_warp.cuh) and the host emulation
// (tests/host_emul/emul_conjunction_is.cu) run this source.
//
// The catalogue, candidates, samples, first, seed, factor, status rules and the pairing of normals with variables are
// K14's (az_conjunction_mc.cuh).  u in R^14 are K14's normals of sample k (0 .. 6 the primary's, 7 .. 13 the
// secondary's) and c in R^14 is the candidate's shift:
//   draw      z = u + c and x_k = x^ + D^1/2 L z for each row; then K14's sets, conj_tca over [-w, w], miss and the
//             failed / edge / hit rules;
//   weight    log w_k = -u . c - |c|^2 / 2 = log phi(z) - log phi(z - c), exactly;
//   estimate  Pc = (1 / N) sum over hits of w_k, N = samples: an unbiased estimate of P(hit) whatever c is.  A failed
//             draw is a non-hit, so where draws fail this is K14's hits / (N - failed) times (1 - P(failed)).
// The linear shift (kind kIsLinear) is built from K11's assessment of the nominal pair: its TCA, plane (x, y) and the
// in-plane miss d = (dr . x, dr . y).  J_o is K10's forward-difference Jacobian of row o's TEME position at the TCA
// (B* held when P's B* row is zero), G = [-Pi J_p D_p^1/2 L_p | Pi J_s D_s^1/2 L_s] the 2 x 14 map from normals to the
// in-plane miss (Pi the projection on x, y), and c = -G^T C+ d the least-norm shift with d + G c = 0, C = G G^T and C+
// its pseudo-inverse by the 2 x 2 eigen-decomposition (an eigenvalue <= 1e-14 trace counts as zero).  |c|^2 = d^T C+ d
// is the Mahalanobis distance of the nominal miss under C (K11's C2 up to the factor's pivot rule).
// Accumulation: each hit's v = exp(-u . c) and v^2 (v * v in fp64) are rounded to multiples of 2^-128 and summed as
// unsigned 256-bit integers (four u64 words, least significant first); a hit with v >= 2^31 enters neither sum and counts
// in `overflow`.  l0 = -|c|^2 / 2 is returned with the shift and is not accumulated, so the counts are integer sums:
// counts over [0, 2N) are those over [0, N) plus those over [N, 2N), as K14's.
#pragma once

#include "az_conjunction_mc.cuh"

namespace az {

// counts words: hits, edge, failed, overflow, V_hit[4], V2_hit[4]; proposal words: c[14], l0; sample words: dt_tca
// [min], miss [km], log w
constexpr int kIsCountWords = 12;
constexpr int kIsProposalWords = 15;
constexpr int kIsSampleWords = 3;
constexpr int kIsShift = 2 * kFitVars;          // 14
constexpr int kIsCountV = 4, kIsCountV2 = 8;    // first word of each 256-bit sum
constexpr double kIsEigenZero = 1e-14;          // eigenvalues <= this times the trace of C count as zero
constexpr double kIsVMax = 0x1p31;              // hits with v >= this count as overflow

// proposal kinds (ASTROZ_CONJ_IS_*)
enum IsKind : uint8_t { kIsLinear = 0, kIsGiven = 1, kIsPlain = 2 };

// The encounter plane of K11's TEME states fp, fs at the TCA: rows e[0] = x, e[1] = y and the in-plane miss
// d = (dr . x, dr . y); false when |dv| = 0 (no plane)
AZ_HD bool is_plane(const double (&fp)[6], const double (&fs)[6], double (&e)[2][3], double (&d)[2]) {
    double dr[3], dv[3];
    for (int c = 0; c < 3; ++c) {
        dr[c] = fs[c] - fp[c];
        dv[c] = fs[3 + c] - fp[3 + c];
    }
    const double speed = std::sqrt(dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2]);
    if (!(speed > 0.0)) return false;
    // conj_geometry's plane rule, restated here so K11's kernels keep their code
    double z[3];
    for (int c = 0; c < 3; ++c) z[c] = dv[c] / speed;
    const double along = dr[0] * z[0] + dr[1] * z[1] + dr[2] * z[2];
    double(&x)[3] = e[0];
    for (int c = 0; c < 3; ++c) x[c] = dr[c] - along * z[c];
    const double dn = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    if (dn > 0.0) {
        for (int c = 0; c < 3; ++c) x[c] /= dn;
    } else {   // exact hit: x from the TEME axis least aligned with z (the first on a tie)
        int k = 0;
        for (int c = 1; c < 3; ++c)
            if (std::fabs(z[c]) < std::fabs(z[k])) k = c;
        for (int c = 0; c < 3; ++c) x[c] = (c == k ? 1.0 : 0.0) - z[k] * z[c];
        const double xn = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        for (int c = 0; c < 3; ++c) x[c] /= xn;
    }
    e[1][0] = z[1] * x[2] - z[2] * x[1];
    e[1][1] = z[2] * x[0] - z[0] * x[2];
    e[1][2] = z[0] * x[1] - z[1] * x[0];
    for (int r = 0; r < 2; ++r) d[r] = dr[0] * e[r][0] + dr[1] * e[r][1] + dr[2] * e[r][2];
    return true;
}

// |c|^2 of a proposal's shift, in the order every proposal kind forms it
AZ_HD double is_norm2(const double *c) {
    double cc = 0.0;
    for (int b = 0; b < kIsShift; ++b) cc += c[b] * c[b];
    return cc;
}

// l0 = -|c|^2 / 2 (+0 for c = 0)
AZ_HD double is_log_scale(double cc) { return 0.0 - 0.5 * cc; }

// Row o's block of G: sign Pi J D^1/2 L (2 x 7), J the 6 x 7 TEME Jacobian (row-major), F the row's factor
AZ_HD void is_row_map(const double *J, const McFactor &F, const double (&e)[2][3], double sign, double (&G)[2][kFitVars]) {
    for (int r = 0; r < 2; ++r) {
        double M[kFitVars];   // Pi J: the plane row r of the position block
        for (int a = 0; a < kFitVars; ++a)
            M[a] = e[r][0] * J[a] + e[r][1] * J[kFitVars + a] + e[r][2] * J[2 * kFitVars + a];
        for (int b = 0; b < kFitVars; ++b) {
            double s = 0.0;
            for (int a = b; a < kFitVars; ++a) s += M[a] * F.sd[a] * F.L[fit_tri(b, a)];
            G[r][b] = sign * s;
        }
    }
}

// The least-norm shift c = -G^T C+ d and |c|^2 from G = [Gp | Gs] and d; false when C = G G^T is zero
AZ_HD bool is_linear_shift(const double (&Gp)[2][kFitVars], const double (&Gs)[2][kFitVars], const double (&d)[2],
                           double (&c)[kIsShift], double &cc) {
    double C[3] = {0.0, 0.0, 0.0};   // xx, xy, yy
    for (int b = 0; b < kFitVars; ++b) {
        C[0] += Gp[0][b] * Gp[0][b] + Gs[0][b] * Gs[0][b];
        C[1] += Gp[0][b] * Gp[1][b] + Gs[0][b] * Gs[1][b];
        C[2] += Gp[1][b] * Gp[1][b] + Gs[1][b] * Gs[1][b];
    }
    const double tr = C[0] + C[2];
    for (int q = 0; q < kIsShift; ++q) c[q] = 0.0;
    cc = 0.0;
    if (!(tr > 0.0)) return false;
    // eigenvalues l1 >= l2 (l2 = det / l1, as conj_pc_params) along (cos phi, sin phi) and (-sin phi, cos phi)
    const double half = 0.5 * tr, q = std::hypot(0.5 * (C[0] - C[2]), C[1]);
    const double l1 = half + q, det = C[0] * C[2] - C[1] * C[1];
    const double l2 = det > 0.0 ? det / l1 : 0.0;
    const double phi = 0.5 * std::atan2(2.0 * C[1], C[0] - C[2]), cp = std::cos(phi), sp = std::sin(phi);
    const double zero = kIsEigenZero * tr;
    const double p1 = cp * d[0] + sp * d[1], p2 = -sp * d[0] + cp * d[1];   // d in the eigenvectors
    const double a1 = l1 > zero ? p1 / l1 : 0.0, a2 = l2 > zero ? p2 / l2 : 0.0;
    const double y[2] = {cp * a1 - sp * a2, sp * a1 + cp * a2};            // C+ d
    for (int b = 0; b < kFitVars; ++b) {
        c[b] = -(Gp[0][b] * y[0] + Gp[1][b] * y[1]);
        c[kFitVars + b] = -(Gs[0][b] * y[0] + Gs[1][b] * y[1]);
    }
    cc = is_norm2(c);
    return true;
}

// Row o's shift added to its normals: z += c_o, and u . c_o over the row (u the normals before the shift)
AZ_HD double is_shift_normals(const double *co, double (&z)[kFitVars]) {
    double uc = 0.0;
    for (int v = 0; v < kFitVars; ++v) {
        uc += z[v] * co[v];
        z[v] += co[v];
    }
    return uc;
}

// x >= 0, x < 2^159: the nearest integer to x 2^128 (ties to even) added to the 256-bit sum S (four u64, least
// significant first)
AZ_HD void is_add_fixed(double x, uint64_t (&S)[4]) {
    const double r = rint(x * 0x1p128);   // the scaling by a power of two is exact
    if (!(r > 0.0)) return;
    int e;
    const double f = std::frexp(r, &e);                              // r = f 2^e, f in [0.5, 1)
    uint64_t mant = (uint64_t)std::ldexp(f, 53);
    int sh = e - 53;
    uint64_t w[4] = {0, 0, 0, 0};
    if (sh <= 0) {
        w[0] = mant >> -sh;                                        // exact: r is an integer
    } else {
        const int q = sh >> 6, b = sh & 63;
        w[q] = mant << b;
        if (b && q + 1 < 4) w[q + 1] = mant >> (64 - b);
    }
    uint64_t carry = 0;
    for (int k = 0; k < 4; ++k) {
        const uint64_t t = S[k] + carry;
        const uint64_t c1 = t < carry ? 1 : 0;
        S[k] = t + w[k];
        carry = c1 + (S[k] < w[k] ? 1 : 0);
    }
}

// One hit of weight factor v = exp(-u . c): into V and V2, or `overflow` when v >= 2^31
AZ_HD void is_hit(double v, uint64_t (&V)[4], uint64_t (&V2)[4], uint64_t &overflow) {
    if (!(v < kIsVMax)) {
        ++overflow;
        return;
    }
    is_add_fixed(v, V);
    is_add_fixed(v * v, V2);
}

}  // namespace az
